#!/usr/bin/env python
"""Cost of the PPO training options on one GPU, one option per command:

    python tools/option_cost.py OPTION [--steps K] [--warmup W] [--repeats R] [--pool P]    (step options)
    python tools/option_cost.py OPTION [--states T] [--repeats R] [--launches N]            (iteration options)

A step option runs the bench.py workload (HLG graphs of seed 111, 256 per step, --pool resident minibatches with
LPT-balanced ids) on one engine per configuration and model: --warmup steps each, then --repeats windows of --steps
steps, the engines alternating, timed with CUDA events.  An iteration option runs whole PPOUpdater.update_params
iterations over --states HLG states (the bench.py graphs, 512 distinct tiled; minibatches of 256, 4 epochs) on one
updater per configuration: one warm-up iteration each, then --repeats rounds, the updaters alternating, np.random
seeded before every iteration, the host clock around each synchronised iteration; then it times the option's own
kernels over --launches calls.  Prints one JSON line with the card's name and power limit.  Writes nothing, and only
reads the device's settings.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload)
from drl_urban_planning_b200 import _lib, params as PL  # noqa: E402
from drl_urban_planning_b200.engine import Engine  # noqa: E402
from drl_urban_planning_b200.packing import infer_caps, pack_and_upload, pack_states  # noqa: E402
from drl_urban_planning_b200.ppo import PPOUpdater  # noqa: E402
from mlp_step_bench import card  # noqa: E402

B = bench.BATCH


def clocks():
    """The SM clock and the active throttle reasons as nvidia-smi reports them now; nothing is set."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20).stdout
        sm, sm_max, reasons = (x.strip() for x in out.strip().split(",")[:3])
        return {"sm_clock": sm, "sm_clock_max": sm_max, "throttle_reasons_active": reasons}
    except Exception:
        return {"sm_clock": None, "sm_clock_max": None, "throttle_reasons_active": None}


def event_ms(fn, warmup, calls):
    """CUDA-event ms per call over the back-to-back calls fn(0) .. fn(calls - 1), after `warmup` untimed ones."""
    for i in range(warmup):
        fn(i)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(calls):
        fn(i)
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / calls


def initial(model, sgnn_init=PL.default_init):
    """The initial parameters: the rl-mlp's from its layout, the SGNN's from `sgnn_init`."""
    return (PL.MLP.default_init if model == "mlp" else sgnn_init)(bench.SEED)


def report(opt, head, models):
    """The JSON line: a one-model option lists its configurations and extra fields at the top level."""
    if len(opt["models"]) > 1:
        return dict(head, models=models)
    (res,) = models.values()
    return dict(head, configs={c: res.pop(c) for c in opt["configs"]}, **res)


# ------------------------------------------------------------------------------------------------- step windows
def step_windows(opt, args):
    dev = torch.device("cuda", 0)
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, args.pool)
    blob = pack_states(states).to(dev)
    total = len(states)
    rng = np.random.default_rng(bench.SEED)
    f32 = lambda x: torch.as_tensor(x.astype(np.float32), device=dev)  # noqa: E731
    adv, ret = f32(rng.standard_normal(total)), f32(rng.standard_normal(total))
    fixed = f32(rng.normal(-3.0, 0.3, total)) if opt["logp"] == "normal" else None
    exps = torch.ones(total, dtype=torch.float32, device=dev)
    act = torch.as_tensor(actions, device=dev)
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    before = clocks() if opt.get("clocks") else None
    step = opt.get("step", fused_step)
    models = {}
    for model in opt["models"]:
        lay, flat = PL.MLP if model == "mlp" else PL.SGNN, initial(model, opt["init"])
        engines = {c: Engine(dev, blob.n_cap, blob.e_cap, model=model, **{"clip_mode": _lib.CLIP_NEVER, **kw})
                   for c, kw in opt["configs"].items()}
        r = SimpleNamespace(model=model, lay=lay, flat=flat, engines=engines, blob=blob, act=act, adv=adv, ret=ret,
                            fixed=fixed, exps=exps, pool=args.pool, steps=args.steps, step=step,
                            params={c: torch.as_tensor(flat, device=dev).clone() for c in engines},
                            grads={c: e.new_grad_buffer() for c, e in engines.items()},
                            so=engines["off"].stat_offset)
        if opt["logp"] != "normal":            # from a forward pass at parameters perturbed by a factor 1 + s N(0, 1)
            pert = r.params["off"] * (1.0 + opt["logp"] * torch.randn(
                r.params["off"].shape, device=dev, generator=torch.Generator(dev).manual_seed(3)))
            out = engines["off"].forward(blob, pert, act, cand_log_probs=opt.get("cand", False))
            r.values, r.fixed, r.cand = out[0], out[1], out[3] if opt.get("cand") else None
        r.ids = [torch.as_tensor(engines["off"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32),
                                 device=dev) for m in range(args.pool)]
        if "setup" in opt:
            opt["setup"](r)
        for c in engines:
            for i in range(args.warmup):
                step(r, c, i)
        torch.cuda.synchronize()
        if "check" in opt:
            opt["check"](r)
        r.res = {c: {"ms_per_step": []} for c in engines}
        r.done = dict.fromkeys(engines, args.warmup)
        order = list(engines)
        for w in range(args.repeats):
            k = w % len(order) if opt.get("rotate") else 0
            for c in order[k:] + order[:k]:
                launches0 = engines[c].launches
                r.res[c]["ms_per_step"].append(event_ms(lambda i: step(r, c, r.done[c] + i), 0, args.steps))
                r.res[c]["gpu_launches_per_step"] = (engines[c].launches - launches0) / args.steps
                r.done[c] += args.steps
        for ms in r.res.values():
            ms.update(median_ms=float(np.median(ms["ms_per_step"])),
                      spread_ms=float(max(ms["ms_per_step"]) - min(ms["ms_per_step"])))
        extra = opt["finish"](r) if "finish" in opt else None
        models[model] = dict(r.res, **(extra or {}))
    head = dict(workload=f"hlg, {B} graphs per step, {args.pool} minibatches, fused "
                         f"{'SGNN ' if len(models) == 1 else ''}step", steps=args.steps, repeats=args.repeats,
                card=card() if before is None else dict(card(), before=before, after_last_window=clocks()))
    return report(opt, head, models)


def inputs(r, c, adv=None):
    return (r.blob, r.params[c], r.act, r.adv if adv is None else adv, r.ret, r.fixed, r.exps, 1.0 / B, 1.0 / B)


def fused_step(r, c, i, adv=None, **refs):
    r.engines[c].ppo_step(*inputs(r, c, adv), ids=r.ids[i % r.pool], out=r.grads[c], **refs)


def value_clip_setup(r):
    r.order, r.norm_adv = torch.cat(r.ids), r.adv.clone()


def value_clip_step(r, c, i):
    adv = None
    if c == "both":
        if i % r.pool == 0:                    # the top of an epoch
            r.engines[c].normalize_advantages(r.adv, r.exps, r.order, B, out=r.norm_adv)
        adv = r.norm_adv
    fused_step(r, c, i, adv, old_values=None if c == "off" else r.values)


def kl_stop_check(r):
    assert float(r.grads["skipped"][r.so + 14]) == 1.0, "the tiny target stopped the first step; later ones are skipped"


def kl_stop_finish(r):
    return {"off_armed_bit_identical": bool(torch.equal(r.params["off"], r.params["armed"]) and all(
        np.array_equal(a, b) for a, b in zip(r.engines["off"].get_opt_state(), r.engines["armed"].get_opt_state())))}


def grad_clip_step(r, c, i):
    if c != "two_call":
        return fused_step(r, c, i)
    r.engines[c].ppo_grad(*inputs(r, c), ids=r.ids[i % r.pool], out=r.grads[c])
    r.engines[c].apply(r.params[c], r.grads[c])


def grad_clip_finish(r):
    for c, res in r.res.items():
        res["last_norm_slot17"] = float(r.grads[c][r.so + 17])


def nonfinite_guard_finish(r):
    for c, res in r.res.items():
        res.update(last_norm_slot17=float(r.grads[c][r.so + 17]), last_skipped_slot19=float(r.grads[c][r.so + 19]),
                   params_finite=bool(torch.isfinite(r.params[c]).all()))


def param_groups_setup(r):
    n = len(r.lay.slots)
    for c in ("one", "frozen"):
        trained = [c == "one" or sl.owner != "enc" for sl in r.lay.slots.values()]
        r.engines[c].set_param_groups([r.engines[c].lr] * n, [0.0] * n, trained)


def param_groups_finish(r):
    enc = r.lay.encoder_end                    # the frozen encoder did not move
    r.res["frozen"]["encoder_unchanged"] = bool(torch.equal(r.params["frozen"][:enc].cpu(),
                                                            torch.as_tensor(r.flat[:enc])))


def adam_options_setup(r):
    n = len(r.lay.slots)
    # the context's lr is upb_create's (double)(float)lr: the table takes the same value
    r.engines["table"].set_param_groups([float(np.float32(r.engines["table"].lr))] * n, [0.0] * n, [True] * n)
    for c in ("adamw", "amsgrad"):
        r.engines[c].set_weight_decay(0.01)
        r.engines[c].set_adam((0.9, 0.999), 1e-8, amsgrad=c == "amsgrad", decoupled_weight_decay=True)


def adam_options_finish(r):
    # the table at the default settings is the default step, bit for bit (SGNN only: the rl-mlp land-use backward sums a
    # node's candidates with shared-memory atomics, so its rows on these graphs differ run to run)
    if r.model == "sgnn":
        r.res["table"]["params_equal_off"] = bool(torch.equal(r.params["table"], r.params["off"]))


def adaptive_lr_finish(r):
    decisions = []
    for i in range(r.steps):                   # untimed: the decisions of as many more steps
        r.step(r, "desired_kl", r.done["desired_kl"] + i)
        decisions.append(r.grads["desired_kl"][r.so + 22].clone())
    d = torch.stack(decisions).cpu().numpy()
    r.res["desired_kl"]["decisions"] = dict(up=int((d > 0).sum()), down=int((d < 0).sum()), none=int((d == 0).sum()))
    r.res["desired_kl"]["final_lr"] = float(r.engines["desired_kl"].get_lr_state()[0])
    assert float(r.grads["target_kl"][r.so + 13]) == 0.0, "the KL stop stopped: raise its target"


# ---------------------------------------------------------------------------------------------- whole iterations
def iterations(opt, args):
    dev = torch.device("cuda", 0)
    T = args.states
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, -(-T // B))
    states, actions = states[:T], actions[:T]
    n_cap, e_cap = infer_caps(states)
    rng = np.random.default_rng(bench.SEED)
    rewards = (rng.standard_normal(T) * 4.0 + 2.0).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 50, replace=False)] = 0.0
    exps = np.ones(T, np.float32)
    r = SimpleNamespace(dev=dev, T=T, n_cap=n_cap, e_cap=e_cap, launches=args.launches,
                        blob=pack_and_upload(states, n_cap, e_cap, dev),
                        act=torch.as_tensor(np.ascontiguousarray(actions, np.float32), device=dev))
    models = {}
    for model in opt["models"]:
        flat = initial(model)
        ups = {c: PPOUpdater(flat, n_cap, e_cap, dev, opt_num_epochs=4, mini_batch_size=B,
                             clip_mode=_lib.CLIP_REFERENCE, process_group=None, model=model, **opt["updater"], **kw)
               for c, kw in opt["configs"].items()}
        for up in ups.values():                # warm-up: module loads, buffers, the packer
            np.random.seed(0)
            up.update_params(states, actions, rewards, masks, exps)
        res, last = {c: {"s_per_iteration": []} for c in ups}, {}
        for rep in range(args.repeats):
            for c, up in ups.items():
                n0 = up.engine.launches
                np.random.seed(1 + rep)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                last[c] = up.update_params(states, actions, rewards, masks, exps)
                torch.cuda.synchronize()
                res[c]["s_per_iteration"].append(time.perf_counter() - t0)
                res[c]["gpu_launches_per_iteration"] = up.engine.launches - n0
        for s in res.values():
            s.update(median_s=float(np.median(s["s_per_iteration"])),
                     spread_s=float(max(s["s_per_iteration"]) - min(s["s_per_iteration"])))
        r.model, r.ups, r.res, r.last = model, ups, res, last
        models[model] = dict(res, **opt["kernels"](r))
    g = opt["updater"]
    head = dict(workload=f"{T} hlg states; update_params with minibatches of {B}, 4 epochs, gamma {g['gamma']:g}, "
                         f"tau {g['tau']:g}", repeats=args.repeats, card=card())
    return report(opt, head, models)


def value_sweeps(r):
    """The value-only sweep (upb_values / upb_mlp_values) against the full forward over the same states, both models."""
    sweeps = {}
    for model in ("sgnn", "mlp"):
        eng = Engine(r.dev, r.n_cap, r.e_cap, model=model)
        params = torch.as_tensor(initial(model), device=r.dev)
        value = torch.zeros(r.T, dtype=torch.float32, device=r.dev)
        for name, fn in (("forward", lambda _: eng.forward(r.blob, params, r.act)),
                         ("values", lambda _: eng.values(r.blob, params, out=value))):
            sweeps[f"{model}_{name}_event_ms_per_call"] = event_ms(fn, 3, r.launches)
        sweeps[f"{model}_values_over_forward"] = (sweeps[f"{model}_values_event_ms_per_call"]
                                                  / sweeps[f"{model}_forward_event_ms_per_call"])
        eng.close()
    return dict(sweeps=sweeps, note="sweep times are CUDA-event times per call over back-to-back calls, the Python "
                                    "call and the forward's output allocations included")


def value_norm_kernels(r):
    """k_value_denorm and k_value_norm over T values: CUDA-event time per call, then their own device time."""
    from torch.profiler import ProfilerActivity, profile
    eng = r.ups["on"].engine
    vals = torch.randn(r.T, device=r.dev)
    ret = torch.randn(r.T, device=r.dev) * 4.0 + 2.0
    params = r.ups["on"].params.clone()
    calls = (("k_value_denorm", lambda _: eng.denormalize_values(vals)),
             ("k_value_norm", lambda _: eng.value_norm_update(ret, params, vals)))
    kernels = {name + "_event_us_per_call": event_ms(fn, 10, r.launches) * 1e3 for name, fn in calls}
    # the kernels' own device time, in a run of its own under the profiler
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, fn in calls:
            for i in range(r.launches):
                fn(i)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for name, _ in calls:
            if name + "E" in ev.key or ev.key.startswith(name) or ("::" + name + "(") in ev.key:
                dt = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                kernels[name + "_device_us"] = dt / max(ev.count, 1)
    return dict(kernels_over_T_values=kernels, note="event times per call include the Python call and the allocation "
                                                    "of its outputs; device times are the kernels' own")


def grad_noise_kernel(r):
    """The estimate of each measuring configuration's last iteration; k_grad_noise's CUDA time per call from the
    profiler over ppo_grad_noise calls on one 256-graph minibatch in a random order, and the CUDA-event time of a whole
    ppo_grad_noise call and of ppo_grad on the same ids.  That order is unbalanced (not the steps' LPT order), so its
    gradient launch may take longer than a fused step's."""
    from torch.profiler import ProfilerActivity, profile
    for c in ("k1", "k8"):
        r.res[c]["estimate"] = {k: r.last[c][k] for k in ("grad_noise_scale", "grad_noise_g2", "grad_noise_trace",
                                                          "grad_noise_samples")}
    eng = Engine(r.dev, r.n_cap, r.e_cap, model=r.model)
    params = torch.as_tensor(initial(r.model), device=r.dev)
    rng = np.random.default_rng(bench.SEED)
    adv = torch.as_tensor(rng.standard_normal(r.T).astype(np.float32), device=r.dev)
    ret = torch.as_tensor(rng.standard_normal(r.T).astype(np.float32), device=r.dev)
    exps = torch.ones(r.T, dtype=torch.float32, device=r.dev)
    _, fixed, _ = eng.forward(r.blob, params, r.act)
    ids = torch.as_tensor(rng.permutation(r.T)[:B].astype(np.int32), device=r.dev)
    a = (r.blob, params, r.act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B)
    g = eng.new_grad_buffer()
    noise = torch.zeros(4, dtype=torch.float64, device=r.dev)
    calls = {"ppo_grad_noise": lambda _: eng.ppo_grad_noise(*a, ids=ids, out=g, noise_out=noise),
             "ppo_grad": lambda _: eng.ppo_grad(*a, ids=ids, out=g)}
    out = {f"{name}_event_ms_per_call": event_ms(fn, 3, r.launches) for name, fn in calls.items()}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(r.launches):
            calls["ppo_grad_noise"](i)
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.key_averages() if "k_grad_noise" in e.key]
    out["k_grad_noise_ms_per_call"] = sum(us) / 1e3 / r.launches if us else None
    out["noise_row"] = noise.cpu().numpy().tolist()
    eng.close()
    return {"kernel": out}


# ----------------------------------------------------------------------------------------------------- the options
# Step options: `configs` gives each configuration's Engine keywords (clip_mode CLIP_NEVER unless set); `init` makes the
# SGNN's initial parameters (the rl-mlp's are PL.MLP.default_init).  `logp` is the fixed log-probs' recipe: a number s
# for a forward pass at the parameters times 1 + s N(0, 1) (generator seed 3), which also gives the old values and, with
# `cand`, the candidates' log-probs; "normal" for rng.normal(-3, 0.3) drawn after the advantages and returns.  Hooks on
# the run's namespace: `setup` after the engines, `step` in place of a plain fused step, `check` after the warm-up,
# `finish` after the windows (it may return fields for the model's result).  `rotate` rotates the engines' order from
# window to window; `clocks` reads the SM clock and throttle reasons before the warm-up and after the last window.
# Iteration options: `configs` gives PPOUpdater keywords, added to `updater`'s; `kernels` times the option's kernels.
STEP = dict(harness=step_windows, steps=48, repeats=5, init=PL.default_init)
OPTIONS = {
    "value_clip": dict(
        STEP, help="clipped value loss (upb_set_value_clip) and advantage normalisation (upb_normalize_advantages)",
        models=("sgnn",), logp=0.05, setup=value_clip_setup, step=value_clip_step,
        finish=lambda r: {"vclip_clipped_graphs_last_step": float(r.grads["vclip"][r.so + 16])},
        configs={"off": {},                                      # neither option
                 "vclip": dict(value_clip=0.2),                  # old values passed to every step
                 "both": dict(value_clip=0.2)}),                 # and one k_adv_norm launch every --pool steps
    "kl_stop": dict(
        STEP, help="KL stop (upb_set_target_kl)", steps=50, models=("sgnn",), logp=0.05, check=kl_stop_check,
        finish=kl_stop_finish, configs={"off": {},
                                        "armed": dict(target_kl=1e30),     # never fires: every step waits for the KL
                                        "skipped": dict(target_kl=1e-30)}),  # fired: every launch returns at entry
    "kl_penalty": dict(
        STEP, help="KL penalty (upb_set_kl_penalty)", models=("sgnn", "mlp"), init=PL.SGNN.default_init, logp=0.05,
        cand=True, step=lambda r, c, i: fused_step(r, c, i, old_cand_log_probs=r.cand if c == "on" else None),
        finish=lambda r: r.res["on"].update(kl_sum_last_step=float(r.grads["on"][r.so + 18])),
        configs={"off": {}, "on": dict(kl_coef=0.2)}),
    "grad_clip": dict(
        STEP, help="global gradient-norm clip (upb_set_max_grad_norm)", models=("sgnn", "mlp"), logp=0.05,
        step=grad_clip_step, finish=grad_clip_finish,
        configs={"off": {},
                 "gate": dict(max_grad_norm=1e9),                # never reached: the in-kernel wait for the norm
                 "clip": dict(max_grad_norm=1e-4),               # every step clips, fused
                 "two_call": dict(max_grad_norm=1e-4),           # the same clip on ppo_grad + apply
                 "always": dict(clip_mode=_lib.CLIP_ALWAYS)}),   # the reference's two-group clip on every step
    "nonfinite_guard": dict(
        STEP, help="non-finite guard (upb_set_nonfinite_guard); every step is finite, so this is the decision's cost",
        models=("sgnn", "mlp"), logp=0.05, finish=nonfinite_guard_finish, rotate=True, clocks=True,
        configs={"off": {}, "guard": dict(skip_nonfinite=True),  # the guard alone: the clip kernel at coefficient 1
                 "guard_clip": dict(skip_nonfinite=True, max_grad_norm=1e-4), "clip": dict(max_grad_norm=1e-4)}),
    "param_groups": dict(
        STEP, help="parameter groups (upb_set_param_groups)", models=("sgnn", "mlp"), init=PL.SGNN.default_init,
        logp="normal", setup=param_groups_setup, finish=param_groups_finish,
        configs={"off": {},                                      # no table: k_sgnn<true> / k_mlp<true>
                 "one": {},                                      # every tensor in one group: k_sgnn_pg / k_mlp_pg
                 "frozen": {}}),                                 # the same table with the shared encoder frozen
    "adam_options": dict(
        STEP, help="Adam options (upb_set_adam)", models=("sgnn", "mlp"), init=PL.SGNN.default_init, logp="normal",
        setup=adam_options_setup, finish=adam_options_finish,
        configs={"off": {},                                      # the default settings: k_sgnn<true> / k_mlp<true>
                 "table": {},                                    # the same through a table: k_sgnn_pg / k_mlp_pg
                 "adamw": {},                                    # torch.optim.AdamW's defaults
                 "amsgrad": {}}),                                # AdamW with amsgrad=True
    "loss_options": dict(
        STEP, help="dual-clip PPO (upb_set_dual_clip) and the Huber value loss (upb_set_huber_delta)",
        models=("sgnn", "mlp"), logp=0.3,
        finish=lambda r: r.res["both"].update(dual_active_graphs_last_step=float(r.grads["both"][r.so + 20]),
                                              huber_linear_graphs_last_step=float(r.grads["both"][r.so + 21])),
        configs={"off": {}, "dual": dict(dual_clip=1.5), "huber": dict(huber_delta=0.5),
                 "both": dict(dual_clip=1.5, huber_delta=0.5)}),
    "adaptive_lr": dict(
        STEP, help="KL-adaptive learning rate (upb_set_adaptive_lr)", models=("sgnn", "mlp"), logp=0.3,
        finish=adaptive_lr_finish,
        # the adaptive engine's bounds pin its lr at the engines' 4e-4: it decides on every step, and all three engines
        # train the same parameters, so only the decision's cost differs
        configs={"off": {}, "desired_kl": dict(desired_kl=0.01, lr_bounds=(4e-4, 4e-4)),
                 "target_kl": dict(target_kl=1e6)}),             # the KL stop's gate that both share, never firing
    "prox_ewma": dict(
        STEP, help="EWMA proximal policy (upb_set_prox_ewma): one proximal forward per step and the EWMA writes",
        models=("sgnn", "mlp"), logp=0.05, step=grad_clip_step,
        setup=lambda r: [r.engines[c].init_prox_params(r.params[c]) for c in ("fused", "two_call")],
        finish=lambda r: r.res["fused"].update(prox_weight_sum_last_step=float(r.grads["fused"][r.so + 23])),
        configs={"off": {}, "fused": dict(prox_ewma=0.9),
                 "two_call": dict(prox_ewma=0.9)}),              # ppo_grad + apply: the EWMA in k_apply
    "recompute_advantage": dict(
        harness=iterations, help="advantage recomputation before every epoch (recompute_advantage)", repeats=6,
        launches=20, models=("sgnn",), updater=dict(gamma=1.0, tau=0.0), kernels=value_sweeps,
        configs={"off": dict(recompute_advantage=False), "on": dict(recompute_advantage=True)}),
    "value_norm": dict(
        harness=iterations, help="value-target normalisation (upb_set_value_norm)", repeats=8, launches=200,
        models=("sgnn",), updater=dict(gamma=0.99, tau=0.95), kernels=value_norm_kernels,
        configs={"off": dict(value_norm=False), "on": dict(value_norm=True)}),
    "grad_noise": dict(
        harness=iterations, help="gradient noise scale measurement (grad_noise_every)", repeats=3, launches=50,
        models=("sgnn", "mlp"), updater=dict(gamma=1.0, tau=0.0), kernels=grad_noise_kernel,
        configs={"off": dict(grad_noise_every=None), "k1": dict(grad_noise_every=1),  # k1: every step measured
                 "k8": dict(grad_noise_every=8)}),
}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="option", required=True, metavar="OPTION")
    for name, opt in OPTIONS.items():
        p = sub.add_parser(name, help=opt["help"])
        steps = opt["harness"] is step_windows
        if steps:
            p.add_argument("--steps", type=int, default=opt["steps"])
            p.add_argument("--warmup", type=int, default=5)
            p.add_argument("--pool", type=int, default=16)
        else:
            p.add_argument("--states", type=int, default=25_000)
            p.add_argument("--launches", type=int, default=opt["launches"], help="timed calls of each kernel measured")
        p.add_argument("--repeats", type=int, default=opt["repeats"],
                       help=f"timed {'windows' if steps else 'iterations'} per configuration, alternating")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device (no CPU fallback)")
    opt = OPTIONS[args.option]
    print(json.dumps(opt["harness"](opt, args)))


if __name__ == "__main__":
    main()
