#!/usr/bin/env python
"""Cost of the gradient-noise measurement (grad_noise_every) on one GPU, both models, on bench.py's iteration workload:
whole PPOUpdater.update_params iterations over 25,000 HLG states (the bench.py graphs, 512 distinct tiled), 4 epochs,
minibatches of 256, three ways that alternate:

    off  the default
    k1   grad_noise_every=1: every minibatch step measured (three more launches per step)
    k8   grad_noise_every=8

and k_grad_noise alone, the kernel's CUDA time per call from torch.profiler over back-to-back Engine.ppo_grad_noise
calls on one 256-graph minibatch in a random order, next to the CUDA-event time of a whole ppo_grad_noise call and of
ppo_grad on the same ids.  The measurement's launch is unbalanced (random order, not the LPT order of the steps), so its
gradient launch may take longer than a fused step's.

    python tools/grad_noise_bench.py [--states T] [--repeats R] [--launches N]

Prints one JSON line with the card's name and power limit; writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload)
from mlp_step_bench import card  # noqa: E402

CONFIGS = {"off": None, "k1": 1, "k8": 8}


def kernel_times(model, blob, actions, n_cap, e_cap, launches):
    """(k_grad_noise CUDA ms per call from the profiler, event ms per ppo_grad_noise call, event ms per ppo_grad call)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from drl_urban_planning_b200 import params as PL
    from drl_urban_planning_b200.engine import Engine

    dev = torch.device("cuda", 0)
    B = bench.BATCH
    eng = Engine(dev, n_cap, e_cap, model=model)
    flat = PL.MLP.default_init(bench.SEED) if model == "mlp" else PL.default_init(bench.SEED)
    params = torch.as_tensor(flat, device=dev)
    rng = np.random.default_rng(bench.SEED)
    T = blob.count
    adv = torch.as_tensor(rng.standard_normal(T).astype(np.float32), device=dev)
    ret = torch.as_tensor(rng.standard_normal(T).astype(np.float32), device=dev)
    exps = torch.ones(T, dtype=torch.float32, device=dev)
    act = torch.as_tensor(np.ascontiguousarray(actions, np.float32), device=dev)
    _, fixed, _ = eng.forward(blob, params, act)
    ids = torch.as_tensor(rng.permutation(T)[:B].astype(np.int32), device=dev)
    args = (blob, params, act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B)
    g = eng.new_grad_buffer()
    noise = torch.zeros(4, dtype=torch.float64, device=dev)
    calls = {"ppo_grad_noise": lambda: eng.ppo_grad_noise(*args, ids=ids, out=g, noise_out=noise),
             "ppo_grad": lambda: eng.ppo_grad(*args, ids=ids, out=g)}
    out = {}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(launches):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        out[f"{name}_event_ms_per_call"] = ev0.elapsed_time(ev1) / launches
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            calls["ppo_grad_noise"]()
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.key_averages() if "k_grad_noise" in e.key]
    out["k_grad_noise_ms_per_call"] = sum(us) / 1e3 / launches if us else None
    out["noise_row"] = noise.cpu().numpy().tolist()
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--states", type=int, default=25_000)
    ap.add_argument("--repeats", type=int, default=3, help="timed iterations per configuration, alternating")
    ap.add_argument("--launches", type=int, default=50, help="timed calls of each kind for the kernel times")
    args = ap.parse_args()

    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.packing import infer_caps, pack_and_upload
    from drl_urban_planning_b200.ppo import PPOUpdater

    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    T = args.states
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, -(-T // bench.BATCH))
    states, actions = states[:T], actions[:T]
    n_cap, e_cap = infer_caps(states)
    rng = np.random.default_rng(bench.SEED)
    rewards = (rng.standard_normal(T) * 4.0 + 2.0).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 50, replace=False)] = 0.0
    exps = np.ones(T, np.float32)
    blob = pack_and_upload(states, n_cap, e_cap, dev)

    models = {}
    for model in ("sgnn", "mlp"):
        res = {"kernel": kernel_times(model, blob, actions, n_cap, e_cap, args.launches)}
        flat = PL.MLP.default_init(bench.SEED) if model == "mlp" else PL.default_init(bench.SEED)
        ups = {c: PPOUpdater(flat, n_cap, e_cap, dev, gamma=1.0, tau=0.0, opt_num_epochs=4, mini_batch_size=bench.BATCH,
                             clip_mode=_lib.CLIP_REFERENCE, process_group=None, model=model, grad_noise_every=k)
               for c, k in CONFIGS.items()}
        for c in CONFIGS:                                # warm-up: module loads, buffers, the packer
            np.random.seed(0)
            ups[c].update_params(states, actions, rewards, masks, exps)
        for c in CONFIGS:
            res[c] = {"s_per_iteration": []}
        for r in range(args.repeats):
            for c in CONFIGS:
                up = ups[c]
                n0 = up.engine.launches
                np.random.seed(1 + r)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = up.update_params(states, actions, rewards, masks, exps)
                torch.cuda.synchronize()
                res[c]["s_per_iteration"].append(time.perf_counter() - t0)
                res[c]["gpu_launches_per_iteration"] = up.engine.launches - n0
                if CONFIGS[c] is not None:
                    res[c]["estimate"] = {k: out[k] for k in ("grad_noise_scale", "grad_noise_g2", "grad_noise_trace",
                                                              "grad_noise_samples")}
        for c in CONFIGS:
            s = res[c]["s_per_iteration"]
            res[c]["median_s"] = float(np.median(s))
            res[c]["spread_s"] = float(max(s) - min(s))
        models[model] = res
    print(json.dumps(dict(workload=f"{T} hlg states; update_params with minibatches of {bench.BATCH}, 4 epochs, "
                                   "gamma 1, tau 0",
                          repeats=args.repeats, card=card(), models=models)))


if __name__ == "__main__":
    main()
