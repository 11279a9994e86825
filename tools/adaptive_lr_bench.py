#!/usr/bin/env python
"""Cost of the KL-adaptive lr (upb_set_adaptive_lr) on the fused step of both models, one GPU, the bench.py workload (256
HLG graphs per step, 16 resident minibatches, seed 111).  Per model, three engines alternate in timed windows:

    off         neither option (the default)
    desired_kl  the adaptive lr on (desired_kl = 0.01, both bounds at the engines' lr 4e-4)
    target_kl   the KL stop on at a target no step reaches (the existing cost of the statistics-slice gate both share)

The fixed log-probs come from perturbed parameters, so the ratios spread; the adaptive engine's decisions over the
timed steps (statistics slot 22) and its final lr are printed with the times.

    python tools/adaptive_lr_bench.py [--steps K] [--warmup W] [--repeats R]

Prints one JSON line: per model and configuration the CUDA-event step time of every window, launches per step and the
card's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload)
from mlp_step_bench import card  # noqa: E402

# the adaptive engine's bounds pin its lr at the engines' 4e-4: it decides on every step, and all three engines train the
# same parameters, so only the decision's cost differs
CONFIGS = {"off": {}, "desired_kl": dict(desired_kl=0.01, lr_bounds=(4e-4, 4e-4)), "target_kl": dict(target_kl=1e6)}


def run(model, args, blob, states, actions):
    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.engine import Engine

    dev = torch.device("cuda", 0)
    B = bench.BATCH
    total = len(states)
    rng = np.random.default_rng(bench.SEED)
    adv = torch.as_tensor(rng.standard_normal(total).astype(np.float32), device=dev)
    ret = torch.as_tensor(rng.standard_normal(total).astype(np.float32), device=dev)
    exps = torch.ones(total, dtype=torch.float32, device=dev)
    act = torch.as_tensor(actions, device=dev)
    flat = PL.MLP.default_init(bench.SEED) if model == "mlp" else PL.default_init(bench.SEED)
    engines = {c: Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_NEVER, model=model, **kw)
               for c, kw in CONFIGS.items()}
    params = {c: torch.as_tensor(flat, device=dev).clone() for c in CONFIGS}
    grads = {c: engines[c].new_grad_buffer() for c in CONFIGS}
    pert = params["off"] * (1.0 + 0.3 * torch.randn(params["off"].shape, device=dev,
                                                    generator=torch.Generator(dev).manual_seed(3)))
    _, fixed, _ = engines["off"].forward(blob, pert, act)
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    mb = [engines["off"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32) for m in range(args.pool)]
    mb_ids = [torch.as_tensor(x, device=dev) for x in mb]

    def step(c, i):
        engines[c].ppo_step(blob, params[c], act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B, ids=mb_ids[i % args.pool],
                            out=grads[c])

    for c in CONFIGS:
        for i in range(args.warmup):
            step(c, i)
    torch.cuda.synchronize()
    res = {c: {"ms_per_step": []} for c in CONFIGS}
    done = {c: args.warmup for c in CONFIGS}
    so = engines["off"].stat_offset
    decisions = []
    for _ in range(args.repeats):
        for c in CONFIGS:
            launches0 = engines[c].launches
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for i in range(args.steps):
                step(c, done[c] + i)
            ev1.record()
            torch.cuda.synchronize()
            done[c] += args.steps
            res[c]["ms_per_step"].append(ev0.elapsed_time(ev1) / args.steps)
            res[c]["gpu_launches_per_step"] = (engines[c].launches - launches0) / args.steps
    for c in CONFIGS:
        ms = res[c]["ms_per_step"]
        res[c]["median_ms"] = float(np.median(ms))
        res[c]["spread_ms"] = float(max(ms) - min(ms))
    for i in range(args.steps):                   # untimed: the decisions of as many more steps
        step("desired_kl", done["desired_kl"] + i)
        decisions.append(grads["desired_kl"][so + 22].clone())
    d = torch.stack(decisions).cpu().numpy()
    res["desired_kl"]["decisions"] = dict(up=int((d > 0).sum()), down=int((d < 0).sum()), none=int((d == 0).sum()))
    res["desired_kl"]["final_lr"] = float(engines["desired_kl"].get_lr_state()[0])
    assert float(grads["target_kl"][so + 13]) == 0.0, "the KL stop stopped: raise its target"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5, help="timed windows per configuration, alternating")
    ap.add_argument("--pool", type=int, default=16)
    args = ap.parse_args()

    import torch
    from drl_urban_planning_b200.packing import pack_states

    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, args.pool)
    blob = pack_states(states).to(torch.device("cuda", 0))
    out = {m: run(m, args, blob, states, actions) for m in ("sgnn", "mlp")}
    print(json.dumps(dict(workload=f"hlg, {bench.BATCH} graphs per step, {args.pool} minibatches, fused step",
                          steps=args.steps, repeats=args.repeats, card=card(), models=out)))


if __name__ == "__main__":
    main()
