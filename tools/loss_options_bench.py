#!/usr/bin/env python
"""Cost of dual-clip PPO (upb_set_dual_clip) and the Huber value loss (upb_set_huber_delta) on the fused step of both
models, one GPU, the bench.py workload (256 HLG graphs per step, 16 resident minibatches, seed 111).  Per model, four
engines alternate in timed windows:

    off     neither option (the default)
    dual    dual clip on (c = 1.5)
    huber   the Huber value loss on (delta = 0.5)
    both    both on

The fixed log-probs come from perturbed parameters, so the ratios spread; the last step's counts of graphs where each
option bound (statistics slots 20 and 21) are printed with the times.

    python tools/loss_options_bench.py [--steps K] [--warmup W] [--repeats R]

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

CONFIGS = {"off": {}, "dual": dict(dual_clip=1.5), "huber": dict(huber_delta=0.5),
           "both": dict(dual_clip=1.5, huber_delta=0.5)}


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
    so = engines["both"].stat_offset
    res["both"]["dual_active_graphs_last_step"] = float(grads["both"][so + 20])
    res["both"]["huber_linear_graphs_last_step"] = float(grads["both"][so + 21])
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
