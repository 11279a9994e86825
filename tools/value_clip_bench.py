#!/usr/bin/env python
"""Cost of the clipped value loss (upb_set_value_clip) and the per-minibatch advantage normalisation
(upb_normalize_advantages) on the fused SGNN step, one GPU, the bench.py workload (256 HLG graphs per step, 16 resident
minibatches, seed 111).  Three engines alternate in timed windows:

    off     neither option (the default)
    vclip   value clipping on (c = 0.2), old values passed to every step
    both    value clipping on, and one k_adv_norm launch over the 16 minibatches every 16 steps (one epoch)

    python tools/value_clip_bench.py [--steps K] [--warmup W] [--repeats R]

Prints one JSON line: per configuration the CUDA-event step time of every window, launches per step and the card's name
and power limit.  Writes nothing.
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

CONFIGS = ("off", "vclip", "both")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5, help="timed windows per configuration, alternating")
    ap.add_argument("--pool", type=int, default=16)
    args = ap.parse_args()

    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.engine import Engine
    from drl_urban_planning_b200.packing import pack_states

    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    B = bench.BATCH
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, args.pool)
    blob = pack_states(states).to(dev)
    total = len(states)
    rng = np.random.default_rng(bench.SEED)
    adv = torch.as_tensor(rng.standard_normal(total).astype(np.float32), device=dev)
    ret = torch.as_tensor(rng.standard_normal(total).astype(np.float32), device=dev)
    exps = torch.ones(total, dtype=torch.float32, device=dev)
    act = torch.as_tensor(actions, device=dev)
    flat = PL.default_init(bench.SEED)
    clip = {"off": None, "vclip": 0.2, "both": 0.2}
    engines = {c: Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_NEVER, value_clip=clip[c]) for c in CONFIGS}
    params = {c: torch.as_tensor(flat, device=dev).clone() for c in CONFIGS}
    grads = {c: engines[c].new_grad_buffer() for c in CONFIGS}
    pert = params["off"] * (1.0 + 0.05 * torch.randn(params["off"].shape, device=dev,
                                                     generator=torch.Generator(dev).manual_seed(3)))
    old_values, fixed, _ = engines["off"].forward(blob, pert, act)
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    mb = [engines["off"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32) for m in range(args.pool)]
    mb_ids = [torch.as_tensor(x, device=dev) for x in mb]
    order = torch.as_tensor(np.concatenate(mb), device=dev)
    norm_adv = adv.clone()

    def step(c, i):
        a = adv
        if c == "both":
            if i % args.pool == 0:           # the top of an epoch
                engines[c].normalize_advantages(adv, exps, order, B, out=norm_adv)
            a = norm_adv
        engines[c].ppo_step(blob, params[c], act, a, ret, fixed, exps, 1.0 / B, 1.0 / B, ids=mb_ids[i % args.pool],
                            out=grads[c], old_values=None if c == "off" else old_values)

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
    so = engines["vclip"].stat_offset
    print(json.dumps(dict(workload=f"hlg, {B} graphs per step, {args.pool} minibatches, fused SGNN step",
                          steps=args.steps, repeats=args.repeats, card=card(), configs=res,
                          vclip_clipped_graphs_last_step=float(grads["vclip"][so + 16]))))


if __name__ == "__main__":
    main()
