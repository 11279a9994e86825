#!/usr/bin/env python
"""Cost of the KL stop (upb_set_target_kl) on the fused SGNN step, one GPU, the bench.py workload (256 HLG graphs per
step, 16 resident minibatches, seed 111).  Three engines alternate in timed windows:

    off     the stop off (the default)
    armed   the stop on with a target that never fires: every step waits for the statistics slice before Adam
    skipped the stop on after it fired: every launch returns at entry

    python tools/kl_stop_bench.py [--steps K] [--warmup W] [--repeats R]

Prints one JSON line: per configuration the CUDA-event step time of every window, launches per step, the card's name
and power limit, and whether `off` and `armed` left bit-identical parameters.  Writes nothing.
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

CONFIGS = ("off", "armed", "skipped")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
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
    target = {"off": None, "armed": 1e30, "skipped": 1e-30}
    engines = {c: Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_NEVER, target_kl=target[c]) for c in CONFIGS}
    params = {c: torch.as_tensor(flat, device=dev).clone() for c in CONFIGS}
    grads = {c: engines[c].new_grad_buffer() for c in CONFIGS}
    pert = params["off"] * (1.0 + 0.05 * torch.randn(params["off"].shape, device=dev,
                                                     generator=torch.Generator(dev).manual_seed(3)))
    _, fixed, _ = engines["off"].forward(blob, pert, act)
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    mb_ids = [torch.as_tensor(engines["off"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32),
                              device=dev) for m in range(args.pool)]

    def step(c, i):
        engines[c].ppo_step(blob, params[c], act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B, ids=mb_ids[i % args.pool],
                            out=grads[c])

    for c in CONFIGS:
        for i in range(args.warmup):
            step(c, i)
    torch.cuda.synchronize()
    so = engines["skipped"].stat_offset
    assert float(grads["skipped"][so + 14]) == 1.0, "the tiny target stopped the first step; later ones are skipped"
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
    same = (torch.equal(params["off"], params["armed"]) and
            all(np.array_equal(a, b) for a, b in zip(engines["off"].get_opt_state(), engines["armed"].get_opt_state())))
    print(json.dumps(dict(workload=f"hlg, {B} graphs per step, {args.pool} minibatches, fused SGNN step",
                          steps=args.steps, repeats=args.repeats, card=card(), configs=res,
                          off_armed_bit_identical=bool(same))))


if __name__ == "__main__":
    main()
