#!/usr/bin/env python
"""Cost of the global gradient-norm clip (upb_set_max_grad_norm) on the fused step of both models, one GPU, the bench.py
workload (256 HLG graphs per step, 16 resident minibatches, seed 111).  Per model, five engines alternate in timed
windows:

    off       CLIP_NEVER, no clip (the default of the option)
    gate      max_grad_norm above every step's norm: the in-kernel wait for the norm, no scaling
    clip      max_grad_norm below every step's norm: every step clips, fused (one launch)
    two_call  the same clip on the two-call path (ppo_grad + apply), which the fused clip must beat
    always    CLIP_ALWAYS, the reference's two-group clip on every step (the three-launch path)

    python tools/grad_clip_bench.py [--steps K] [--warmup W] [--repeats R]

Prints one JSON line: per model and configuration the CUDA-event step time of every window, the median and spread,
launches per step, and the card's name and power limit.  Writes nothing.
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

CONFIGS = ("off", "gate", "clip", "two_call", "always")


def run_model(model, args, blob, act, adv, ret, exps, dev):
    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.engine import Engine

    B = bench.BATCH
    kw = {"off": dict(clip_mode=_lib.CLIP_NEVER), "gate": dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=1e9),
          "clip": dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=1e-4),
          "two_call": dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=1e-4), "always": dict(clip_mode=_lib.CLIP_ALWAYS)}
    engines = {c: Engine(dev, blob.n_cap, blob.e_cap, model=model, **kw[c]) for c in CONFIGS}
    flat = (PL.MLP.default_init if model == "mlp" else PL.default_init)(bench.SEED)
    params = {c: torch.as_tensor(flat, device=dev).clone() for c in CONFIGS}
    grads = {c: engines[c].new_grad_buffer() for c in CONFIGS}
    pert = params["off"] * (1.0 + 0.05 * torch.randn(params["off"].shape, device=dev,
                                                     generator=torch.Generator(dev).manual_seed(3)))
    _, fixed, _ = engines["off"].forward(blob, pert, act)
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    mb_ids = [torch.as_tensor(engines["off"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32),
                              device=dev) for m in range(args.pool)]

    def step(c, i):
        e, a = engines[c], (blob, params[c], act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B)
        if c == "two_call":
            e.ppo_grad(*a, ids=mb_ids[i % args.pool], out=grads[c])
            e.apply(params[c], grads[c])
        else:
            e.ppo_step(*a, ids=mb_ids[i % args.pool], out=grads[c])

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
    so = engines["clip"].stat_offset
    for c in CONFIGS:
        ms = res[c]["ms_per_step"]
        res[c]["median_ms"] = float(np.median(ms))
        res[c]["spread_ms"] = float(max(ms) - min(ms))
        res[c]["last_norm_slot17"] = float(grads[c][so + 17])
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
    dev = torch.device("cuda", 0)
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, args.pool)
    blob = pack_states(states).to(dev)
    total = len(states)
    rng = np.random.default_rng(bench.SEED)
    adv = torch.as_tensor(rng.standard_normal(total).astype(np.float32), device=dev)
    ret = torch.as_tensor(rng.standard_normal(total).astype(np.float32), device=dev)
    exps = torch.ones(total, dtype=torch.float32, device=dev)
    act = torch.as_tensor(actions, device=dev)
    out = {m: run_model(m, args, blob, act, adv, ret, exps, dev) for m in ("sgnn", "mlp")}
    print(json.dumps(dict(workload=f"hlg, {bench.BATCH} graphs per step, {args.pool} minibatches, fused step",
                          steps=args.steps, repeats=args.repeats, card=card(), models=out)))


if __name__ == "__main__":
    main()
