#!/usr/bin/env python
"""Cost of the non-finite guard (upb_set_nonfinite_guard) on the fused step of both models, one GPU, the bench.py
workload (256 HLG graphs per step, 16 resident minibatches, seed 111).  Every step is finite, so this is the cost of
the decision, not of a skip.  Per model, four engines alternate in timed windows:

    off         CLIP_NEVER, no clip, no guard (the default)
    guard       the guard alone: the clipping kernel with coefficient 1, every CTA waits for the norm
    guard_clip  the guard and max_grad_norm below every step's norm
    clip        that max_grad_norm alone

    python tools/nonfinite_guard_bench.py [--steps K] [--warmup W] [--repeats R]

The order of the engines rotates from window to window, so that no configuration always follows the same one.  The
card's SM clock and throttle reasons are read (read only) before the warm-up and right after the last timed window.

Prints one JSON line: per model and configuration the CUDA-event step time of every window, the median and spread,
launches per step, and the card's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload)
from mlp_step_bench import card  # noqa: E402

CONFIGS = ("off", "guard", "guard_clip", "clip")


def clocks():
    """The SM clock and the active throttle reasons as nvidia-smi reports them now; nothing is set."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20).stdout
        sm, sm_max, reasons = (x.strip() for x in out.strip().split(",")[:3])
        return {"sm_clock": sm, "sm_clock_max": sm_max, "throttle_reasons_active": reasons}
    except Exception:
        return {"sm_clock": None, "sm_clock_max": None, "throttle_reasons_active": None}


def run_model(model, args, blob, act, adv, ret, exps, dev):
    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.engine import Engine

    B = bench.BATCH
    kw = {"off": {}, "guard": dict(skip_nonfinite=True), "guard_clip": dict(skip_nonfinite=True, max_grad_norm=1e-4),
          "clip": dict(max_grad_norm=1e-4)}
    engines = {c: Engine(dev, blob.n_cap, blob.e_cap, model=model, clip_mode=_lib.CLIP_NEVER, **kw[c]) for c in CONFIGS}
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
        engines[c].ppo_step(blob, params[c], act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B, ids=mb_ids[i % args.pool],
                            out=grads[c])

    for c in CONFIGS:
        for i in range(args.warmup):
            step(c, i)
    torch.cuda.synchronize()
    res = {c: {"ms_per_step": []} for c in CONFIGS}
    done = {c: args.warmup for c in CONFIGS}
    for w in range(args.repeats):
        for c in CONFIGS[w % len(CONFIGS):] + CONFIGS[:w % len(CONFIGS)]:
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
    torch.cuda.synchronize()
    for c in CONFIGS:
        ms = res[c]["ms_per_step"]
        res[c]["median_ms"] = float(np.median(ms))
        res[c]["spread_ms"] = float(max(ms) - min(ms))
        res[c]["last_norm_slot17"] = float(grads[c][so + 17])
        res[c]["last_skipped_slot19"] = float(grads[c][so + 19])
        res[c]["params_finite"] = bool(torch.isfinite(params[c]).all())
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
    before = clocks()
    out = {m: run_model(m, args, blob, act, adv, ret, exps, dev) for m in ("sgnn", "mlp")}
    after = clocks()
    print(json.dumps(dict(workload=f"hlg, {bench.BATCH} graphs per step, {args.pool} minibatches, fused step",
                          steps=args.steps, repeats=args.repeats, card=dict(card(), before=before, after_last_window=after), models=out)))


if __name__ == "__main__":
    main()
