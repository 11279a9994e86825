#!/usr/bin/env python
"""Cost of the Adam options (upb_set_adam) on the fused step of both models, one GPU, the bench.py workload (256 HLG
graphs per step, 16 resident minibatches, seed 111).  For each model four engines alternate in timed windows:

    off       the default settings: k_sgnn<true> / k_mlp<true>
    table     the default settings through a table (every tensor in one group): k_sgnn_pg / k_mlp_pg
    adamw     torch.optim.AdamW's defaults (weight_decay 0.01, eps 1e-8, decoupled): k_sgnn_pg / k_mlp_pg
    amsgrad   AdamW with amsgrad=True

    python tools/adam_options_bench.py [--steps K] [--warmup W] [--repeats R]

Prints one JSON line: per model and configuration the CUDA-event step time of every window, their median and spread,
launches per step and the card's name and power limit.  Writes nothing.
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

CONFIGS = ("off", "table", "adamw", "amsgrad")


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
    fixed = torch.as_tensor(rng.normal(-3.0, 0.3, total).astype(np.float32), device=dev)
    exps = torch.ones(total, dtype=torch.float32, device=dev)
    act = torch.as_tensor(actions, device=dev)
    out = dict(workload=f"hlg, {B} graphs per step, {args.pool} minibatches, fused step", steps=args.steps,
               repeats=args.repeats, card=card(), models={})
    for model in ("sgnn", "mlp"):
        lay = PL.MLP if model == "mlp" else PL.SGNN
        flat = lay.default_init(bench.SEED)
        engines = {c: Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_NEVER, model=model) for c in CONFIGS}
        n = len(lay.slots)
        # the context's lr is upb_create's (double)(float)lr: the table takes the same value
        engines["table"].set_param_groups([float(np.float32(engines["table"].lr))] * n, [0.0] * n, [True] * n)
        for c in ("adamw", "amsgrad"):
            engines[c].set_weight_decay(0.01)
            engines[c].set_adam((0.9, 0.999), 1e-8, amsgrad=c == "amsgrad", decoupled_weight_decay=True)
        params = {c: torch.as_tensor(flat, device=dev).clone() for c in CONFIGS}
        grads = {c: engines[c].new_grad_buffer() for c in CONFIGS}
        cost = Engine.graph_cost(blob.info.astype(np.int64))
        mb_ids = [torch.as_tensor(engines["off"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32),
                                  device=dev) for m in range(args.pool)]

        def step(c, i):
            engines[c].ppo_step(blob, params[c], act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B,
                                ids=mb_ids[i % args.pool], out=grads[c])

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
        # the table at the default settings is the default step, bit for bit (SGNN only: the rl-mlp land-use backward
        # sums a node's candidates with shared-memory atomics, so its rows on these graphs differ run to run)
        if model == "sgnn":
            res["table"]["params_equal_off"] = bool(torch.equal(params["table"], params["off"]))
        out["models"][model] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
