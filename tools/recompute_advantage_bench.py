#!/usr/bin/env python
"""Cost of recompute_advantage on one GPU: the CUDA-event time of the value-only sweep (upb_values / upb_mlp_values)
against the full forward (upb_forward / upb_mlp_forward) over the same 25,000 HLG states (the bench.py graphs, 512
distinct tiled), both models; then whole PPOUpdater.update_params iterations of those states (minibatches of 256, 4
epochs, 388 optimiser steps) with the option off and on, alternating in one session.

    python tools/recompute_advantage_bench.py [--states T] [--repeats R] [--launches N]

Prints one JSON line with both sweeps' mean time per call per model, every iteration's time per configuration, launches
per iteration, and the card's name and power limit.  Writes nothing.
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

CONFIGS = ("off", "on")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--states", type=int, default=25_000)
    ap.add_argument("--repeats", type=int, default=6, help="timed iterations per configuration, alternating")
    ap.add_argument("--launches", type=int, default=20, help="timed sweeps of each kind")
    args = ap.parse_args()

    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.engine import Engine
    from drl_urban_planning_b200.packing import infer_caps, pack_and_upload
    from drl_urban_planning_b200.ppo import PPOUpdater

    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    T = args.states
    states, actions = bench.make_pool(bench.SEED, "hlg", 512, -(-T // bench.BATCH))
    states, actions = states[:T], actions[:T]
    n_cap, e_cap = infer_caps(states)

    sweeps = {}
    blob = pack_and_upload(states, n_cap, e_cap, dev)
    act = torch.as_tensor(np.ascontiguousarray(actions, np.float32), device=dev)
    for model in ("sgnn", "mlp"):
        eng = Engine(dev, n_cap, e_cap, model=model)
        flat = PL.MLP.default_init(bench.SEED) if model == "mlp" else PL.default_init(bench.SEED)
        params = torch.as_tensor(flat, device=dev)
        value = torch.zeros(T, dtype=torch.float32, device=dev)
        calls = (("forward", lambda: eng.forward(blob, params, act)), ("values", lambda: eng.values(blob, params, out=value)))
        for name, fn in calls:
            for _ in range(3):
                fn()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(args.launches):
                fn()
            ev1.record()
            torch.cuda.synchronize()
            sweeps[f"{model}_{name}_event_ms_per_call"] = ev0.elapsed_time(ev1) / args.launches
        sweeps[f"{model}_values_over_forward"] = (sweeps[f"{model}_values_event_ms_per_call"]
                                                  / sweeps[f"{model}_forward_event_ms_per_call"])
        eng.close()

    rng = np.random.default_rng(bench.SEED)
    rewards = (rng.standard_normal(T) * 4.0 + 2.0).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 50, replace=False)] = 0.0
    exps = np.ones(T, np.float32)
    flat = PL.default_init(bench.SEED)
    ups = {c: PPOUpdater(flat, n_cap, e_cap, dev, gamma=1.0, tau=0.0, opt_num_epochs=4, mini_batch_size=bench.BATCH,
                         clip_mode=_lib.CLIP_REFERENCE, process_group=None, recompute_advantage=(c == "on"))
           for c in CONFIGS}
    res = {c: {"s_per_iteration": []} for c in CONFIGS}
    for c in CONFIGS:                                    # warm-up: module loads, buffers, the packer
        np.random.seed(0)
        ups[c].update_params(states, actions, rewards, masks, exps)
    for r in range(args.repeats):
        for c in CONFIGS:
            up = ups[c]
            n0 = up.engine.launches
            np.random.seed(1 + r)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            up.update_params(states, actions, rewards, masks, exps)
            torch.cuda.synchronize()
            res[c]["s_per_iteration"].append(time.perf_counter() - t0)
            res[c]["gpu_launches_per_iteration"] = up.engine.launches - n0
    for c in CONFIGS:
        s = res[c]["s_per_iteration"]
        res[c]["median_s"] = float(np.median(s))
        res[c]["spread_s"] = float(max(s) - min(s))
    print(json.dumps(dict(workload=f"{T} hlg states; update_params with minibatches of {bench.BATCH}, 4 epochs, "
                                   "gamma 1, tau 0 (the shipped configs)",
                          repeats=args.repeats, card=card(), sweeps=sweeps, configs=res,
                          note="sweep times are CUDA-event times per call over back-to-back calls, the Python call "
                               "and the forward's output allocations included")))


if __name__ == "__main__":
    main()
