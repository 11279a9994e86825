#!/usr/bin/env python
"""Cost of value-target normalisation (upb_set_value_norm) on one GPU: whole PPOUpdater.update_params iterations of
25,000 HLG states (the bench.py graphs, 512 distinct tiled; minibatches of 256, 4 epochs, 388 optimiser steps) with the
option off and on, alternating in one session, and the CUDA-event time of its two launches, k_value_denorm and
k_value_norm, over the same 25,000 values.

    python tools/value_norm_bench.py [--states T] [--repeats R] [--launches N]

Prints one JSON line with every iteration's time per configuration, launches per iteration, the two kernels' mean time
and the card's name and power limit.  Writes nothing.
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
    ap.add_argument("--repeats", type=int, default=8, help="timed iterations per configuration, alternating")
    ap.add_argument("--launches", type=int, default=200, help="timed launches of each new kernel")
    args = ap.parse_args()

    import torch
    from drl_urban_planning_b200 import _lib, params as PL
    from drl_urban_planning_b200.packing import infer_caps
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
    flat = PL.default_init(bench.SEED)
    ups = {c: PPOUpdater(flat, n_cap, e_cap, dev, gamma=0.99, tau=0.95, opt_num_epochs=4, mini_batch_size=bench.BATCH,
                         clip_mode=_lib.CLIP_REFERENCE, process_group=None, value_norm=(c == "on")) for c in CONFIGS}
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

    eng = ups["on"].engine
    vals = torch.randn(T, device=dev)
    ret = torch.randn(T, device=dev) * 4.0 + 2.0
    params = ups["on"].params.clone()
    kernels = {}
    calls = (("k_value_denorm", lambda: eng.denormalize_values(vals)),
             ("k_value_norm", lambda: eng.value_norm_update(ret, params, vals)))
    for name, fn in calls:
        for _ in range(10):
            fn()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.launches):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        kernels[name + "_event_us_per_call"] = ev0.elapsed_time(ev1) * 1e3 / args.launches
    # the kernels' own device time, in a run of its own under the profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, fn in calls:
            for _ in range(args.launches):
                fn()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for name, _ in calls:
            if name + "E" in ev.key or ev.key.startswith(name) or ("::" + name + "(") in ev.key:
                dt = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                kernels[name + "_device_us"] = dt / max(ev.count, 1)
    print(json.dumps(dict(workload=f"update_params, {T} hlg states, minibatches of {bench.BATCH}, 4 epochs",
                          repeats=args.repeats, card=card(), configs=res, kernels_over_T_values=kernels,
                          note="event times per call include the Python call and the allocation of its outputs; "
                               "device times are the kernels' own")))


if __name__ == "__main__":
    main()
