#!/usr/bin/env python
"""rl-mlp optimiser-step throughput on one GPU: the fused step (upb_mlp_ppo_step, one launch) against the two-call
path (upb_mlp_ppo_grad + upb_mlp_apply, three launches), alternated in one process on the bench.py workload
(256 HLG graphs per step, 16 resident minibatches, seed 111).

    python tools/mlp_step_bench.py [--steps K] [--warmup W] [--repeats R] [--iter-states T] [--dump-outputs DIR]

Prints one JSON line: per path the step time and graph-samples/s of every repeat, launches per step and the
event-bracketed k_mlp time; the card name and power limit; optionally one whole PPOUpdater(model="mlp") iteration.
--dump-outputs writes what each path's last timed step returned to DIR/<path>/<name>.npy.  Writes nothing else.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload, clock sampler, output dump of the main bench line)

PATHS = ("two-call", "fused")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = (x.strip() for x in out.split(",")[:2])
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3, help="timed windows per path, the paths alternating")
    ap.add_argument("--pool", type=int, default=16)
    ap.add_argument("--iter-states", type=int, default=25000,
                    help="rollout states of one whole PPOUpdater(model='mlp').update_params iteration (0 = skip)")
    ap.add_argument("--dump-outputs", metavar="DIR", default="")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)

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
    flat = PL.MLP.default_init(bench.SEED)
    engines = {p: Engine(dev, blob.n_cap, blob.e_cap, model="mlp") for p in PATHS}
    params = {p: torch.as_tensor(flat, device=dev).clone() for p in PATHS}
    grads = {p: engines[p].new_grad_buffer() for p in PATHS}
    # old log-probs from perturbed weights so that importance ratios straddle the clip range
    pert = params["fused"] * (1.0 + 0.05 * torch.randn(params["fused"].shape, device=dev,
                                                        generator=torch.Generator(dev).manual_seed(3)))
    _, fixed, _ = engines["fused"].forward(blob, pert, act)
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    mb_ids = [torch.as_tensor(engines["fused"].balance_ids(np.arange(m * B, (m + 1) * B), cost).astype(np.int32),
                              device=dev) for m in range(args.pool)]

    def step(p, i):
        e, a = engines[p], (blob, params[p], act, adv, ret, fixed, exps, 1.0 / B, 1.0 / B)
        if p == "fused":
            e.ppo_step(*a, ids=mb_ids[i % args.pool], out=grads[p])
        else:
            e.ppo_grad(*a, ids=mb_ids[i % args.pool], out=grads[p])
            e.apply(params[p], grads[p])

    for p in PATHS:
        for i in range(args.warmup):
            step(p, i)
    torch.cuda.synchronize()
    clocks = bench.ClockSampler(0)
    clocks.start()
    time.sleep(0.15)
    res = {p: {"ms_per_step": [], "graph_samples_per_s": []} for p in PATHS}
    done = {p: args.warmup for p in PATHS}
    for _ in range(args.repeats):
        for p in PATHS:
            launches0 = engines[p].launches
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for i in range(args.steps):
                step(p, done[p] + i)
            ev1.record()
            torch.cuda.synchronize()
            done[p] += args.steps
            ms = ev0.elapsed_time(ev1) / args.steps
            res[p]["ms_per_step"].append(ms)
            res[p]["graph_samples_per_s"].append(B / (ms * 1e-3))
            res[p]["gpu_launches_per_step"] = (engines[p].launches - launches0) / args.steps
    clk = clocks.stop()
    for p in PATHS:
        if args.dump_outputs:
            bench.dump_outputs(os.path.join(args.dump_outputs, p), engines[p], params[p], grads[p])
        res[p]["losses_last_step"] = [float(x) for x in engines[p].read_losses(grads[p])]
        engines[p].profile(True)
        for i in range(args.steps):
            step(p, done[p] + i)
        kms, kn = engines[p].profile_read()
        engines[p].profile(False)
        res[p]["k_mlp_ms"] = kms / max(kn, 1)
        res[p]["k_mlp_covers"] = ("the whole step (gradient, reduction, Adam)" if p == "fused" else
                                  "the gradient kernel only (k_mlp_reduce and k_apply are not bracketed)")

    iteration = None
    if args.iter_states > 0:
        from drl_urban_planning_b200.ppo import PPOUpdater
        T = args.iter_states
        reps = (T + total - 1) // total
        it_states = (states * reps)[:T]
        it_actions = np.concatenate([actions] * reps)[:T]
        rng_i = np.random.default_rng(9)
        rewards = rng_i.standard_normal(T).astype(np.float32)
        masks = np.ones(T, np.float32); masks[99::100] = 0.0
        up = PPOUpdater(flat, blob.n_cap, blob.e_cap, dev, opt_num_epochs=4, mini_batch_size=B,
                        clip_mode=_lib.CLIP_REFERENCE, process_group=None, model="mlp")
        np.random.seed(1)
        secs = []
        for _ in range(2):                       # the first pass allocates the pinned / device buffers
            torch.cuda.synchronize(); t1 = time.perf_counter()
            up.update_params(it_states, it_actions, rewards, masks)
            torch.cuda.synchronize(); secs.append(time.perf_counter() - t1)
        nsteps = 4 * (T // B)
        iteration = {"states": T, "optimiser_steps": nsteps, "seconds": secs[1], "first_call_seconds": secs[0],
                     "graph_samples_per_s": nsteps * B / secs[1], "step": "PPOUpdater.minibatch_step (fused)"}

    print(json.dumps({"model": "rl-mlp", "workload": f"hlg, {B} graphs per step, {args.pool} resident minibatches, "
                                                     f"caps {blob.n_cap}/{blob.e_cap}",
                      "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "paths": res,
                      "e2e_iteration": iteration, "card": card(), "clocks": clk}), flush=True)


if __name__ == "__main__":
    main()
