"""Builders and float64 oracles of tests/test_gpu_update_scale.py: one `update_params` iteration at the product's size
(25,000 HLG-shaped states, minibatches of 256, 4 epochs, 388 optimiser steps), an instrumented updater that records
every step, and the teacher-forced minibatch oracles a sampled step is checked against.

Teacher forcing: a 388-step fp32 trajectory cannot be compared with a float64 one (Adam runs drift apart with no useful
bound), but each single step can.  The oracle starts from the kernel's own parameters, moments and counters just before
the step and from the kernel's own advantages, returns and pre-pass results, so its error does not accumulate."""
import multiprocessing as mp
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

import klpen_oracle as KO
import ppo_oracle as PPO
from drl_urban_planning_b200 import params as PL, synth
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from shape_cases import BOUNDARY, boundary_batch, is_big

T_PRODUCT, B, EPOCHS = 25_000, 256, 4
POOL = 2048                      # distinct synth HLG states a rollout is tiled from
BOUNDARY_COPIES = 4              # positions per shape_cases boundary graph in a rollout
GAMMA, TAU = 0.99, 0.95


# ---- the rollout -----------------------------------------------------------------------------------------------------
def _pool_chunk(seed):
    states, _ = synth.make_states(seed, "hlg", 128, stages=[int(i % 4 == 3) for i in range(128)])
    return states


def workers():
    return max(1, min(32, len(os.sched_getaffinity(0))))


def _pool(fn, jobs):
    """fn over jobs in forked worker processes (numpy only: a child never touches CUDA or torch)."""
    if workers() == 1:
        return [fn(j) for j in jobs]
    with ProcessPoolExecutor(workers(), mp_context=mp.get_context("fork")) as ex:
        return list(ex.map(fn, jobs))


def make_pool(seed=11):
    """POOL distinct HLG states (caps 1000 / 3000; one in four a road state), then one state per shape_cases boundary
    row: graphs above 464 nodes and above 160 candidates up to the caps, so minibatches take the large-graph path."""
    pool = [s for chunk in _pool(_pool_chunk, [seed * 1000 + c for c in range(POOL // 128)]) for s in chunk]
    bstates, _, labels = boundary_batch(seed)
    return pool + bstates, labels


def candidates(state):
    stage = int(np.argmax(state[8][:2]))
    return stage, np.flatnonzero(state[6] if stage == 0 else state[7])


class Rollout:
    """T samples drawn from a state pool: the pool tiled in a seeded shuffle, each boundary graph at BOUNDARY_COPIES
    known positions, an action of its own for every sample (a repeated state is an independent sample), rewards
    N(0, 1), about 3 % of exps 0, and episodes of mixed lengths (length 1, longer than a minibatch) whose last one is
    left open (masks[T - 1] = 1)."""

    def __init__(self, pool, T, seed):
        rng = np.random.default_rng(seed)
        n_plain = len(pool) - len(BOUNDARY)
        src = rng.permutation(np.resize(np.arange(n_plain), T))
        self.boundary_pos = rng.choice(T, size=(len(BOUNDARY), BOUNDARY_COPIES), replace=False)
        for b, pos in enumerate(self.boundary_pos):
            src[pos] = n_plain + b
        self.T, self.src = T, src
        self.states = [pool[i] for i in src]
        self.actions = np.zeros((T, 2), np.float32)
        for i, p in enumerate(src):
            stage, cand = candidates(pool[p])
            self.actions[i, stage] = cand[rng.integers(cand.size)]
        self.rewards = rng.standard_normal(T).astype(np.float32)
        self.exps = np.where(rng.random(T) < 0.03, 0.0, 1.0).astype(np.float32)
        lengths = []
        while sum(lengths) < T:
            u = rng.random()
            lengths.append(1 if u < 0.15 else int(rng.integers(257, 700)) if u < 0.3 else int(rng.integers(2, 200)))
        ends = np.cumsum(lengths) - 1
        self.masks = np.ones(T, np.float32)
        self.masks[ends[ends < T - 1]] = 0.0                      # the last episode stays open
        self.lengths = np.diff(np.r_[-1, np.flatnonzero(self.masks == 0), T - 1])
        big = np.array([is_big(n, e, k) for _, n, e, k, *_ in BOUNDARY])
        self.big_pos = self.boundary_pos[big].ravel()


def epoch_orders(seed, T, epochs=EPOCHS):
    """PPOUpdater._epoch_order's np.random replay: epoch k walks perm_1 o ... o perm_k."""
    np.random.seed(seed)
    order, out = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        out.append(order)
    return out


# ---- instrumenting the update ----------------------------------------------------------------------------------------
class Recorder:
    """Wraps minibatch_step on one updater instance (update_policy calls it through self): every step's ids (host
    copy), arguments and ring row, a device copy of the row it wrote, and for the steps in `sample` the parameters
    and engine.get_opt_state() before and after it; with normalize_advantage the normalised advantages at each epoch's
    first step."""

    def __init__(self, up, sample, nb):
        self.up, self.sample, self.nb = up, set(sample), nb
        self.inner = up.minibatch_step
        up.minibatch_step = self.step
        self.ids, self.args, self.rows, self.bufs = [], [], [], []
        self.before, self.after, self.norm_adv = {}, {}, {}

    def _state(self):
        torch.cuda.synchronize()
        m, v, steps = self.up.engine.get_opt_state()
        return self.up.params.cpu().numpy().copy(), m, v, steps

    def step(self, ids, global_batch, global_ind):
        k = len(self.ids)
        ring = self.up._grad_ring
        self.rows.append((self.up.grad.data_ptr() - ring.data_ptr()) // (ring.stride(0) * ring.element_size()))
        self.ids.append(ids.cpu().numpy().copy())
        self.args.append((global_batch, global_ind))
        if self.up.normalize_advantage and k % self.nb == 0:
            self.norm_adv[k // self.nb] = self.up.norm_advantages.cpu().numpy().copy()
        if k in self.sample:
            self.before[k] = self._state()
        self.inner(ids, global_batch, global_ind)
        self.bufs.append(self.up.grad.clone())
        if k in self.sample:
            self.after[k] = self._state()


def sample_steps(orders, big_pos, nb, seed, extra=8):
    """Step 0 (the two-call path with the first-step clip), step 1 (the first fused step), the first and last step of
    every epoch, the first step whose minibatch holds a boundary graph on the large-graph path (from the replayed
    epoch orders, so the sample is known before the run), and `extra` seeded others."""
    total = nb * len(orders)
    s = {0, 1} | {e * nb for e in range(len(orders))} | {e * nb + nb - 1 for e in range(len(orders))}
    big = np.zeros(orders[0].size, bool)
    big[big_pos] = True
    s.add(next(k for k in range(total) if big[orders[k // nb][(k % nb) * B:(k % nb + 1) * B]].any()))
    s.update(int(k) for k in np.random.default_rng(seed).choice(sorted(set(range(total)) - s), extra, replace=False))
    return sorted(s)


# ---- step counters and the per-entry Adam step counts ----------------------------------------------------------------
def segment_ranges(layout):
    return {"lu": slice(layout.slots["lu_w0"].offset, layout.slots["road_w0"].offset),
            "road": slice(layout.slots["road_w0"].offset, layout.policy_end)}


def entry_steps(steps, layout):
    """Per-parameter Adam step count from the four counters {global, encoder + value, land-use head, road head}."""
    t = np.full(layout.num_params, float(steps[1]))
    r = segment_ranges(layout)
    t[r["lu"]], t[r["road"]] = float(steps[2]), float(steps[3])
    return t


def live_entries(stages, layout):
    live = np.ones(layout.num_params, bool)
    r = segment_ranges(layout)
    if not (stages == 0).any():
        live[r["lu"]] = False
    if not (stages == 1).any():
        live[r["road"]] = False
    return live


def clip_groups(grad, layout):
    """The reference's first-step clip (policy group, then value group; clip_grad_norm_ at 1.0) on `layout`."""
    if layout is PL.SGNN:
        return ON.clip_groups(grad)
    g = np.array(grad, np.float64)
    for owners in (("enc", "pol"), ("enc", "val")):
        sel = np.concatenate([np.arange(s.offset, s.offset + s.size) for s in layout.slots.values() if s.owner in owners])
        g[sel] *= min(1.0, 1.0 / (np.sqrt((g[sel] ** 2).sum()) + 1e-6))
    return g


# ---- float64 oracles, run in forked workers ---------------------------------------------------------------------------
# set by the parent before it forks; the workers only read them
JOB = {}


def _prepass_one(p):
    fw = ON.forward(JOB["P"], ON.unpad(JOB["pool"][p]), keep=True)
    c = fw["cache"]
    return fw["value"], (c["idx"], c["logp"]) if "idx" in c else (np.zeros(0, np.int64), np.zeros(0))


def sgnn_prepass(pool, flat):
    """float64 value and candidate log-probs of every pool state."""
    JOB.update(pool=pool, P=ON._p64(np.asarray(flat, np.float64)))
    return _pool(_prepass_one, range(len(pool)))


def prepass_of_samples(per_pool, pool, src, actions):
    """Per-sample float64 value and log-prob of its action from the per-pool-state results."""
    T = len(src)
    values, logp = np.zeros(T), np.zeros(T)
    for i, p in enumerate(src):
        v, (idx, lp) = per_pool[p]
        values[i] = v
        stage, _ = candidates(pool[p])
        logp[i] = lp[np.flatnonzero(idx == int(actions[i, stage]))[0]]
    return values, logp


def _sgnn_step(job):
    """One minibatch in float64 at the shipped loss settings: ON.ppo_minibatch on the kernel's own inputs."""
    flat, ids = job
    J = JOB
    return ON.ppo_minibatch(flat, [J["states"][i] for i in ids], J["actions"][ids], J["adv"][ids], J["ret"][ids],
                            J["fixed"][ids], J["exps"][ids])


def _options_step(job):
    """ppo_oracle.sgnn_minibatch on one sampled step with the options in JOB["opts"]: (parameters, ids, the kernel's
    normalised advantages) from the job, the rest from JOB."""
    flat, ids, adv = job
    J = JOB
    return PPO.sgnn_minibatch(flat, [J["states"][i] for i in ids], J["actions"][ids], adv[ids], J["ret"][ids],
                              J["fixed"][ids], J["exps"][ids], old_values=J["old_values"][ids],
                              lp_old=[J["lp_old"][i] for i in ids], **J["opts"])


def run_steps(fn, jobs, **data):
    JOB.update(data)
    return _pool(fn, jobs)


# ---- rl-mlp: the torch port in float64 -------------------------------------------------------------------------------
def mlp_prepass(pool, flat, chunk=64):
    """float64 value and candidate log-probs of every pool state through the rl-mlp port."""
    P = KO.mlp_params64(flat)
    out = []
    for a in range(0, len(pool), chunk):
        sts = pool[a:a + chunk]
        b = MP.stack_states(sts)
        with torch.no_grad():
            v = MP.value(P, b).reshape(-1).numpy()
        lps = KO.mlp_cand_logp64(flat, sts)
        for j, st in enumerate(sts):
            _, cand = candidates(st)
            out.append((float(v[j]), (cand, lps[j])))
    return out
