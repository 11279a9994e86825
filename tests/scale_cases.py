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
import vclip_oracle as VO
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


def all_options_minibatch(flat, states, actions, adv, ret, flp, exps, old_v, lp_old, value_clip, beta,
                          clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01):
    """One minibatch with the clipped value loss and the KL penalty, in float64: ON.forward / ON.backward with the value
    seed of vclip_oracle.seed64 and the KL logit seed of klpen_oracle.kl64 (fed to ON.backward as
    klpen_oracle.ppo_minibatch does).  The statistics sums of slots 1, 2, 15 and 18 and the flat gradient."""
    P = ON._p64(flat)
    n = len(states)
    adv, ret, flp = (np.asarray(x, np.float64).reshape(-1) for x in (adv, ret, flp))
    ind = set(np.flatnonzero(np.asarray(exps).reshape(-1) != 0).tolist())
    n_ind = max(len(ind), 1)
    fws = []
    for i, st in enumerate(states):
        g = ON.unpad(st)
        sid = int(np.argmax(g.stage[:2]))
        fws.append((g, ON.forward(P, g, action=int(actions[i, sid]), keep=True)))
    gv, vl_terms, _ = VO.seed64([fw["value"] for _, fw in fws], ret, old_v, value_clip)
    G = {k: np.zeros_like(v) for k, v in P.items()}
    surr = ent = kl = 0.0
    for i, (g, fw) in enumerate(fws):
        g_lp = g_en = 0.0
        if i in ind:
            r = np.exp(fw["log_prob"] - flp[i])
            s1, s2 = r * adv[i], np.clip(r, 1 - clip_epsilon, 1 + clip_epsilon) * adv[i]
            surr += -min(s1, s2)
            ent += -fw["entropy"]
            if (1 - clip_epsilon) <= r <= (1 + clip_epsilon) or s1 < s2:
                g_lp = -adv[i] * r / n_ind
            g_en = -entropy_coef / n_ind
        Gi = ON.backward(P, g, fw, value_pred_coef * gv[i] / n, g_lp, g_en)
        c = fw["cache"]
        if i in ind and c.get("logp") is not None and c["logp"].size:
            kl_g, seed = KO.kl64(lp_old[i], c["logp"])
            kl += kl_g
            G2 = ON.backward(P, g, dict(fw, cache=dict(c, p=beta / n_ind * seed), action_pos=-1), 0.0, -1.0, 0.0)
            Gi = {k: Gi[k] + G2[k] for k in Gi}
        for k in G:
            G[k] += Gi[k]
    grad = np.zeros(PL.NUM_PARAMS)
    for s in PL.SLOTS.values():
        grad[s.offset:s.offset + s.size] = G[s.name].reshape(-1)
    return dict(surr_sum=surr, ent_sum=ent, vclip_sum=float(vl_terms.sum()), kl_sum=kl, n=n, n_ind=len(ind), grad=grad)


def _all_options_step(job):
    flat, ids, adv = job
    J = JOB
    return all_options_minibatch(flat, [J["states"][i] for i in ids], J["actions"][ids], adv[ids], J["ret"][ids],
                                 J["fixed"][ids], J["exps"][ids], J["old_values"][ids], [J["lp_old"][i] for i in ids],
                                 J["value_clip"], J["beta"])


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


def mlp_step(flat, states, actions, adv, ret, fixed, exps, clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01,
             chunk=32):
    """One rl-mlp minibatch in float64 through the port's autograd, in sub-batches (the padded land-use features of 256
    graphs are 400 MB in float64): the four losses and the flat gradient."""
    P = KO.mlp_params64(flat, requires_grad=True)
    n = len(states)
    exps = np.asarray(exps).reshape(-1)
    n_ind = max(int((exps != 0).sum()), 1)
    sums = np.zeros(3)
    for a in range(0, n, chunk):
        sl = slice(a, min(a + chunk, n))
        b = MP.stack_states(states[sl])
        v = MP.value(P, b).reshape(-1)
        lp, en = MP.log_prob_entropy(P, b, torch.tensor(actions[sl]))
        lp, en = lp.reshape(-1), en.reshape(-1)
        ind = torch.tensor(exps[sl] != 0)
        r = torch.exp(lp - torch.tensor(fixed[sl], dtype=torch.float64).reshape(-1))
        A = torch.tensor(adv[sl], dtype=torch.float64).reshape(-1)
        surr = -torch.min(r * A, torch.clamp(r, 1 - clip_epsilon, 1 + clip_epsilon) * A)[ind].sum()
        ent = -en[ind].sum()
        vl = (v - torch.tensor(ret[sl], dtype=torch.float64).reshape(-1)).pow(2).sum()
        loss = surr / n_ind + value_pred_coef * vl / n + entropy_coef * ent / n_ind
        loss.backward()
        sums += [vl.item(), surr.item(), ent.item()]
    grad = PL.MLP.flatten({k: (t.grad.numpy() if t.grad is not None else np.zeros(tuple(t.shape)))
                           for k, t in P.items()})
    vl, sl_, el = sums[0] / n, sums[1] / n_ind, sums[2] / n_ind
    return dict(loss=sl_ + value_pred_coef * vl + entropy_coef * el, value_loss=vl, surr_loss=sl_, entropy_loss=el,
                grad=np.asarray(grad, np.float64))
