"""Graphs at the shape limits where the SGNN and rl-mlp kernels change code path (csrc/sgnn_kernel.cuh,
csrc/mlp_kernel.cuh; static_asserts there pin the values below to this file's cases), built with exact sizes by
synth.make_exact_state on the hlg caps (1000 nodes, 3000 edges).  Used by tests/test_packing.py (CPU) and the GPU tests."""
import numpy as np

from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.packing import pack_states
from harness import t
from oracle import sgnn_numpy as ON

NS, AS, KS = 464, 5632, 160      # shared-memory fast path: n <= NS, 2e <= AS, k <= KS; beyond it, global scratch
XEARLY_NODES = 381               # encoder-backward features come back early (dead list stretch) up to this n
HIN_NODES = 416                  # g_W reads the h rows from shared memory up to this n, from L2 beyond
CH = 96                          # candidate chunk of the head backward
SPEC = synth.COMMUNITIES["hlg"]
BATCH_SEED = 3                   # Batch: the boundary batch of the GPU tests

# label, n, e, k, stage, hub, isolated
BOUNDARY = [
    # n alone decides the path (e, k small)
    ("n381", 381, 900, 40, 0, False, 0),
    ("n382", 382, 900, 40, 1, False, 0),
    ("n416", 416, 1000, 40, 0, False, 0),
    ("n417", 417, 1000, 40, 1, False, 0),
    ("n463", 463, 1100, 40, 0, False, 0),
    ("n464", 464, 1100, 40, 0, False, 0),
    ("n464r", 464, 1100, 40, 1, False, 0),
    ("n465", 465, 1100, 40, 0, False, 0),
    ("n465r", 465, 1100, 40, 1, False, 0),
    # 2e alone decides (n <= NS); e = 2815 is odd, so the adjacency copy is rounded up to 16 bytes
    ("e2815", 464, 2815, 40, 0, False, 0),
    ("e2816", 460, 2816, 40, 1, False, 0),
    ("e2817", 450, 2817, 40, 0, False, 0),
    # k alone decides (n <= NS, 2e <= AS): one and two head-backward chunks, the shared-memory candidate limit
    ("k96", 300, 1500, 96, 0, False, 0),
    ("k97", 300, 1500, 97, 0, False, 0),
    ("k160", 300, 1500, 160, 0, False, 0),
    ("k161", 300, 1500, 161, 0, False, 0),
    ("k192", 300, 1500, 192, 0, False, 0),
    ("k193", 300, 1500, 193, 0, False, 0),
    ("road_k160", 400, 1200, 160, 1, False, 0),
    ("road_k161", 400, 1200, 161, 1, False, 0),
    # a hub row (degree n - 1) at the node limit, isolated nodes (degree 0)
    ("hub", 464, 2000, 60, 0, True, 0),
    ("isolated", 200, 600, 30, 1, False, 12),
    # around the 16-row tensor-core tiles of g_h
    ("n15", 15, 30, 8, 0, False, 0),
    ("n16", 16, 30, 8, 1, False, 0),
    ("n17", 17, 30, 8, 0, False, 0),
    # the caps: every edge a candidate
    ("caps", 1000, 3000, 3000, 0, False, 0),
]


def is_big(n, e, k):
    return n > NS or 2 * e > AS or k > KS


def boundary_batch(seed=0):
    """(states, actions, labels): one state per BOUNDARY row, in that order."""
    rng = np.random.default_rng(seed)
    states, actions, labels = [], np.zeros((len(BOUNDARY), 2), np.float32), []
    for i, (label, n, e, k, stage, hub, isolated) in enumerate(BOUNDARY):
        st, a = synth.make_exact_state(rng, SPEC, n, e, k, stage, hub=hub, isolated=isolated)
        states.append(st)
        actions[i, stage] = a
        labels.append(label)
    return states, actions, labels


def degrees(state):
    n, e = int(state[4].sum()), int(state[5].sum())
    ei = state[2][:e]
    return np.bincount(ei[:, 0], minlength=n) + np.bincount(ei[:, 1], minlength=n)


def big_states(seed, count):
    """Graphs beyond the shared-memory fast path (n > 464 or 2e > 5632 or > 160 candidates), up to the caps."""
    spec = synth.CommunitySpec("big", 1000, 3000, 470, 1000, 3.0, 0.3)
    rng = np.random.default_rng(seed)
    states, actions = [], np.zeros((count, 2), np.float32)
    for i in range(count):
        n = 1000 if i == 0 else None            # node cap reached
        st, a = synth.make_state(rng, spec, n=n)
        if i == 1:                               # every real edge is an action candidate (k = e > 256)
            st[8][:] = [1, 0, 0]
            st[7][:] = False
            st[6][:int(st[5].sum())] = True
            a = 5
        states.append(st)
        actions[i, int(st[8].argmax())] = a
    return states, actions


class Batch:
    def __init__(self, dev):
        self.states, self.actions, self.labels = boundary_batch(BATCH_SEED)
        self.count = len(self.states)
        self.adv, self.ret, self.exps = synth.make_ppo_targets(BATCH_SEED, self.count)
        self.exps[5] = 0.0
        self.fixed = np.random.default_rng(BATCH_SEED).normal(-3.0, 0.3, size=(self.count, 1)).astype(np.float32)
        self.flat = PL.default_init(BATCH_SEED)
        self.blob = pack_states(self.states).to(dev)
        self.info = self.blob.info.astype(np.int64)
        self.big = np.array([is_big(*r[:3]) for r in self.info])
        self.dev_args = tuple(t(x, dev) for x in (self.actions, self.adv, self.ret, self.fixed, self.exps))
        self.n_ind = int((self.exps != 0).sum())

    def oracle(self, flat, sel=None):
        sel = np.arange(self.count) if sel is None else np.asarray(sel)
        return ON.ppo_minibatch(flat, [self.states[i] for i in sel], self.actions[sel], self.adv[sel], self.ret[sel],
                                self.fixed[sel], self.exps[sel])


def walk_order(b):
    """The batch's graph ids in an order that makes one CTA walk fast -> big -> fast, big-because-of-k -> a few
    candidates, land-use -> road: big and fast graphs alternate, each big graph followed by a small-k fast graph."""
    k = b.info[:, 2]
    big = [i for i in range(b.count) if b.big[i]]
    fast = sorted((i for i in range(b.count) if not b.big[i]), key=lambda i: k[i])     # fewest candidates first
    out = []
    for i in big:
        out += [fast.pop(0), i]
    out += fast
    assert sorted(out) == list(range(b.count))
    return out


def placed(walk, grid):
    """ids such that CTA c walks the c-th contiguous piece of `walk` (item i -> CTA i % grid, round i // grid)."""
    count = len(walk)
    ids, pos = np.zeros(count, np.int32), 0
    for c in range(grid):
        slots = list(range(c, count, grid))
        ids[slots] = walk[pos:pos + len(slots)]
        pos += len(slots)
    return ids
