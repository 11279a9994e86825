"""Graphs at the shape limits where the SGNN and rl-mlp kernels change code path (csrc/sgnn_kernel.cuh,
csrc/mlp_kernel.cuh; static_asserts there pin the values below to this file's cases), built with exact sizes by
synth.make_exact_state on the hlg caps (1000 nodes, 3000 edges).  Used by tests/test_packing.py (CPU) and
tests/test_gpu_shapes.py (GPU)."""
import numpy as np

from drl_urban_planning_b200 import synth

NS, AS, KS = 464, 5632, 160      # shared-memory fast path: n <= NS, 2e <= AS, k <= KS; beyond it, global scratch
XEARLY_NODES = 381               # encoder-backward features come back early (dead list stretch) up to this n
HIN_NODES = 416                  # g_W reads the h rows from shared memory up to this n, from L2 beyond
CH = 96                          # candidate chunk of the head backward
SPEC = synth.COMMUNITIES["hlg"]

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
