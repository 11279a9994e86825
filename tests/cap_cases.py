"""Graphs above the hlg caps: the shipped concept configs' caps (1500 nodes, 4000 edges) and the blob format's 16-bit
limits (csrc/blob.h: n_cap <= 65535, 2 e_cap <= 65535), each built with exact sizes by synth.make_exact_state.

In the blob a node id is a uint16 (0xFFFF is the pull schedule's "no node"), a CSR row pointer a uint16 running up to
2e, an adjacency entry `neighbour | (slot + 1) << 16 | first << 31` with a 15-bit slot field, and a candidate edge
`u | v << 16`.  The cases below put a value with bit 15 set into every one of these fields: node ids 32768 .. 65534
(both halves of cand_uv), row pointers 32768 .. 65534, slot + 1 = 32767, and the longest row the format holds (a hub of
degree 32767).  Used by tests/test_caps.py (CPU) and tests/test_gpu_caps.py (H100)."""
import numpy as np

from drl_urban_planning_b200 import synth

CONCEPT = synth.COMMUNITIES["hlg_concept"]                   # 1500 / 4000, as shipped
ABI = synth.CommunitySpec("abi", 65535, 32767, 200, 400, 5.0, 0.3)
MAX_N, MAX_E = ABI.max_num_nodes, ABI.max_num_edges          # the largest caps upb_create and the packer accept
TOP = MAX_N - 1                                              # 65534: the largest node id (0xFFFF is kNoNode)
MAX_LU_K = MAX_E                                             # land-use candidates: k <= e <= e_cap; slot + 1 = 32767
MAX_ROAD_K = MAX_N                                           # road candidates: k <= n <= n_cap

# label, n, e, k, stage, hub, isolated
CONCEPT_CASES = [
    ("c_lu_full", 1500, 4000, 4000, 0, False, 0),            # every edge a candidate
    ("c_road", 1500, 4000, 1500, 1, False, 0),               # every node a candidate
    ("c_past_hlg", 1001, 3001, 3001, 0, False, 0),           # one past each hlg cap
    ("c_hub", 1500, 4000, 200, 0, True, 0),                  # a hub row of degree 1499
]
ABI_CASES = [
    ("n32768_lu", 32768, 20000, 3000, 0, False, 0),
    ("n32768_road", 32768, 20000, 3000, 1, False, 0),
    ("n32769_lu", 32769, 20000, 3000, 0, False, 0),          # node 32768: the first id with bit 15 set
    ("n32769_road", 32769, 20000, 3000, 1, False, 0),
    ("rp_e16383", 30000, 16383, 500, 0, False, 0),           # last row pointer 32766, 32768, 32770
    ("rp_e16384", 30000, 16384, 500, 1, False, 0),
    ("rp_e16385", 30000, 16385, 500, 0, False, 0),
    ("hub32767", 32768, 32767, 1000, 0, True, 0),            # the longest row: degree 32767, row pointers 0 .. 65534
    ("max_lu", MAX_N, MAX_E, MAX_LU_K, 0, False, 1),         # every edge a candidate: slot + 1 up to 32767
    ("max_road", MAX_N, MAX_E, MAX_ROAD_K, 1, False, 1),     # every node a candidate, node 65534 among them
    # 32767 live nodes spread over ids 0 .. 65534, about two edges each: half of every pull's neighbour ids, in the
    # two-neighbour trips as well as the single tail, have bit 15 set (the graphs above have degree 1 there)
    ("dense_high", MAX_N, MAX_E, 4000, 0, False, 32768),
]
# cases whose hub row alone outweighs the pull schedule's balance bound (see test_caps.py)
UNBALANCED = {"hub32767"}


def _build(rng, spec, row):
    label, n, e, k, stage, hub, isolated = row
    if not isolated:
        return synth.make_exact_state(rng, spec, n, e, k, stage, hub=hub, isolated=isolated)
    # the lone node is never the top id, so node n - 1 is an endpoint (at max_lu the second endpoint of a candidate);
    # at max_lu node n - 2's edge is stored the other way round, (n - 2, u) with u < n - 2, so that a node id with bit
    # 15 set lands in cand_uv's lower half too (the packer and the kernels take either orientation, as the reference)
    for _ in range(64):
        st, a = synth.make_exact_state(rng, spec, n, e, k, stage, hub=hub, isolated=isolated)
        ei = st[2]
        if ei[:e].max() != n - 1:
            continue
        if label == "max_lu":
            j = np.flatnonzero(ei[:e, 1] == n - 2)
            if j.size != 1:
                continue
            ei[j[0]] = ei[j[0], ::-1].copy()
        return st, a
    raise AssertionError(label)


def _batch(spec, rows, seed, fillers):
    """(states, actions, labels): the rows' graphs with `fillers` ordinary concept-sized graphs (padded to the spec's
    caps) between them, so that one CTA walking the batch in order goes big -> small -> big."""
    rng = np.random.default_rng(seed)
    states, acts, labels = [], [], []
    for i, row in enumerate(rows):
        st, a = _build(rng, spec, row)
        states.append(st); acts.append((int(row[4]), a)); labels.append(row[0])
        if i < fillers:
            small, sa = synth.make_state(rng, spec, n=int(rng.integers(CONCEPT.n_lo, CONCEPT.n_hi + 1)),
                                         stage=i % 2)
            states.append(small); acts.append((i % 2, sa)); labels.append(f"small{i}")
    actions = np.zeros((len(states), 2), np.float32)
    for i, (s, a) in enumerate(acts):
        actions[i, s] = a
    return states, actions, labels


def concept_batch(seed=0):
    """The concept-cap cases, each followed by an ordinary concept graph."""
    return _batch(CONCEPT, CONCEPT_CASES, seed, len(CONCEPT_CASES))


def abi_batch(seed=1, rows=ABI_CASES, fillers=2):
    """The ABI-limit cases on 65535 / 32767 caps, the first `fillers` followed by an ordinary concept-sized graph."""
    return _batch(ABI, rows, seed, fillers)


def abi_case(label, seed=1):
    """One ABI-limit case alone: (state, action row)."""
    rows = [r for r in ABI_CASES if r[0] == label]
    states, actions, _ = _batch(ABI, rows, seed + 1000 * ABI_CASES.index(rows[0]), 0)
    return states[0], actions[0]
