"""Seeded synthetic rollout states in the reference's own 9-array layout.

The geometry environment (`urban_planning/envs/city.py`, geopandas stack) cannot run in this image,
so every input of the update path is synthetic.  The layout is the contract of
`ObservationExtractor.get_obs` (reference `urban_planning/envs/observation_extractor.py:207-228`):

    [numerical (52,) f32, node_features (N,23) f32, edge_index (E,2) i64 (pad value N-1),
     current_node (23,) f32, node_mask (N,) bool, edge_mask (E,) bool,
     land_use_mask (E,) bool, road_mask (N,) bool, stage (3,) f32 one-hot]

Shapes and distributions follow SURVEY.md section 8(d): HLG n~U{223..400}, e~5.45 n; DHM n~U{269..460},
e~5.55 n; concept caps 1500/4000; grid n~U{81..160} with both stages.  Graphs are contiguity-like:
n points in the unit square joined to their nearest neighbours, every undirected edge stored once with
u < v and the list sorted by u (the order `np.array(nx.Graph.edges)` yields, plan_client.py:823).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

NODE_DIM = 23          # 14 one-hot types + 9 reals (observation_extractor.py:112-121)
NUM_TYPE_SLOTS = 14    # city_config.NUM_TYPES + 1
NUMERICAL_DIM = 52     # observation_extractor.py:38,49,193
STAGE_DIM = 3          # ['land_use', 'road', 'done'] (city.py:139)

# type ids (city_config.py:26-58)
_ROAD, _BOUNDARY, _INTERSECTION = 2, 3, 13
_POLYGON_TYPES = (1, 4, 5, 6, 7, 8, 9, 10, 11, 12)


@dataclass(frozen=True)
class CommunitySpec:
    name: str
    max_num_nodes: int
    max_num_edges: int
    n_lo: int
    n_hi: int
    edge_ratio: float
    road_stage_prob: float  # fraction of states in stage 1 ('road')


COMMUNITIES = {
    # caps: cfg/exp_cfg/real/hlg.yaml:27-28 ; sizes: SURVEY.md section 8(d) / appendix B
    "hlg": CommunitySpec("hlg", 1000, 3000, 223, 400, 5.45, 0.0),
    "dhm": CommunitySpec("dhm", 1000, 3000, 269, 460, 5.55, 0.0),
    "grid": CommunitySpec("grid", 1000, 3000, 81, 160, 5.45, 0.3),
    "hlg_concept": CommunitySpec("hlg_concept", 1500, 4000, 226, 410, 5.50, 0.0),
    "dhm_concept": CommunitySpec("dhm_concept", 1500, 4000, 272, 470, 5.55, 0.0),
    # small shapes for fixtures and fast parity tests (caps chosen small so the padded oracle is quick)
    "tiny": CommunitySpec("tiny", 48, 160, 6, 40, 3.2, 0.4),
    "small": CommunitySpec("small", 128, 512, 20, 120, 4.0, 0.3),
}


def _knn_edges(rng: np.random.Generator, n: int, e_target: int) -> np.ndarray:
    """Undirected contiguity-like edge list, u < v, sorted by (u, v), exactly min(e_target, n(n-1)/2) rows."""
    e_target = int(min(e_target, n * (n - 1) // 2))
    if e_target <= 0 or n < 2:
        return np.zeros((0, 2), dtype=np.int64)
    pts = rng.random((n, 2))
    d2 = ((pts[:, None, :] - pts[None, :, :]) ** 2).sum(-1)
    iu, iv = np.triu_indices(n, k=1)
    order = np.argsort(d2[iu, iv], kind="stable")
    # keep every node attached: first its nearest neighbour, then globally shortest pairs
    nn = np.argsort(d2 + np.eye(n) * 1e9, axis=1)[:, 0]
    pairs = set()
    for i in range(n):
        a, b = (i, int(nn[i])) if i < nn[i] else (int(nn[i]), i)
        if len(pairs) < e_target:
            pairs.add((a, b))
    for k in order:
        if len(pairs) >= e_target:
            break
        pairs.add((int(iu[k]), int(iv[k])))
    edges = np.array(sorted(pairs), dtype=np.int64).reshape(-1, 2)
    return edges


def make_state(rng: np.random.Generator, spec: CommunitySpec, n: Optional[int] = None,
               stage: Optional[int] = None, e: Optional[int] = None) -> Tuple[list, int]:
    """One rollout state + a feasible action index for its active stage.

    Returns (state, action_index) with `state` the 9-array list described in the module docstring.
    """
    N, E = spec.max_num_nodes, spec.max_num_edges
    if n is None:
        n = int(rng.integers(spec.n_lo, spec.n_hi + 1))
    n = int(min(n, N))
    if e is None:
        e = int(round(spec.edge_ratio * n * (1.0 + rng.uniform(-0.05, 0.05))))
    e = int(min(e, E))
    edges = _knn_edges(rng, n, e)
    e = edges.shape[0]
    if stage is None:
        stage = int(rng.random() < spec.road_stage_prob)

    kind = rng.choice(3, size=n, p=[0.50, 0.32, 0.18])       # segment / intersection / polygon
    types = np.where(kind == 0, np.where(rng.random(n) < 0.8, _ROAD, _BOUNDARY),
                     np.where(kind == 1, _INTERSECTION, rng.choice(_POLYGON_TYPES, size=n)))
    node_features = np.zeros((N, NODE_DIM), dtype=np.float32)
    node_features[np.arange(n), types] = 1.0
    node_features[:n, NUM_TYPE_SLOTS:] = rng.uniform(-1, 1, size=(n, NODE_DIM - NUM_TYPE_SLOTS)).astype(np.float32)

    edge_index = np.full((E, 2), N - 1, dtype=np.int64)      # pad value N-1 (observation_extractor.py:97)
    edge_index[:e] = edges

    numerical = rng.random(NUMERICAL_DIM).astype(np.float32)
    current_node = np.zeros(NODE_DIM, dtype=np.float32)      # cf. plan_client.py:337-345
    current_node[int(rng.choice(_POLYGON_TYPES))] = 1.0
    current_node[NUM_TYPE_SLOTS + 2:NUM_TYPE_SLOTS + 6] = rng.uniform(-1, 1, size=4).astype(np.float32)
    current_node[NUM_TYPE_SLOTS + 6:] = 1.0

    node_mask = np.zeros(N, dtype=bool); node_mask[:n] = True
    edge_mask = np.zeros(E, dtype=bool); edge_mask[:e] = True
    land_use_mask = np.zeros(E, dtype=bool)
    road_mask = np.zeros(N, dtype=bool)
    stage_vec = np.zeros(STAGE_DIM, dtype=np.float32)
    stage_vec[stage] = 1.0
    if stage == 0:
        k = int(min(max(e, 1), rng.integers(20, 121)))
        k = max(1, min(k, e)) if e > 0 else 0
        idx = rng.choice(e, size=k, replace=False) if e > 0 else np.zeros(0, dtype=np.int64)
        land_use_mask[idx] = True
        action = int(rng.choice(idx)) if k > 0 else 0
    else:
        seg = np.flatnonzero(kind == 0)
        if seg.size == 0:
            seg = np.arange(n)
        k = int(max(1, rng.integers(1, seg.size + 1)))
        idx = rng.choice(seg, size=k, replace=False)
        road_mask[idx] = True
        action = int(rng.choice(idx))

    state = [numerical, node_features, edge_index, current_node, node_mask, edge_mask,
             land_use_mask, road_mask, stage_vec]
    return state, action


def make_exact_state(rng: np.random.Generator, spec: CommunitySpec, n: int, e: int, k: int, stage: int,
                     hub: bool = False, isolated: int = 0) -> Tuple[list, int]:
    """One rollout state with exactly `n` nodes, `e` undirected edges and `k` action candidates (land-use edges for
    stage 0, road nodes for stage 1), for tests that need a graph on a given side of a kernel's shape limits.

    `hub`: one node (neither the first nor the last) is joined to every other connected node, so its degree is
    n - 1 - isolated.  `isolated`: exactly that many nodes have no edge (every other node has one).  The other edges
    are distinct random pairs of connected nodes, so node degrees come out of both parities.  The edge-list contract of make_state holds: u < v,
    sorted by (u, v), prefix masks, pad value N - 1.  Returns (state, action) with the action a random candidate."""
    N, E = spec.max_num_nodes, spec.max_num_edges
    assert 1 <= n <= N and 0 <= e <= E and stage in (0, 1) and 0 <= isolated < n
    state, _ = make_state(rng, spec, n=n, stage=stage, e=0)         # features, numerical, current node, stage
    lone = rng.choice(n, size=isolated, replace=False) if isolated else np.zeros(0, np.int64)
    live = np.setdiff1d(np.arange(n), lone)
    pairs = set()
    if hub:
        h = int(live[len(live) // 2])
        pairs.update((min(h, int(j)), max(h, int(j))) for j in live if j != h)
    elif len(live) > 1:          # a random perfect matching (plus one edge for an odd count): no other node is isolated
        p = rng.permutation(live).tolist()
        p += p[:1] if len(p) % 2 else []
        pairs.update((min(u, v), max(u, v)) for u, v in zip(p[0::2], p[1::2]))
    assert len(pairs) <= e <= len(live) * (len(live) - 1) // 2, "edge count out of reach for this graph"
    while len(pairs) < e:
        a, b = live[rng.integers(0, len(live), size=(2, 2 * (e - len(pairs)) + 8))]
        for u, v in zip(a.tolist(), b.tolist()):
            if u != v and len(pairs) < e:
                pairs.add((min(u, v), max(u, v)))
    edges = np.array(sorted(pairs), dtype=np.int64).reshape(-1, 2)
    state[2][:] = N - 1
    state[2][:e] = edges
    state[5][:] = False
    state[5][:e] = True
    state[6][:] = False
    state[7][:] = False
    if stage == 0:
        assert k <= e
        idx = rng.choice(e, size=k, replace=False)
        state[6][idx] = True
    else:
        assert k <= n
        idx = rng.choice(n, size=k, replace=False)
        state[7][idx] = True
    return state, int(rng.choice(idx)) if k else 0


def make_states(seed: int, community: str, count: int, sizes: Optional[Sequence[int]] = None,
                stages: Optional[Sequence[int]] = None) -> Tuple[List[list], np.ndarray]:
    """`count` states of one community plus the (count, 2) float32 action array the reference stores
    (column 0 = land-use edge index, column 1 = road node index; policy.py:67-85)."""
    spec = COMMUNITIES[community]
    rng = np.random.default_rng(seed)
    states, actions = [], np.zeros((count, 2), dtype=np.float32)
    for i in range(count):
        st, a = make_state(rng, spec,
                           n=None if sizes is None else int(sizes[i]),
                           stage=None if stages is None else int(stages[i]))
        states.append(st)
        actions[i, int(st[8].argmax())] = float(a)
    return states, actions


def make_mixed_states(seed: int, communities: Sequence[str], count: int) -> Tuple[List[list], np.ndarray]:
    """Config 5: a minibatch mixing several communities that share caps (hlg_concept + dhm_concept)."""
    specs = [COMMUNITIES[c] for c in communities]
    assert len({(s.max_num_nodes, s.max_num_edges) for s in specs}) == 1, "mixed batches need equal caps"
    rng = np.random.default_rng(seed)
    states, actions = [], np.zeros((count, 2), dtype=np.float32)
    for i in range(count):
        st, a = make_state(rng, specs[i % len(specs)])
        states.append(st)
        actions[i, int(st[8].argmax())] = float(a)
    return states, actions


def make_ppo_targets(seed: int, count: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """advantages, returns ~ N(0,1) as (count,1) float32 and exps == 1 (noise_rate=1.0, agent.py:26)."""
    rng = np.random.default_rng(seed + 7919)
    adv = rng.standard_normal((count, 1)).astype(np.float32)
    ret = rng.standard_normal((count, 1)).astype(np.float32)
    exps = np.ones(count, dtype=np.float32)
    return adv, ret, exps
