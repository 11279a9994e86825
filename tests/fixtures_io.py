"""Compact (unpadded) storage of reference-format rollout states inside the golden .npz fixtures."""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np


def compact_states(states: Sequence[Sequence[np.ndarray]]) -> Dict[str, np.ndarray]:
    ns = np.array([int(s[4].sum()) for s in states], dtype=np.int32)
    es = np.array([int(s[5].sum()) for s in states], dtype=np.int32)
    out = dict(
        n=ns, e=es,
        n_cap=np.int32(states[0][1].shape[0]), e_cap=np.int32(states[0][2].shape[0]),
        numerical=np.stack([s[0] for s in states]).astype(np.float32),
        current_node=np.stack([s[3] for s in states]).astype(np.float32),
        stage=np.stack([s[8] for s in states]).astype(np.float32),
        node_features=np.concatenate([s[1][:n] for s, n in zip(states, ns)]).astype(np.float32),
        edges=np.concatenate([s[2][:e] for s, e in zip(states, es)]).astype(np.int32),
        land_use_mask=np.concatenate([s[6][:e] for s, e in zip(states, es)]).astype(bool),
        road_mask=np.concatenate([s[7][:n] for s, n in zip(states, ns)]).astype(bool),
    )
    return out


def expand_states(z) -> List[list]:
    """Inverse of compact_states: the padded 9-array states the reference consumes."""
    N, E = int(z["n_cap"]), int(z["e_cap"])
    states, no, eo = [], 0, 0
    for i, (n, e) in enumerate(zip(z["n"], z["e"])):
        n, e = int(n), int(e)
        nf = np.zeros((N, z["node_features"].shape[1]), np.float32); nf[:n] = z["node_features"][no:no + n]
        ei = np.full((E, 2), N - 1, np.int64); ei[:e] = z["edges"][eo:eo + e]
        nm = np.zeros(N, bool); nm[:n] = True
        em = np.zeros(E, bool); em[:e] = True
        lm = np.zeros(E, bool); lm[:e] = z["land_use_mask"][eo:eo + e]
        rm = np.zeros(N, bool); rm[:n] = z["road_mask"][no:no + n]
        states.append([z["numerical"][i].copy(), nf, ei, z["current_node"][i].copy(), nm, em, lm, rm,
                       z["stage"][i].copy()])
        no += n; eo += e
    return states


def synth_states(seed: int, community: str, count: int):
    """The seeded states and actions of a golden fixture that stores no states.  `community` names one community, or
    several joined by '+' for a minibatch mixing them (synth.make_mixed_states)."""
    from drl_urban_planning_b200 import synth
    if "+" in community:
        return synth.make_mixed_states(seed, community.split("+"), count)
    return synth.make_states(seed, community, count)


def states_digest(states) -> str:
    """sha256 over the compact form of the states (the big golden fixtures store this instead of the states, which
    are regenerated from the seed by drl_urban_planning_b200/synth.py)."""
    import hashlib
    h = hashlib.sha256()
    c = compact_states(states)
    for k in sorted(c):
        h.update(np.ascontiguousarray(c[k]).tobytes())
    return h.hexdigest()
