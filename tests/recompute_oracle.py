"""Float64 oracle of the targets one more PPO epoch trains on with recompute_advantage (upb_gae_targets): GAE on the value
head's outputs, each episode scanned on its own, and with value normalisation the head's outputs denormalised and the
returns normalised by tests/vnorm_oracle.py's fp32 operations with fixed statistics."""
from __future__ import annotations

import numpy as np

import vnorm_oracle as VN


def episodes(masks):
    """(first, last) of every episode: an episode ends where masks == 0, and the last one at T - 1."""
    masks = np.asarray(masks).reshape(-1)
    ends = np.flatnonzero(masks == 0)
    if not ends.size or ends[-1] != masks.size - 1:
        ends = np.r_[ends, masks.size - 1]
    return list(zip(np.r_[0, ends[:-1] + 1], ends))


def gae64(rewards, masks, values, gamma, tau):
    """estimate_advantages (khrylib/rl/core/common.py:5-26) in float64, one episode at a time from zero:
    (advantages, returns)."""
    r, m, v = (np.asarray(x, np.float64).reshape(-1) for x in (rewards, masks, values))
    adv = np.zeros(r.size)
    for a, e in episodes(m):
        prev_v = prev_a = 0.0
        for i in range(e, a - 1, -1):
            d = r[i] + gamma * prev_v * m[i] - v[i]
            adv[i] = d + gamma * tau * prev_a * m[i]
            prev_v, prev_a = v[i], adv[i]
    return adv, v + adv


def targets(rewards, masks, head, gamma, tau, state=None):
    """(advantages, returns, anchors) in float64 from the head outputs `head`.  state: the value normaliser's state
    (m1, m2, d), or None while value normalisation is off.  On, the values are fmaf(fp32 std, head, fp32 mean) (the head
    itself while d == 0) and the returns (R - fp32 mean) / fp32 std; the anchors are the head outputs."""
    n = np.asarray(head, np.float32).reshape(-1)
    values = n if state is None else VN.denormalize(n, state)
    adv, ret = gae64(rewards, masks, values, gamma, tau)
    if state is not None:
        mu, sd = VN.stats(*state)
        ret = (ret - float(np.float32(mu))) / float(np.float32(sd))
    return adv, ret, n.astype(np.float64)
