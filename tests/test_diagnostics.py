"""CPU: the PPO diagnostics formed from summed statistics rows and squared gradient norms
(drl_urban_planning_b200/diagnostics.py) against known answers, and their invariance to splitting a minibatch into
rank shards."""
import numpy as np

from drl_urban_planning_b200.diagnostics import NAMES, ppo_diagnostics


def stat_terms(V, R, logp, flp, exps, eps=0.2):
    """Per-graph terms of statistics slots 0-12 as the step kernels add them (include/upb200.h), in float64."""
    V, R, logp, flp, exps = (np.asarray(x, np.float64) for x in (V, R, logp, flp, exps))
    B = V.shape[0]
    ind = exps != 0
    d = logp - flp
    r = np.exp(d)
    rows = np.zeros((B, 16))
    rows[:, 0] = (V - R) ** 2
    rows[:, 3] = 1.0
    rows[:, 4] = ind
    rows[:, 8] = np.where(ind, np.expm1(d) - d, 0.0)
    rows[:, 9] = np.where(ind & ~((r >= 1 - eps) & (r <= 1 + eps)), 1.0, 0.0)
    rows[:, 10] = R
    rows[:, 11] = R * R
    rows[:, 12] = V - R
    return rows


def sums(V, R, logp, flp, exps, eps=0.2):
    return stat_terms(V, R, logp, flp, exps, eps).sum(0, keepdims=True)


def test_kl_is_zero_when_the_policy_did_not_move():
    rng = np.random.default_rng(0)
    lp = rng.normal(-3.0, 1.0, 32)
    d = ppo_diagnostics(sums(rng.normal(size=32), rng.normal(size=32), lp, lp, np.ones(32)), np.ones((1, 3)))
    assert d["approx_kl"][0] == 0.0 and d["clip_fraction"][0] == 0.0


def test_kl_matches_the_ratio_estimator():
    rng = np.random.default_rng(1)
    flp = rng.normal(-3.0, 1.0, 64)
    lp = flp + rng.normal(0.0, 0.1, 64)
    exps = np.ones(64); exps[::3] = 0.0
    d = ppo_diagnostics(sums(np.zeros(64), rng.normal(size=64), lp, flp, exps), np.ones((1, 3)))
    ind = exps != 0
    r = np.exp(lp - flp)[ind]
    want = ((r - 1) - np.log(r)).mean()
    assert want > 0 and abs(d["approx_kl"][0] - want) <= 1e-12 * want + 1e-15


def test_clip_counts_are_exact_at_ratios_clearly_inside_and_outside():
    ratios = np.array([1.0, 0.9, 1.1, 0.81, 1.19, 0.5, 0.79, 1.21, 2.0, 1e-3])
    outside = np.array([0, 0, 0, 0, 0, 1, 1, 1, 1, 1], bool)
    flp = np.full(ratios.size, -2.0)
    lp = flp + np.log(ratios)
    exps = np.ones(ratios.size)
    d = ppo_diagnostics(sums(np.zeros(ratios.size), np.arange(ratios.size), lp, flp, exps), np.ones((1, 3)))
    assert d["clip_fraction"][0] == outside.sum() / ratios.size
    # graphs with exps == 0 are not counted, and the fraction is over |ind| only
    exps[outside.nonzero()[0][:2]] = 0.0
    d = ppo_diagnostics(sums(np.zeros(ratios.size), np.arange(ratios.size), lp, flp, exps), np.ones((1, 3)))
    assert d["clip_fraction"][0] == (outside.sum() - 2) / (ratios.size - 2)


def test_explained_variance_known_answers():
    rng = np.random.default_rng(2)
    R = rng.normal(1.0, 2.0, 40)
    lp = np.zeros(40)
    one = ppo_diagnostics(sums(R, R, lp, lp, np.ones(40)), np.ones((1, 3)))
    assert one["explained_variance"][0] == 1.0
    zero = ppo_diagnostics(sums(np.full(40, R.mean()), R, lp, lp, np.ones(40)), np.ones((1, 3)))
    assert abs(zero["explained_variance"][0]) < 1e-12
    V = R + rng.normal(0.0, 0.5, 40)
    got = ppo_diagnostics(sums(V, R, lp, lp, np.ones(40)), np.ones((1, 3)))["explained_variance"][0]
    assert abs(got - (1 - np.var(V - R) / np.var(R))) < 1e-12
    for c in (0.0, 0.1, 3.7, -12.25):                     # constant returns: no spread to explain
        flat = ppo_diagnostics(sums(V, np.full(40, c), lp, lp, np.ones(40)), np.ones((1, 3)))
        assert np.isnan(flat["explained_variance"][0]), c


def test_all_zero_exps_and_empty_rows_do_not_divide_by_zero():
    rng = np.random.default_rng(3)
    lp = rng.normal(size=8)
    with np.errstate(all="raise"):
        d = ppo_diagnostics(sums(rng.normal(size=8), rng.normal(size=8), lp, lp - 1.0, np.zeros(8)), np.zeros((1, 3)))
        assert d["approx_kl"][0] == 0.0 and d["clip_fraction"][0] == 0.0
        assert d["grad_norm_policy"][0] == 0.0 and d["grad_norm_value"][0] == 0.0
        empty = ppo_diagnostics(np.zeros((1, 16)), np.zeros((1, 3)))
    assert empty["approx_kl"][0] == 0.0 and np.isnan(empty["explained_variance"][0])


def test_gradient_norms_are_the_two_clip_group_totals():
    sq = np.array([[4.0, 5.0, 12.0], [0.0, 9.0, 16.0]])
    d = ppo_diagnostics(np.zeros((2, 16)), sq)
    assert np.array_equal(d["grad_norm_policy"], [3.0, 3.0])
    assert np.array_equal(d["grad_norm_value"], [4.0, 4.0])


def test_rank_shards_sum_to_the_same_diagnostics():
    """Every input is a sum over graphs: the shards order[i*B:(i+1)*B][rank::world] of several ranks, summed, give the
    diagnostics of one rank holding the whole minibatch."""
    rng = np.random.default_rng(4)
    B, nb = 48, 3
    V, R = rng.normal(size=B * nb), rng.normal(0.5, 1.5, B * nb)
    flp = rng.normal(-3.0, 1.0, B * nb)
    lp = flp + rng.normal(0.0, 0.3, B * nb)
    exps = (rng.random(B * nb) > 0.2).astype(np.float64)
    terms = stat_terms(V, R, lp, flp, exps)
    sq = rng.random((nb, 3))
    whole = ppo_diagnostics(np.stack([terms[i * B:(i + 1) * B].sum(0) for i in range(nb)]), sq)
    for world in (2, 3, 8):
        per_rank = [np.stack([terms[i * B:(i + 1) * B][rank::world].sum(0) for i in range(nb)]) for rank in range(world)]
        split = ppo_diagnostics(sum(per_rank), sq)
        for name in NAMES:
            assert np.allclose(split[name], whole[name], rtol=1e-12, atol=1e-15), (world, name)
