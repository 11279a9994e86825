"""CPU: the gradient-noise measurement (grad_noise_every) -- the argument checks before any CUDA call, the host mirror
of the kernels' item-to-CTA assignment, the float64 estimator against synthetic gradients and against McCandlish's
two-batch formula, the cross-rank combination and the update's bookkeeping of the measured rows."""
import numpy as np
import pytest

import grad_noise_oracle as GO
from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.engine import (Engine, check_grad_noise_every, cta_group_sizes, grad_noise_estimate,
                                            grad_noise_terms)
from drl_urban_planning_b200.ppo import KL_SKIP_SLOT, KL_STOP_SLOT, NONFINITE_SLOT, PPOUpdater, UpdateLog
from test_adaptive_lr import fake_agent, no_cuda

BAD = [True, False, np.bool_(True), 1.0, 2.5, np.float64(4.0), 0, -1, np.int64(-3), "2", [2]]


@pytest.mark.parametrize("bad", BAD)
def test_bad_values_are_refused_before_cuda(monkeypatch, bad):
    from drl_urban_planning_b200.agent import use_b200_update
    no_cuda(monkeypatch)
    with pytest.raises(ValueError, match="grad_noise_every"):
        check_grad_noise_every(bad)
    with pytest.raises(ValueError, match="grad_noise_every"):
        Engine("cuda:0", 64, 64, grad_noise_every=bad)
    with pytest.raises(ValueError, match="grad_noise_every"):
        PPOUpdater(PL.default_init(0), 64, 64, "cuda:0", grad_noise_every=bad)
    with pytest.raises(ValueError, match="grad_noise_every"):
        use_b200_update(fake_agent(), grad_noise_every=bad)


def test_good_values_pass():
    assert check_grad_noise_every(None) is None
    assert check_grad_noise_every(1) == 1
    got = check_grad_noise_every(np.int64(8))
    assert got == 8 and type(got) is int


@pytest.mark.parametrize("grid", [1, 64, 132])
@pytest.mark.parametrize("count", [0, 1, 5, 63, 64, 65, 131, 132, 133, 256, 300, 1000])
def test_group_sizes_follow_the_kernels_schedule(count, grid):
    want = [len(g) for g in GO.assignment(count, grid)]
    got = cta_group_sizes(count, grid)
    assert got.tolist() == want
    assert int(got.sum()) == count
    if count:
        assert got.max() - got.min() <= 1


def test_one_graph_per_cta_below_the_grid():
    assert cta_group_sizes(100, 132).tolist() == [1] * 100
    assert sorted(set(cta_group_sizes(300, 132).tolist())) == [2, 3]


@pytest.mark.parametrize("N,grid", [(256, 132), (256, 64), (300, 132)])
def test_estimator_is_unbiased_on_synthetic_gradients(N, grid):
    rng = np.random.default_rng(N + grid)
    P = 12
    mu = rng.normal(0.0, 1.0, P)
    sigma = rng.uniform(1.0, 3.0, P)
    want = float(np.square(sigma).sum() / np.square(mu).sum())
    U = V = D = 0.0
    for _ in range(40):                     # 40 x 100 draws of a minibatch
        x = mu + sigma * rng.standard_normal((100, N, P))
        for k in range(x.shape[0]):
            u, v, d = grad_noise_terms(GO.measure(x[k], grid))
            U, V, D = U + u, V + v, D + d
    est = grad_noise_estimate(U, V, D, N, 4000)
    assert abs(est["grad_noise_scale"] / want - 1.0) < 0.05, (est, want)
    # |G|^2 and tr Sigma in the units of one graph's gradient, N times its term
    assert abs(est["grad_noise_g2"] / (N * N * np.square(mu).sum()) - 1.0) < 0.05
    assert abs(est["grad_noise_trace"] / (N * N * np.square(sigma).sum()) - 1.0) < 0.05


@pytest.mark.parametrize("C,b", [(64, 4), (132, 2), (10, 7)])
def test_equal_groups_give_mccandlishs_two_batch_estimator(C, b):
    rng = np.random.default_rng(C * b)
    x = rng.normal(0.3, 1.0, (C * b, 9))
    N = C * b
    A, S, Q, n = GO.measure(x, C)
    assert (Q, n) == (C * b * b, N)
    U, V, D = grad_noise_terms([A, S, Q, n])
    # McCandlish's notation: mean gradients of the small batches (the CTA groups) and of the big one (the shard)
    small = x.reshape(b, C, -1).transpose(1, 0, 2).mean(1)            # group c holds rows c, c + C, ...
    g_small_sq = float(np.square(small).sum(1).mean())
    g_big_sq = float(np.square(x.mean(0)).sum())
    g2, tr, bsimple = GO.mccandlish(g_small_sq, g_big_sq, b, N)
    assert np.isclose(U / D, g2, rtol=1e-12) and np.isclose(V / D, tr, rtol=1e-12)
    assert np.isclose(V / U, bsimple, rtol=1e-12)


def test_combining_per_rank_sums_equals_combining_the_pooled_measurements():
    rng = np.random.default_rng(3)
    rows = [GO.measure(rng.normal(0.2, 1.0, (n, 6)), 5) for n in (40, 37, 12, 40, 1, 8)]
    rank0, rank1 = rows[::2], rows[1::2]
    sums = np.add(grad_noise_terms(rank0), grad_noise_terms(rank1))
    pooled = grad_noise_terms(rows)
    assert np.allclose(sums, pooled, rtol=1e-13, atol=0)
    a, b = grad_noise_estimate(*sums, 80, 6), grad_noise_estimate(*pooled, 80, 6)
    assert all(np.isclose(a[k], b[k], rtol=1e-12) for k in a)


def test_no_sample_rows_add_nothing_and_an_empty_update_is_nan():
    assert grad_noise_terms([[0.0, 0.0, 0.0, 0.0]]) == (0.0, 0.0, 0.0)
    est = grad_noise_estimate(0.0, 0.0, 0.0, 256, 0)
    assert np.isnan(est["grad_noise_scale"]) and np.isnan(est["grad_noise_g2"]) and np.isnan(est["grad_noise_trace"])
    assert est["grad_noise_samples"] == 0
    # an unresolved mean gradient is reported as computed
    assert grad_noise_estimate(-1.0, 5.0, 2.0, 4, 1)["grad_noise_scale"] == -5.0
    assert grad_noise_estimate(0.0, 5.0, 2.0, 4, 1)["grad_noise_scale"] == np.inf


def test_update_log_counts_only_steps_that_applied_adam():
    logged = []
    book = UpdateLog(2, 0.5, 0.01, iteration=7, log_fn=lambda tag, v, s: logged.append((tag, v, s)), kl_stop=True,
                     skip_nonfinite=True, grad_noise_batch=16)
    st = np.zeros((5, 22))
    st[:, 3] = st[:, 4] = 16
    st[1, NONFINITE_SLOT] = 1
    st[3, KL_STOP_SLOT] = 1
    st[4, KL_SKIP_SLOT] = 1
    rng = np.random.default_rng(0)
    noise = np.stack([GO.measure(rng.normal(0.1, 1.0, (16, 4)), 6) for _ in range(5)])
    noise[2, 0] = np.nan                                  # not finite: left out
    book.grad_noise(st, [0, 1, 2, 3, 4], noise)
    assert book.noise_samples == 1
    assert np.allclose(book.noise_terms, grad_noise_terms(noise[0]))
    book.epoch(0, st)
    out = book.finish(False)
    want = grad_noise_estimate(*grad_noise_terms(noise[0]), 16, 1)
    assert {k: out[k] for k in want} == want
    tags = [(tag, s) for tag, _, s in logged if tag.startswith("diag/grad_noise")]
    assert sorted(tags) == sorted(("diag/" + k, 7) for k in want)


def test_update_log_without_the_option_reports_nothing():
    book = UpdateLog(1, 0.5, 0.01)
    book.epoch(0, np.zeros((2, 22)))
    assert not any(k.startswith("grad_noise") for k in book.finish(False))


def test_entry_points_without_a_context():
    L = _lib.lib()
    assert L.upb_ppo_grad_noise(None, None, None, 0, None, None, None, None, None, None, None, 1.0, 1.0, None, None,
                                None) == -1
    assert b"ppo_grad_noise" in L.upb_last_error()
    assert L.upb_mlp_ppo_grad_noise(None, None, None, 0, None, None, None, None, None, None, None, 1.0, 1.0, None,
                                    None, None) == -1
    assert b"mlp_ppo_grad_noise" in L.upb_last_error()
