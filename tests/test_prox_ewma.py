"""CPU: the EWMA proximal policy's validation, its float64 oracle against a direct torch-autograd evaluation of the
decoupled loss, the oracle's reduction to the existing one at theta_prox = theta_old, the age helpers and the fp32 EWMA
replay's rounding."""
import math

import numpy as np
import pytest
import torch

import ppo_oracle as PPO
import prox_oracle as PO
from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.engine import Engine, check_prox_ewma, prox_ewma_age, prox_ewma_for_batch
from drl_urban_planning_b200.ppo import PPOUpdater
from oracle import sgnn_numpy as ON


@pytest.mark.parametrize("bad", [True, False, np.bool_(True), float("nan"), float("inf"), -float("inf"), -1e-9, 1.0,
                                 1.5, 0.99999999, "x"])
def test_refuses_bad_values(bad):
    with pytest.raises((ValueError, TypeError)):
        check_prox_ewma(bad)
    # before any CUDA call: the device argument is never touched
    with pytest.raises((ValueError, TypeError)):
        Engine("cpu", 64, 64, prox_ewma=bad)
    with pytest.raises((ValueError, TypeError)):
        PPOUpdater(PL.default_init(0), 64, 64, "cpu", prox_ewma=bad)


def test_accepts():
    assert check_prox_ewma(None) is None
    assert check_prox_ewma(0) == 0.0
    assert check_prox_ewma(0.99) == 0.99
    assert np.float32(check_prox_ewma(0.9999999)) < 1.0


def test_age_helpers():
    assert prox_ewma_age(0.5) == 1.0
    assert prox_ewma_age(0.9, 256) == pytest.approx(2304.0)
    # 8x the minibatch: the same age in graphs takes a smaller weight
    b = prox_ewma_for_batch(0.9, 256, 2048)
    assert prox_ewma_age(b, 2048) == pytest.approx(prox_ewma_age(0.9, 256))
    assert prox_ewma_for_batch(0.9, 256, 256) == pytest.approx(0.9)


def small(seed=3, count=6):
    states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    adv, ret, exps = synth.make_ppo_targets(seed, count)
    exps[1] = 0.0
    return states, actions, adv, ret, exps


def test_oracle_against_direct_evaluation():
    """The identity w min(r A, clamp(r) A) = min(r A', clamp(r) A') against the decoupled loss evaluated directly in
    float64, graph by graph (oracle/sgnn_numpy's forward and backward with the seed d(-w clip(r) A)/d lp), with the dual
    clip; and the surrogate's r-derivative against torch autograd of the written-out loss."""
    states, actions, adv, ret, exps = small()
    flat = PL.default_init(3).astype(np.float64)
    rng = np.random.default_rng(1)
    prox = flat * (1 + 0.05 * rng.standard_normal(flat.shape))
    lp_p = PO.sgnn_log_probs(prox, states, actions)
    fixed = lp_p + rng.choice([-0.5, 0.0, 0.4], len(states))
    got = PPO.sgnn_minibatch(flat, states, actions, adv, ret, fixed, exps, dual_clip=2.0, prox_flat=prox)

    P = ON._p64(flat)
    B, ind = len(states), np.flatnonzero(exps.reshape(-1) != 0)
    A = adv.reshape(-1).astype(np.float64)
    G = {k: np.zeros_like(v) for k, v in P.items()}
    loss = 0.0
    for i, st in enumerate(states):
        g = ON.unpad(st)
        fw = ON.forward(P, g, action=int(actions[i, int(np.argmax(g.stage[:2]))]), keep=True)
        V = fw["value"]
        loss += 0.5 * (V - ret[i, 0] if ret.ndim == 2 else V - ret[i]) ** 2 / B
        g_lp = g_en = 0.0
        if i in ind:
            w = math.exp(lp_p[i] - fixed[i])
            lp = torch.tensor(fw["log_prob"], dtype=torch.float64, requires_grad=True)
            r = torch.exp(lp - lp_p[i])
            clip1 = torch.min(r * A[i], torch.clamp(r, 0.8, 1.2) * A[i])
            term = -w * (torch.max(clip1, torch.tensor(2.0 * A[i], dtype=torch.float64)) if A[i] < 0 else clip1)
            term.backward()
            loss += term.item() / len(ind) - 0.01 * fw["entropy"] / len(ind)
            g_lp = lp.grad.item() / len(ind)
            g_en = -0.01 / len(ind)
        Gi = ON.backward(P, g, fw, 2.0 * 0.5 * (V - float(np.ravel(ret)[i])) / B, g_lp, g_en)
        for k in G:
            G[k] += Gi[k]
    grad = np.zeros(PL.NUM_PARAMS)
    for sl in PL.SLOTS.values():
        grad[sl.offset:sl.offset + sl.size] = G[sl.name].reshape(-1)
    assert abs(got["loss"] - loss) < 1e-6 * max(1.0, abs(loss))       # the oracle reports its loss in fp32
    assert np.abs(got["grad"] - grad).max() < 1e-10 * max(1.0, np.abs(grad).max())


def test_reduces_to_existing_oracle():
    """theta_prox = theta_old (the parameters the fixed log-probs come from): w = 1, r = the ordinary ratio."""
    states, actions, adv, ret, exps = small(5)
    old = PL.default_init(5).astype(np.float64)
    flat = old * (1 + 0.02 * np.random.default_rng(2).standard_normal(old.shape))
    fixed = PO.sgnn_log_probs(old, states, actions)
    got = PPO.sgnn_minibatch(flat, states, actions, adv, ret, fixed, exps, prox_flat=old)
    want = ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)
    assert got["prox_weight"] == float((exps != 0).sum()) and got["prox_kl"] == 0.0
    assert np.allclose(got["grad"], want["grad"], rtol=1e-12, atol=1e-14)
    assert got["loss"] == pytest.approx(want["loss"], rel=1e-12)
    wl = PPO.sgnn_minibatch(flat, states, actions, adv, ret, fixed, exps)
    assert np.array_equal(got["grad"], wl["grad"])


def test_mlp_oracle_reduces():
    states, actions, adv, ret, exps = small(7)
    old = PL.MLP.default_init(7).astype(np.float64)
    flat = old * (1 + 0.02 * np.random.default_rng(3).standard_normal(old.shape))
    lp_old = PPO.mlp_minibatch(old, states, actions, adv, ret, np.zeros(len(states)), exps)["log_prob"]
    got = PPO.mlp_minibatch(flat, states, actions, adv, ret, lp_old, exps, prox_flat=old)
    assert got["prox_weight"] == float((exps != 0).sum()) and got["prox_kl"] == 0.0
    assert np.isfinite(got["grad"]).all() and np.abs(got["grad"]).max() > 0


def test_ewma_replay_rounding():
    """fma32 rounds once: it matches an exact rational evaluation, halfway cases included."""
    from fractions import Fraction
    rng = np.random.default_rng(0)
    x = rng.standard_normal(2000).astype(np.float32)
    y = rng.standard_normal(2000).astype(np.float32)
    b = np.float32(0.9)
    got = PO.fma32(b, x, y)
    for i in range(0, 2000, 7):
        exact = Fraction(float(b)) * Fraction(float(x[i])) + Fraction(float(y[i]))
        cand = [np.nextafter(got[i], np.float32(-np.inf)), got[i], np.nextafter(got[i], np.float32(np.inf))]
        errs = [abs(Fraction(float(c)) - exact) for c in cand]
        assert errs[1] <= errs[0] and errs[1] <= errs[2], i
    # beta = 0 copies theta, and the replay of a constant theta converges to it
    assert np.array_equal(PO.ewma_replay(x, [y], 0.0), y)
    p = PO.ewma_replay(x, [y] * 400, 0.9)
    assert np.abs(p - y).max() <= 4 * np.abs(np.spacing(y)).max()
    assert math.isclose(prox_ewma_age(0.9), 9.0)
