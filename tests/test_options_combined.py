"""CPU: the float64 minibatch with several options at once, and the host models of tests/test_gpu_options_combined.py.

1. The rl-mlp ppo_oracle.mlp_minibatch with the clipped value loss and the KL penalty is the float64 rl-mlp port with
   both options (torch.optim-free backward) to 1e-12.
2. The SGNN ppo_oracle.sgnn_minibatch: with every option off it is oracle/sgnn_numpy.ppo_minibatch bit for bit; with
   the clipped value loss and the KL penalty its gradient is the sum of the one-option gradients less the option-off
   one (the loss is a sum of terms and the backward is linear), to 1e-12.
3. The parameter-group table: every tensor its own lr (neighbours at least 1/32 apart at every update), distinct weight
   decays with some 0, frozen tensors that are not a prefix, val_w2 / val_b2 trained.
4. The host count model and the non-finite position rule on hand-built cases; the element-wise Adam bar takes a step
   at the right lr and refuses one at an lr 1/32 off."""
import numpy as np
import pytest
import torch

import combined_cases as CC
import klpen_oracle as KO
import ppo_oracle as PPO
from drl_urban_planning_b200 import params as PL
from harness import reproducible_states
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON

N = 12


def close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)) <= tol


@pytest.fixture(scope="module")
def case():
    states, actions = reproducible_states(3, N)
    rng = np.random.default_rng(3)
    exps = np.ones(N, np.float32)
    exps[5] = 0.0
    return dict(states=states, actions=actions, adv=rng.normal(0, 1, N).astype(np.float32),
                ret=rng.normal(0, 1, N).astype(np.float32), fixed=rng.normal(-2, 0.3, N).astype(np.float32), exps=exps,
                old_v=rng.normal(0, 1, N).astype(np.float32))


def port_grad(port, case):
    b = MP.stack_states(case["states"])
    col = lambda k: torch.tensor(case[k].reshape(-1, 1), dtype=torch.float64)           # noqa: E731
    out = port.backward(b, torch.tensor(case["actions"]), col("adv"), col("ret"), col("fixed"),
                        torch.tensor(case["exps"] != 0))
    return port.flat_grad(), out


def oracle(minibatch, case, flat, **kw):
    return minibatch(flat, case["states"], case["actions"], case["adv"], case["ret"], case["fixed"], case["exps"], **kw)


# ---- 1. rl-mlp -------------------------------------------------------------------------------------------------------
def test_mlp_value_clip_and_kl_penalty_are_the_port(case):
    """The port snapshots the old parameters as the KL's reference policy and then takes the new ones, so that the KL
    is not 0."""
    flat, old = PL.MLP.default_init(6), PL.MLP.default_init(5)
    coefs = dict(clip_epsilon=0.25, value_pred_coef=0.8, entropy_coef=0.03)
    got = oracle(PPO.mlp_minibatch, case, flat, old_values=case["old_v"], value_clip=0.05,
                 lp_old=KO.mlp_cand_logp64(old, case["states"]), kl_coef=0.3, chunk=5, **coefs)
    port = PPO.MLPPortAgent(old, value_clip=0.05, kl_coef=0.3, dtype=torch.float64, **coefs)
    port.snapshot()
    with torch.no_grad():
        for name, p in MP.params_from_flat(flat, torch.float64).items():
            port.P[name].copy_(p)
    port.old_values = torch.tensor(case["old_v"].reshape(-1, 1), dtype=torch.float64)
    g, (loss, vl, surr, el) = port_grad(port, case)
    assert close(got["grad"], g)
    assert close([got["loss"], got["value_loss"], got["surr_loss"], got["entropy_loss"]], [loss, vl, surr, el])
    assert close(got["kl_loss"], port.last_kl) and got["kl_loss"] > 1e-6
    assert 0 < got["clipped"] < N                       # the clip is active on some graphs


# ---- 2. the SGNN -----------------------------------------------------------------------------------------------------
def test_sgnn_every_option_off_is_the_oracle_bit_for_bit(case):
    coefs = dict(clip_epsilon=0.25, value_pred_coef=0.8, entropy_coef=0.03)
    for kw in ({}, coefs):
        got = oracle(PPO.sgnn_minibatch, case, PL.default_init(6).astype(np.float64), **kw)
        want = oracle(ON.ppo_minibatch, case, PL.default_init(6).astype(np.float64), **kw)
        for k in ("loss", "value_loss", "surr_loss", "entropy_loss", "grad", "value", "log_prob"):
            assert np.array_equal(got[k], want[k]), k


def test_sgnn_value_clip_and_kl_penalty_add_through_the_backward(case):
    flat = PL.default_init(6).astype(np.float64)
    kw = dict(clip_epsilon=0.25, value_pred_coef=0.8, entropy_coef=0.03, old_values=case["old_v"],
              lp_old=KO.cand_logp64(PL.default_init(5), case["states"]))
    off = oracle(PPO.sgnn_minibatch, case, flat, **kw)
    vclip = oracle(PPO.sgnn_minibatch, case, flat, value_clip=0.05, **kw)
    kl = oracle(PPO.sgnn_minibatch, case, flat, kl_coef=0.3, **kw)
    both = oracle(PPO.sgnn_minibatch, case, flat, value_clip=0.05, kl_coef=0.3, **kw)
    assert close(both["grad"], vclip["grad"] + kl["grad"] - off["grad"])
    assert close(both["loss"], vclip["loss"] + kl["loss"] - off["loss"])
    assert both["value_loss_sum"] == vclip["value_loss_sum"] and both["clipped"] == vclip["clipped"] > 0
    assert both["kl_sum"] == kl["kl_sum"] == off["kl_sum"] > 1e-6
    assert (both["surr_sum"], both["ent_sum"]) == (off["surr_sum"], off["ent_sum"])
    assert not close(vclip["grad"], off["grad"], 1e-3) and not close(kl["grad"], off["grad"], 1e-3)


# ---- 3. the table ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_the_table_makes_every_mapping_error_visible(model):
    layout = CC.layout_of(model)
    names = list(layout.slots)
    for it in range(3):
        lr, wd, trained = CC.table(model, it)
        on = lr[trained]
        assert (np.abs(np.diff(on)) >= on[1:] / 32).all() and (np.abs(np.diff(on)) >= on[:-1] / 32).all(), it
        assert len(set(wd[wd > 0].tolist())) == (wd > 0).sum() and (wd[trained] == 0).any(), it
        assert trained[names.index("val_w2")] and trained[names.index("val_b2")], it
        frozen = np.flatnonzero(~trained)
        assert frozen.size and frozen[0] > 0 and all(trained[k - 1] and trained[k + 1] for k in frozen if k + 1 < len(names)
                                                     ), it
        assert (wd == np.float32(wd)).all()
    first, later = ~CC.table(model, 0)[2], ~CC.table(model, 1)[2]
    assert (first & ~later).sum() == 1 and not (later & ~first).any()      # one tensor unfrozen at the second update


# ---- 4. host models --------------------------------------------------------------------------------------------------
def test_count_model():
    seg = np.array([0, 0, 1, 1, 2, 0])
    trained = np.array([True, False, True, True, True, True])
    c = np.array([5, 0, 3, 3, 4, 5])
    assert CC.next_counts(c, trained, seg, [0, 0, 1], False).tolist() == [6, 0, 4, 4, 5, 6]
    assert CC.next_counts(c, trained, seg, [0, 0], False).tolist() == [6, 0, 4, 4, 4, 6]       # the road head is absent
    assert CC.next_counts(c, trained, seg, [1], False).tolist() == [6, 0, 3, 3, 5, 6]
    assert CC.next_counts(c, trained, seg, [0, 1], True).tolist() == c.tolist()               # a skipped step


def test_nonfinite_positions_stay_in_their_episode():
    T = 12
    masks = np.ones(T, np.float32)
    masks[[3, 7]] = 0.0                                    # episodes [0, 3], [4, 7], [8, 11] (open)
    values = np.linspace(-1, 1, T).astype(np.float32)
    rewards = np.linspace(0.5, -0.5, T).astype(np.float32)
    assert CC.episodes(masks) == [(0, 3), (4, 7), (8, 11)]
    adv, ret = ON.estimate_advantages(rewards, masks, values, 0.99, 0.95)
    got = CC.gae_per_episode(rewards, masks, values, 0.99, 0.95)
    assert np.array_equal(got[0], adv.ravel()) and np.array_equal(got[1], ret.ravel())    # finite: the same bits
    assert CC.nonfinite_positions(rewards, masks, values, 0.99, 0.95).size == 0
    for pos, want in [(4, [4]), (6, [4, 5, 6]), (8, [8]), (11, [8, 9, 10, 11]), (0, [0])]:
        r = rewards.copy()
        r[pos] = np.inf
        assert CC.nonfinite_positions(r, masks, values, 0.99, 0.95).tolist() == want, pos
        # the whole-buffer scan carries inf * 0 = NaN across the episode boundary to every earlier sample
        with np.errstate(invalid="ignore"):
            whole = ON.estimate_advantages(r, masks, values, 0.99, 0.95)[0].ravel()
        assert np.flatnonzero(~np.isfinite(whole)).tolist() == list(range(pos + 1))
    ro = CC.small_rollout(4, 400, 1.0, 0.0)
    pos = CC.poison(ro)
    assert ro.masks[pos - 1] == 0 and ro.exps[pos] == 1 and np.isinf(ro.rewards[pos])
    assert CC.nonfinite_positions(ro.rewards, ro.masks, np.zeros(400), 0.99, 0.95).tolist() == [pos]


def test_elementwise_bar_refuses_an_lr_off_by_one_32nd():
    rng = np.random.default_rng(8)
    n = 4096
    p0 = rng.normal(0, 0.1, n).astype(np.float32)
    m0 = (rng.normal(0, 1e-3, n)).astype(np.float32)
    v0 = (rng.random(n) * 1e-6).astype(np.float32)
    g = rng.normal(0, 1e-3, n)
    t = np.full(n, 40.0)
    live = np.ones(n, bool)
    lr, wd = np.full(n, CC.LR_BASE), np.full(n, 2.0 ** -8)
    want = CC.adam_want((p0, m0, v0), g, live, lr, wd, t)
    # the fp32 step: each of p, m rounded once
    p1, m1 = want[0].astype(np.float32), want[1].astype(np.float32)
    assert CC.elem_excess(p1, p0, want[0]).max() <= 1 and CC.elem_excess(m1, m0, want[1]).max() <= 1
    off = CC.adam_want((p0, m0, v0), g, live, lr * (1 + 1 / 32), wd, t)[0].astype(np.float32)
    excess = CC.elem_excess(off, p0, want[0])
    assert (excess > 1).mean() > 0.99 and np.median(excess) > 30
