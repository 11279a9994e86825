"""H100: the EWMA proximal policy (PPO-EWMA, upb_set_prox_ewma) on both models.

  * anchor: with theta_prox at the step's starting parameters and the fixed log-probs from the forward there, one step
    is bit-identical to the option off (parameters, moments, counters, the whole buffer but slots 23 and 24), fused and
    two-call, at the fused tails' grid sizes; slot 23 is then #ind and slot 24 zero, and both are zero while off;
  * the whole gradient and slots 23 / 24 against the float64 oracle with theta_prox != theta, where w and the clip
    both matter, alone and with dual_clip, normalize_advantage, value_clip and kl_coef;
  * the EWMA after several applied steps against its fp32 replay, with absent heads, frozen tensors and AMSGrad;
  * target_kl stops and the steps after them, and skip_nonfinite skips, leave theta_prox bit-unchanged;
  * PPOUpdater / use_b200_update: an update against its replay, and checkpoints with and without "prox_params"."""
import numpy as np
import pytest
import torch

import ppo_oracle as PPO
import prox_oracle as PO
from cross_path import MLP_GRIDS, SGNN_GRIDS
from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.agent import use_b200_update
from drl_urban_planning_b200.packing import infer_caps
from drl_urban_planning_b200.ppo import PROX_KL_SLOT, PROX_WEIGHT_SLOT, PPOUpdater
from harness import Case, nan_buffer, rel, reproducible_states, sgnn_agent, t

pytestmark = pytest.mark.gpu


def case(d, model, seed=3, count=12):
    states, actions = reproducible_states(seed, count)
    return Case(d, model, states, actions, seed, zero_exps=(1,))


def set_fixed(c, fixed):
    c.fixed = np.asarray(fixed, np.float32).reshape(-1, 1)
    c.dev_args = tuple(t(x, c.dev) for x in (c.actions, c.adv, c.ret, c.fixed, c.exps))


def log_probs(eng, c, params):
    _, lp, _ = eng.forward(c.blob, params, c.dev_args[0])
    torch.cuda.synchronize()
    return lp.cpu().numpy()


def step(eng, c, params, fused, sel=None, **kw):
    g = nan_buffer(eng)
    if fused:
        eng.ppo_step(c.blob, params, *c.step_args(sel), ids=c.ids(sel), out=g, **kw)
    else:
        eng.ppo_grad(c.blob, params, *c.step_args(sel), ids=c.ids(sel), out=g, **kw)
        eng.apply(params, g)
    return g


def stats(eng, g):
    torch.cuda.synchronize()
    return g.cpu().numpy()[eng.stat_offset:eng.stat_offset + _lib.UPB_STAT_COUNT].astype(np.float64)


def launches(eng):
    return int(_lib.lib().upb_launch_count(eng._ctx))


def perturbed(flat, seed, scale):
    rng = np.random.default_rng(seed)
    return (flat * (1.0 + scale * rng.standard_normal(flat.shape))).astype(np.float32)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("model,grid", [("sgnn", g) for g in SGNN_GRIDS] + [("mlp", g) for g in MLP_GRIDS])
def test_anchor_bit_identical(model, grid, fused):
    d = torch.device("cuda", 0)
    c = case(d, model)
    off = c.engine(grid_limit=grid)
    on = c.engine(grid_limit=grid, prox_ewma=0.9)
    p_off, p_on = t(c.flat, d).clone(), t(c.flat, d).clone()
    set_fixed(c, log_probs(off, c, p_off))
    on.init_prox_params(p_on)
    l_off, l_on = launches(off), launches(on)
    g_off = step(off, c, p_off, fused)
    g_on = step(on, c, p_on, fused)
    torch.cuda.synchronize()
    a, b = g_off.cpu().numpy().copy(), g_on.cpu().numpy().copy()
    so = off.stat_offset
    n_ind = float((c.exps != 0).sum())
    assert a[so + PROX_WEIGHT_SLOT] == 0.0 and a[so + PROX_KL_SLOT] == 0.0
    assert b[so + PROX_WEIGHT_SLOT] == n_ind and b[so + PROX_KL_SLOT] == 0.0, b[so + 20:so + 28]
    a[so + PROX_WEIGHT_SLOT] = b[so + PROX_WEIGHT_SLOT] = 0.0
    assert np.isfinite(b).all() and np.array_equal(a, b), np.flatnonzero(a != b)[:8]
    assert np.array_equal(p_off.cpu().numpy(), p_on.cpu().numpy())
    m1, v1, s1 = off.get_opt_state()
    m2, v2, s2 = on.get_opt_state()
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2) and s1.tolist() == s2.tolist()
    # one proximal forward more than the option-off step
    assert launches(on) - l_on == launches(off) - l_off + 1


def oracle(model, flat, prox, c, **kw):
    args = (c.states, c.actions, c.adv, c.ret, c.fixed, c.exps)
    return (PPO.mlp_minibatch if model == "mlp" else PPO.sgnn_minibatch)(flat, *args, prox_flat=prox, **kw)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_gradient_against_float64(model):
    d = torch.device("cuda", 0)
    c = case(d, model, seed=11)
    eng = c.engine(prox_ewma=0.5, clip_epsilon=0.003)        # a narrow range, so that the clip binds on some graphs
    params = t(c.flat, d)
    prox = perturbed(c.flat, 1, 0.08)
    # behaviour log-probs far enough from both so that w ranges widely and the clip binds on some graphs
    lp_prox = log_probs(eng, c, t(prox, d))
    rng = np.random.default_rng(4)
    set_fixed(c, lp_prox.reshape(-1) + rng.choice([-0.6, -0.2, 0.0, 0.3, 0.7], c.count))
    eng.set_prox_params(prox)
    g = nan_buffer(eng)
    eng.ppo_grad(c.blob, params, *c.step_args(), out=g)
    st = stats(eng, g)
    ref = oracle(model, c.flat.astype(np.float64), prox.astype(np.float64), c, clip_epsilon=0.003)
    w = np.exp(ref["prox_log_prob"] - c.fixed.reshape(-1))
    assert w.max() > 1.5 and w.min() < 0.7, w
    got = g.cpu().numpy()[:eng.num_params]
    assert rel(got, ref["grad"]) < 2e-4
    assert abs(st[PROX_WEIGHT_SLOT] - ref["prox_weight"]) < 1e-4 * ref["prox_weight"]
    assert abs(st[PROX_KL_SLOT] - ref["prox_kl"]) < 1e-3 * ref["prox_kl"] + 1e-5
    # the clip binds on some graphs and not on others
    lp = log_probs(eng, c, params)
    r = np.exp(lp.reshape(-1) - ref["prox_log_prob"])[c.exps.reshape(-1) != 0]
    out = (r < 0.997) | (r > 1.003)
    assert out.any() and not out.all(), r


def test_composition_sgnn():
    """dual_clip, value_clip, normalize_advantage-style advantages and kl_coef together against the oracle (the KL
    penalty's gradient is checked as the difference of two launches: w does not touch it)."""
    d = torch.device("cuda", 0)
    c = case(d, "sgnn", seed=13)
    a = c.adv.reshape(-1)
    c.adv = ((a - a.mean()) / (a.std() + 1e-8)).astype(np.float32).reshape(c.adv.shape)      # normalised advantages
    kw = dict(dual_clip=2.0, value_clip=0.2)
    eng = c.engine(prox_ewma=0.5, **kw)
    params = t(c.flat, d)
    prox = perturbed(c.flat, 2, 0.08)
    lp_prox = log_probs(eng, c, t(prox, d))
    set_fixed(c, lp_prox.reshape(-1) + np.random.default_rng(5).choice([-0.5, 0.0, 0.4], c.count))
    v_old, _ = eng.forward(c.blob, t(perturbed(c.flat, 3, 0.05), d), c.dev_args[0])[:2]
    eng.set_prox_params(prox)
    g = nan_buffer(eng)
    eng.ppo_grad(c.blob, params, *c.step_args(), out=g, old_values=v_old)
    ref = oracle("sgnn", c.flat.astype(np.float64), prox.astype(np.float64), c, dual_clip=2.0,
                 old_values=v_old.cpu().numpy().astype(np.float64), value_clip=0.2)
    assert rel(g.cpu().numpy()[:eng.num_params], ref["grad"]) < 2e-4
    # the KL penalty adds the same gradient with and without the option
    _, _, _, cand = eng.forward(c.blob, params, c.dev_args[0], cand_log_probs=True)
    grads = []
    for prox_on in (None, 0.5):
        e2 = c.engine(prox_ewma=prox_on, **kw)
        if prox_on is not None:
            e2.set_prox_params(prox)
        pair = []
        for k in (None, 0.3):
            e2.set_kl_coef(k or 0.0)
            g2 = nan_buffer(e2)
            e2.ppo_grad(c.blob, params, *c.step_args(), out=g2, old_values=v_old,
                        old_cand_log_probs=cand if k else None)
            torch.cuda.synchronize()
            pair.append(g2.cpu().numpy()[:e2.num_params].astype(np.float64))
        grads.append(pair[1] - pair[0])
    assert rel(grads[1], grads[0]) < 1e-3


def replay_check(c, eng, params, beta, steps, sels, fused):
    prox0 = perturbed(c.flat, 7, 0.05)
    eng.set_prox_params(prox0)
    traj = []
    for k in range(steps):
        step(eng, c, params, fused, sel=sels[k % len(sels)])
        torch.cuda.synchronize()
        traj.append(params.cpu().numpy().copy())
    want = PO.ewma_replay(prox0, traj, beta)
    got = eng.get_prox_params()
    assert np.array_equal(got, want), (np.flatnonzero(got != want)[:8], got[got != want][:4], want[got != want][:4])


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_ewma_replay(model, fused):
    d = torch.device("cuda", 0)
    c = case(d, model, seed=17)
    eng = c.engine(prox_ewma=0.8)
    params = t(c.flat, d).clone()
    set_fixed(c, log_probs(eng, c, params))
    lu = [i for i in range(c.count) if c.stage[i] == 0]
    rd = [i for i in range(c.count) if c.stage[i] != 0]
    assert lu and rd
    replay_check(c, eng, params, 0.8, 5, [None, lu, rd], fused)       # the absent head still averages


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_ewma_param_groups_amsgrad(model):
    d = torch.device("cuda", 0)
    c = case(d, model, seed=19)
    eng = c.engine(prox_ewma=0.6)
    names = list(eng.layout.slots)
    n = len(names)
    eng.set_param_groups([4e-4] * n, [0.01] * n, [i % 3 != 0 for i in range(n)],
                         adam=[(0.9, 0.999, 1e-5, True, True)] * n)
    params = t(c.flat, d).clone()
    set_fixed(c, log_probs(eng, c, params))
    replay_check(c, eng, params, 0.6, 4, [None], True)
    replay_check(c, eng, params, 0.6, 2, [None], False)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_skipped_steps_leave_prox(model, fused):
    d = torch.device("cuda", 0)
    c = case(d, model, seed=23)
    eng = c.engine(prox_ewma=0.9, target_kl=1e-6, skip_nonfinite=True)
    params = t(c.flat, d).clone()
    prox0 = perturbed(c.flat, 8, 0.2)                 # far from the step: the KL passes the limit at once
    set_fixed(c, log_probs(eng, c, t(prox0, d)) - 1.0)
    eng.set_prox_params(prox0)
    g = step(eng, c, params, fused)
    st = stats(eng, g)
    assert st[13] == 1.0
    assert np.array_equal(eng.get_prox_params(), prox0)
    g = step(eng, c, params, fused)                   # skipped after the stop: the proximal forward does nothing
    st = stats(eng, g)
    assert st[14] == 1.0 and st[PROX_WEIGHT_SLOT] == 0.0
    assert np.array_equal(eng.get_prox_params(), prox0)
    assert np.array_equal(params.cpu().numpy(), c.flat)
    # a non-finite step: skipped by the guard, theta_prox unchanged
    eng.reset_kl_stop()
    eng2 = c.engine(prox_ewma=0.9, skip_nonfinite=True)
    eng2.set_prox_params(prox0)
    bad = c.adv.copy()
    bad[0] = np.inf
    c.dev_args = (c.dev_args[0], t(bad, d)) + c.dev_args[2:]
    g = step(eng2, c, params, fused)
    st = stats(eng2, g)
    assert st[19] == 1.0
    assert np.array_equal(eng2.get_prox_params(), prox0)


def test_refusals():
    d = torch.device("cuda", 0)
    c = case(d, "sgnn")
    eng = c.engine(prox_ewma=0.5)
    params = t(c.flat, d).clone()
    with pytest.raises(_lib.UpbError):
        step(eng, c, params, True)
    with pytest.raises(_lib.UpbError):
        eng.get_prox_params()
    with pytest.raises(_lib.UpbError):
        _lib.check(_lib.lib().upb_set_prox_ewma(eng._ctx, 1, 1.0), "upb_set_prox_ewma")


def test_updater_replay_and_checkpoint():
    """PPOUpdater updates of one step each: theta_prox starts from the live parameters at the first update and ends as
    the replay of the step's parameters; a restored theta_prox resumes the same trajectory, and an updater without one
    starts it from its parameters."""
    d = torch.device("cuda", 0)
    states, actions = reproducible_states(29, 16)
    rng = np.random.default_rng(0)
    rewards = rng.normal(size=16).astype(np.float32)
    masks = np.ones(16, np.float32)
    masks[-1] = 0
    flat = PL.default_init(29)
    n_cap, e_cap = infer_caps(states)
    kw = dict(n_cap=n_cap, e_cap=e_cap, device=d, opt_num_epochs=1, mini_batch_size=16, clip_mode=_lib.CLIP_NEVER,
              diagnostics=True)
    up = PPOUpdater(flat, prox_ewma=0.75, **kw)
    out = up.update_params(states, actions, rewards, masks)
    assert "total_prox_weight" in out and "total_prox_kl" in out
    # first update: theta_prox = theta_0, one applied step -> fmaf(beta, theta_0 - theta_1, theta_1)
    want = PO.ewma_replay(flat, [up.flat_params()], 0.75)
    assert np.array_equal(up.engine.get_prox_params(), want)
    assert out["total_prox_weight"] == 1.0 and out["total_prox_kl"] == 0.0
    # a checkpoint round trip resumes the same trajectory; one without prox_params restarts from the parameters
    saved = up.engine.get_prox_params()
    twin = PPOUpdater(up.flat_params(), prox_ewma=0.75, **kw)
    m, v, s = up.engine.get_opt_state()
    twin.engine.set_opt_state(m, v, s)
    twin.engine.set_prox_params(saved)
    twin._prox_ready = True
    o1 = up.update_params(states, actions, rewards, masks)
    o2 = twin.update_params(states, actions, rewards, masks)
    assert np.array_equal(up.flat_params(), twin.flat_params())
    assert np.array_equal(up.engine.get_prox_params(), twin.engine.get_prox_params())
    assert o1["total_prox_weight"] == o2["total_prox_weight"] and o1["total_prox_weight"] != 1.0
    fresh = PPOUpdater(up.flat_params(), prox_ewma=0.75, **kw)
    p0 = fresh.flat_params()
    fresh.update_params(states, actions, rewards, masks)
    assert np.array_equal(fresh.engine.get_prox_params(), PO.ewma_replay(p0, [fresh.flat_params()], 0.75))


def test_use_b200_update_checkpoint_state():
    d = torch.device("cuda", 0)
    states, actions = reproducible_states(31, 16)
    logged = []
    ag = sgnn_agent(d, *infer_caps(states), PL.default_init(31), logged)
    ctl = use_b200_update(ag, prox_ewma=0.5, diagnostics=True)
    batch = type("B", (), dict(states=states, actions=actions, rewards=np.ones(16, np.float32),
                                masks=np.r_[np.ones(15), 0].astype(np.float32), exps=np.ones(16, np.float32)))
    ag.update_params(batch, 0)
    st = ctl.optimizer_state()
    assert "prox_params" in st and st["prox_params"].shape == (PL.NUM_PARAMS,)
    tags = {tag for tag, _, _ in logged}
    assert {"diag/prox_weight", "diag/prox_kl", "diag/total_prox_weight", "diag/total_prox_kl"} <= tags
    st2 = dict(st)
    del st2["prox_params"]
    ctl.load_optimizer_state(st2)
    assert not ctl.updater._prox_ready
    ctl.load_optimizer_state(st)
    assert ctl.updater._prox_ready and np.array_equal(ctl.updater.engine.get_prox_params(), st["prox_params"])
