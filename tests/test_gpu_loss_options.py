"""H100: dual-clip PPO (upb_set_dual_clip) and the Huber value loss (upb_set_huber_delta) on both models.

  * off: a context that never set the options, one that set and cleared them, and one with c = delta = 1e30 give
    bit-identical steps (parameters, moments, counters, the whole gradient / statistics buffer but slots 15, 20 and 21
    for the huge values, launch counts), fused and two-call, with and without value clipping;
  * the per-graph value seeds (the value-head bias gradient of one-graph steps) and slots 0 / 15 / 21 against the fp32
    replay, inside and beyond +-delta, at |e| == delta and with value clipping; the dual bound's effect on the policy
    heads' gradient (zero where active, unchanged where inactive, half on an exact tie) and slot 20;
  * the whole gradient against float64 (SGNN) and the torch port (rl-mlp) where both options bind;
  * fused against two-call at the fused-tail grid sizes, the rl-mlp bit for bit;
  * PPOUpdater / use_b200_update trajectories against a torch-port replay, and the options composed with value_clip,
    value_norm, normalize_advantage, kl_coef and skip_nonfinite."""
import types

import numpy as np
import pytest
import torch

import ppo_oracle as PPO
from cross_path import MLP_GRIDS, SGNN_GRIDS, hlg_case
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.ppo import DUAL_COUNT_SLOT, HUBER_COUNT_SLOT, VCLIP_LOSS_SLOT, PPOUpdater
from harness import (Case, assert_same_state, dev, heads, nan_buffer, per_tensor_rel, rel, reproducible_states,
                     sgnn_agent, t, update_losses)
from oracle import mlp_port as MP
from oracle import torch_port as TP

pytestmark = pytest.mark.gpu
OFFSETS = np.array([0.0, 0.05, -0.07, 0.5, -0.5, 0.35, -0.35, 0.01, 2.0, -2.0, 0.0, 0.12], np.float32)
EXCLUDED = (VCLIP_LOSS_SLOT, DUAL_COUNT_SLOT, HUBER_COUNT_SLOT)


def mixed_case(dev, model, seed=5, count=12, negative=True, reproducible=False):
    """12 graphs of both stages; with `negative`, advantages of both signs, mostly negative.  reproducible: graphs whose
    rl-mlp gradient rows are run-to-run reproducible (harness.reproducible_states), for bit-for-bit comparisons of
    whole minibatches."""
    if reproducible:
        states, actions = reproducible_states(seed, count)
    else:
        states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    c = Case(dev, model, states, actions, seed, zero_exps=(1,))
    if negative:
        c.adv = np.where(np.arange(count)[:, None] % 4 == 0, np.abs(c.adv), -np.abs(c.adv)).astype(np.float32)
        c.dev_args = tuple(t(x, dev) for x in (c.actions, c.adv, c.ret, c.fixed, c.exps))
    return c


def forward(eng, c, params):
    v, lp, _ = eng.forward(c.blob, params, c.dev_args[0])
    torch.cuda.synchronize()
    return v.cpu().numpy(), lp.cpu().numpy()


def with_fixed(c, fixed):
    c.fixed = np.asarray(fixed, np.float32).reshape(-1, 1)
    c.dev_args = tuple(t(x, c.dev) for x in (c.actions, c.adv, c.ret, c.fixed, c.exps))
    return c


def step(eng, c, params, fused, ov=None, sel=None):
    g = nan_buffer(eng)
    fn = eng.ppo_step if fused else eng.ppo_grad
    fn(c.blob, params, *c.step_args(sel), ids=c.ids(sel), out=g, old_values=None if ov is None else t(ov, c.dev))
    if not fused:
        eng.apply(params, g)
    return g


def same_but(e1, p1, g1, e2, p2, g2, skip, what):
    """assert_same_state with the statistics slots `skip` left out of the buffer comparison."""
    torch.cuda.synchronize()
    a, b = g1.cpu().numpy().copy(), g2.cpu().numpy().copy()
    for s in skip:
        a[e1.stat_offset + s] = b[e2.stat_offset + s] = 0.0
    assert np.isfinite(b).all() and np.array_equal(a, b), (what, np.flatnonzero(a != b)[:8])
    assert np.array_equal(p1.cpu().numpy(), p2.cpu().numpy()), what
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2) and s1.tolist() == s2.tolist(), what


@pytest.mark.parametrize("vclip", [None, 0.2])
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_bit_identical(dev, model, fused, vclip):
    c = mixed_case(dev, model, reproducible=True)
    never = c.engine(value_clip=vclip)
    cleared = c.engine(value_clip=vclip, dual_clip=3.0, huber_delta=0.5)
    _lib.check(_lib.lib().upb_set_dual_clip(cleared._ctx, 0.0))
    _lib.check(_lib.lib().upb_set_huber_delta(cleared._ctx, 0.0))
    huge = c.engine(value_clip=vclip, dual_clip=1e30, huber_delta=1e30)
    ps = [t(c.flat, dev).clone() for _ in range(3)]
    ov = None
    if vclip is not None:
        v, _ = forward(never, c, ps[0])
        ov = (v + np.resize(OFFSETS, v.shape)).astype(np.float32)
    for k in range(3):
        before = [e.launches for e in (never, cleared, huge)]
        g0 = step(never, c, ps[0], fused, ov)
        g1 = step(cleared, c, ps[1], fused, ov)
        g2 = step(huge, c, ps[2], fused, ov)
        assert_same_state(never, ps[0], g0, cleared, ps[1], g1, (model, k))
        same_but(never, ps[0], g0, huge, ps[2], g2, EXCLUDED, (model, k))
        assert len({e.launches - b for e, b in zip((never, cleared, huge), before)}) == 1
        s0, s2 = (g.cpu().numpy()[never.stat_offset:] for g in (g0, g2))
        assert not s0[[DUAL_COUNT_SLOT, HUBER_COUNT_SLOT]].any() and s2[HUBER_COUNT_SLOT] == 0
        assert s2[DUAL_COUNT_SLOT] == 0
        if vclip is None:
            assert s0[VCLIP_LOSS_SLOT] == 0 and np.isclose(s2[VCLIP_LOSS_SLOT], s2[0], rtol=1e-6)


@pytest.mark.parametrize("vclip", [None, 0.2])
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_huber_per_graph_seeds_and_slots(dev, model, fused, vclip):
    """One-graph steps (B = 1): the value-head bias gradient, slots 0, 15 and 21 equal the fp32 replay of the kernel's
    own V, R (and V_old) bit for bit; delta puts graphs inside and beyond +-delta, one exactly at |e| == delta."""
    c = mixed_case(dev, model)
    b2 = c.layout.slots["val_b2"].offset
    probe = c.engine()
    p0 = t(c.flat, dev)
    V, _ = forward(probe, c, p0)
    R = c.ret.reshape(-1)
    e = np.abs((V - R).astype(np.float32))
    delta = float(np.sort(e)[len(e) // 2])            # a graph with |e| == fp32(delta) exactly
    assert (e == np.float32(delta)).any() and (e > delta).any() and (e < delta).any()
    eng = c.engine(huber_delta=delta, value_clip=vclip, clip_mode=_lib.CLIP_NEVER)
    ov = None if vclip is None else (V + np.resize(OFFSETS, V.shape)).astype(np.float32)
    for i in range(c.count):
        g = step(eng, c, p0.clone(), fused, ov, sel=[i])
        want, loss, _, lin = PPO.value_seed32(V[i], R[i], delta, c_value=0.5, inv_batch=1.0,
                                              V_old=None if ov is None else ov[i], value_clip=vclip)
        gg = g.cpu().numpy()
        st = gg[eng.stat_offset:]
        assert gg[b2] == want[0], (i, gg[b2], want[0])
        assert st[VCLIP_LOSS_SLOT] == loss[0] and st[HUBER_COUNT_SLOT] == float(lin[0]), (i, st[15], st[21], loss, lin)
        assert st[0] == np.float32(V[i] - R[i]) ** 2, i
    g = step(eng, c, p0.clone(), fused, ov)
    st = g.cpu().numpy()[eng.stat_offset:]
    _, loss, _, lin = PPO.value_seed32(V, R, delta, V_old=ov, value_clip=vclip)
    assert st[HUBER_COUNT_SLOT] == lin.sum() and 0 < lin.sum() < c.count
    assert np.isclose(st[VCLIP_LOSS_SLOT], loss.astype(np.float64).sum(), rtol=1e-5)
    assert np.isclose(eng.read_losses(g)[1], st[VCLIP_LOSS_SLOT] / c.count, rtol=1e-6)


def tie_fixed(logp, A, c, hi):
    """Per graph, a fixed log-prob whose ratio expf(logp - flp) (torch's CUDA exp, the kernel's expf) gives clip1 ==
    fp32(c) A exactly with r > hi, or None."""
    c32 = np.float32(c)
    base = np.float32(logp - np.log(c))
    cand = (base + np.arange(-400, 401, dtype=np.float32) * np.spacing(np.float32(np.abs(base)))).astype(np.float32)
    r = torch.exp(torch.tensor(np.float32(logp) - cand, device="cuda")).cpu().numpy()
    ok = (r > hi) & ((r * np.float32(A)).astype(np.float32) == (c32 * np.float32(A)).astype(np.float32))
    return cand[np.flatnonzero(ok)[0]] if ok.any() else None


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_dual_clip_per_graph(dev, model, fused):
    """entropy_coef = 0, one-graph steps with A < 0: the policy head's gradient is exactly zero where the bound is
    active, equal to the option-off step where it is not, and half of it on an exact tie; slot 20 is exact."""
    C = 2.0
    c = mixed_case(dev, model)
    probe = c.engine()
    p0 = t(c.flat, dev)
    _, logp = forward(probe, c, p0)
    A = c.adv.reshape(-1)
    # ratios: far beyond c (active), between hi and c (inactive), and on the tie
    fixed = np.empty(c.count, np.float32)
    kinds = []
    for i in range(c.count):
        kind = ("active", "inactive", "tie")[i % 3]
        if kind == "tie" and A[i] < 0:
            f = tie_fixed(logp[i], A[i], C, 1.2)
            if f is not None:
                fixed[i] = f
                kinds.append(kind)
                continue
            kind = "active"
        fixed[i] = np.float32(logp[i] - (np.log(3 * C) if kind == "active" else np.log(1.5)))
        kinds.append(kind)
    with_fixed(c, fixed)
    assert kinds.count("tie") >= 2
    off = c.engine(entropy_coef=0.0, clip_mode=_lib.CLIP_NEVER)
    on = c.engine(entropy_coef=0.0, clip_mode=_lib.CLIP_NEVER, dual_clip=C)
    hd = heads(c.layout)
    n_active = 0
    for i in range(c.count):
        if c.exps[i] == 0:
            continue
        g0 = step(off, c, p0.clone(), fused, sel=[i]).cpu().numpy()
        g1 = step(on, c, p0.clone(), fused, sel=[i]).cpu().numpy()
        h = hd[int(c.stage[i])]
        active = A[i] < 0 and kinds[i] == "active"
        n_active += active
        assert g1[on.stat_offset + DUAL_COUNT_SLOT] == float(active), i
        assert g0[h].any() or A[i] > 0, i       # a positive A above the clip range has no policy gradient
        if active:
            assert not g1[h].any(), i
        elif A[i] < 0 and kinds[i] == "tie":
            assert np.array_equal(g1[h], np.float32(0.5) * g0[h]), (i, np.abs(g1[h] - 0.5 * g0[h]).max())
        else:
            assert np.array_equal(g1[h], g0[h]), i
        # the value head never sees the policy's bound
        v = slice(c.layout.slots["val_w0"].offset, c.layout.num_params)
        assert np.array_equal(g1[v], g0[v]), i
    assert n_active >= 2
    g = step(on, c, p0.clone(), fused).cpu().numpy()
    want = sum(1 for i in range(c.count) if c.exps[i] != 0 and A[i] < 0 and kinds[i] == "active")
    assert g[on.stat_offset + DUAL_COUNT_SLOT] == want


def binding_case(dev, model):
    """A mixed minibatch where both options bind on several graphs: ratios spread around c on both signs of A, delta
    the median |V - R|."""
    c = mixed_case(dev, model)
    probe = c.engine()
    V, logp = forward(probe, c, t(c.flat, dev))
    spread = np.resize(np.array([1.2, -0.3, 0.9, 0.2, 1.6, -0.1], np.float32), c.count)
    with_fixed(c, (logp - spread).astype(np.float32))
    delta = float(np.median(np.abs(V - c.ret.reshape(-1))))
    return c, 1.5, delta


def test_sgnn_gradient_against_the_float64_oracle(dev):
    c, C, delta = binding_case(dev, "sgnn")
    eng = c.engine(dual_clip=C, huber_delta=delta)
    p = t(c.flat, dev).clone()
    g = eng.ppo_grad(c.blob, p, *c.step_args())
    r = PPO.sgnn_minibatch(c.flat.astype(np.float64), c.states, c.actions, c.adv, c.ret, c.fixed, c.exps,
                           dual_clip=float(np.float32(C)), huber_delta=float(np.float32(delta)))
    worst, where = per_tensor_rel(g.cpu().numpy()[:PL.NUM_PARAMS], r["grad"])
    assert worst < 1e-4, (worst, where)
    assert np.allclose(eng.read_losses(g), [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]],
                       rtol=1e-4, atol=1e-5)
    st = g.cpu().numpy()[eng.stat_offset:]
    assert st[DUAL_COUNT_SLOT] == r["dual"] >= 2 and st[HUBER_COUNT_SLOT] == r["linear"] >= 2
    assert np.isclose(st[VCLIP_LOSS_SLOT], r["value_loss_sum"], rtol=1e-5)


def test_mlp_trajectory_against_the_torch_port(dev):
    """Three fused steps (the first clipped by the reference's rule) against MLPPortAgent with both options."""
    c, C, delta = binding_case(dev, "mlp")
    eng = c.engine(dual_clip=C, huber_delta=delta)
    p = t(c.flat, dev).clone()
    agent = PPO.MLPPortAgent(c.flat, dual_clip=C, huber_delta=delta)
    b = MP.stack_states(c.states)
    ind = torch.tensor(c.exps).nonzero(as_tuple=False).squeeze(1)
    for k in range(3):
        want = agent.step(b, torch.tensor(c.actions), torch.tensor(c.adv), torch.tensor(c.ret), torch.tensor(c.fixed),
                          ind)
        g = step(eng, c, p, True)
        torch.cuda.synchronize()
        assert np.allclose(eng.read_losses(g), want, rtol=1e-4, atol=1e-5), k
        assert rel(p.cpu().numpy(), agent.flat()) < 2e-5, k
        if k == 0:
            st = g.cpu().numpy()[eng.stat_offset:]
            assert st[DUAL_COUNT_SLOT] >= 2 and st[HUBER_COUNT_SLOT] >= 2


@pytest.mark.parametrize("grid", MLP_GRIDS)
def test_mlp_fused_bit_identical(dev, grid):
    states, actions = reproducible_states(11, 40)
    c = Case(dev, "mlp", states, actions, 11)
    kw = dict(grid_limit=grid, dual_clip=1.2, huber_delta=0.3)
    e1, e2 = c.engine(**kw), c.engine(**kw)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for k in range(3):
        g1 = step(e1, c, p1, False)
        g2 = step(e2, c, p2, True)
        assert_same_state(e1, p1, g1, e2, p2, g2, (grid, k))
    assert g2.cpu().numpy()[e2.stat_offset + HUBER_COUNT_SLOT] > 0


@pytest.mark.parametrize("grid", SGNN_GRIDS)
def test_sgnn_fused_against_two_call(dev, grid):
    c = hlg_case(dev, 3)
    kw = dict(grid_limit=grid, dual_clip=1.2, huber_delta=0.3)
    e1, e2 = c.engine(**kw), c.engine(**kw)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for k in range(3):
        g1 = step(e1, c, p1, False)
        before = e2.launches
        g2 = step(e2, c, p2, True)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (k > 0)
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (k, worst, where)
        s1, s2 = (g.cpu().numpy()[e1.stat_offset:] for g in (g1, g2))
        assert np.isclose(s1[VCLIP_LOSS_SLOT], s2[VCLIP_LOSS_SLOT], rtol=1e-5)
        if k == 0:
            assert s1[HUBER_COUNT_SLOT] == s2[HUBER_COUNT_SLOT] > 0
            assert s1[DUAL_COUNT_SLOT] == s2[DUAL_COUNT_SLOT]
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, k


# ---- whole updates ---------------------------------------------------------------------------------------------------
def rollout(seed, T):
    states, actions = synth.make_states(seed, "small", T, stages=[int(i % 3 == 1) for i in range(T)])
    rng = np.random.default_rng(seed)
    rewards = rng.normal(scale=2.0, size=T).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[[9, 19, 29, T - 1]] = 0.0
    exps = np.ones(T, np.float32)
    exps[[2, 17]] = 0.0
    return states, actions, rewards, masks, exps


def port_replay(model, flat, ro, B, epochs, np_seed, gamma, tau, dual_clip=None, huber_delta=None, value_clip=None,
                normalize=False):
    """The reference's update_params with the options, in the torch ports, on the same permutations."""
    states, actions, rewards, masks, exps = ro
    mlp = model == "mlp"
    stack = MP.stack_states if mlp else TP.stack_states
    agent = (PPO.MLPPortAgent if mlp else PPO.PortAgent)(flat, dual_clip=dual_clip, huber_delta=huber_delta,
                                                         value_clip=value_clip, lr=LR)
    b_all = stack(states)
    act = torch.tensor(actions)
    with torch.no_grad():
        P = agent.P if mlp else agent.params()
        values = (MP.value if mlp else TP.value)(P, b_all).reshape(-1, 1).float()
        fixed, _ = (MP.log_prob_entropy if mlp else TP.log_prob_entropy)(P, b_all, act)
    adv, ret = TP.estimate_advantages(torch.tensor(rewards), torch.tensor(masks), values, gamma, tau)
    T = len(states)
    e_t = torch.tensor(exps)
    np.random.seed(np_seed)
    order, losses = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(T // B):
            idx = order[i * B:(i + 1) * B]
            ind = e_t[idx].nonzero(as_tuple=False).squeeze(1)
            a = adv[idx].clone()
            if normalize and ind.numel() > 1:
                a = (a - a[ind].mean()) / (a[ind].std() + 1e-8)
            agent.old_values = values[idx]
            losses.append(agent.step(stack([states[j] for j in idx]), act[idx], a, ret[idx], fixed[idx], ind))
    return np.array(losses), agent.flat()


def run_updater(dev, model, flat, ro, B, epochs, gamma, tau, **kw):
    up = PPOUpdater(flat, 128, 512, dev, lr=LR, gamma=gamma, tau=tau, opt_num_epochs=epochs, mini_batch_size=B,
                    model=model, **kw)
    logged = []
    np.random.seed(7)
    out = up.update_params(*ro, log_fn=lambda tg, v, s: logged.append((tg, v, s)))
    return up, up.flat_params(), logged, out


# a learning rate and a bound at which the ratios of later minibatches pass c on some graphs
LR, DUAL = 2e-3, 1.001
OPTION_SETS = {"dual": dict(dual_clip=DUAL), "huber": dict(huber_delta=0.5),
               "both_vclip_norm": dict(dual_clip=DUAL, huber_delta=0.5, value_clip=0.2, normalize_advantage=True)}


@pytest.mark.parametrize("name", sorted(OPTION_SETS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_updater_against_the_port(dev, model, name):
    T, B, epochs, gamma, tau = 40, 16, 2, 0.99, 0.95
    ro = rollout(21, T)
    flat = PL.MLP.default_init(21) if model == "mlp" else PL.default_init(21)
    kw = OPTION_SETS[name]
    want_losses, want_flat = port_replay(model, flat, ro, B, epochs, 7, gamma, tau, kw.get("dual_clip"),
                                         kw.get("huber_delta"), kw.get("value_clip"),
                                         kw.get("normalize_advantage", False))
    _, got, logged, out = run_updater(dev, model, flat, ro, B, epochs, gamma, tau, diagnostics=True, **kw)
    losses = update_losses(logged)
    assert losses.shape == want_losses.shape
    assert np.allclose(losses, want_losses, rtol=2e-4, atol=2e-5), np.abs(losses - want_losses).max()
    assert rel(got, want_flat) < 5e-5
    tags = {tg for tg, _, _ in logged}
    for opt, tag in (("dual_clip", "dual_clip_fraction"), ("huber_delta", "huber_fraction")):
        assert (("diag/" + tag) in tags) == (opt in kw) and (("total_" + tag) in out) == (opt in kw)
        if opt in kw:
            per = [v for tg, v, _ in logged if tg == "diag/" + tag]
            assert np.isclose(out["total_" + tag], np.mean(per)) and 0 < np.mean(per) < 1, (tag, per)
    # the options change the trajectory
    _, plain, _, _ = run_updater(dev, model, flat, ro, B, epochs, gamma, tau,
                                 **{k: v for k, v in kw.items() if k not in ("dual_clip", "huber_delta")})
    assert rel(plain, want_flat) > 1e-5


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_updater_composed_with_the_other_options(dev, model):
    """With value_norm, kl_coef, skip_nonfinite, value_clip and normalize_advantage: huge c and delta reproduce the
    update without the options bit for bit (the composition adds nothing when the options never bind), and finite ones
    bind and change it; the logged value loss is slot 15 and the fractions are logged."""
    T, B, epochs, gamma, tau = 40, 16, 2, 0.99, 0.95
    ro = rollout(23, T)
    flat = PL.MLP.default_init(23) if model == "mlp" else PL.default_init(23)
    base = dict(value_norm=True, kl_coef=0.2, skip_nonfinite=True, value_clip=0.2, normalize_advantage=True,
                clip_mode=_lib.CLIP_NEVER, diagnostics=True)
    _, p_off, log_off, out_off = run_updater(dev, model, flat, ro, B, epochs, gamma, tau, **base)
    _, p_huge, log_huge, out_huge = run_updater(dev, model, flat, ro, B, epochs, gamma, tau, dual_clip=1e30,
                                                huber_delta=1e30, **base)
    assert np.array_equal(p_off, p_huge) or (model == "mlp" and rel(p_huge, p_off) < 1e-6)
    assert np.allclose(update_losses(log_huge), update_losses(log_off), rtol=1e-6, atol=1e-7)
    assert out_huge["total_huber_fraction"] == 0 and out_huge["total_dual_clip_fraction"] == 0
    _, p_on, log_on, out_on = run_updater(dev, model, flat, ro, B, epochs, gamma, tau, dual_clip=DUAL,
                                          huber_delta=0.05, **base)
    assert np.isfinite(p_on).all() and rel(p_on, p_off) > 1e-5
    assert 0 < out_on["total_huber_fraction"] <= 1 and 0 < out_on["total_dual_clip_fraction"] < 1
    assert out_on["nonfinite_skips"] == 0 and "kl_coef" in out_on


def test_use_b200_update_with_both_options(dev):
    from drl_urban_planning_b200.agent import use_b200_update
    T, B = 40, 16
    ro = rollout(21, T)
    flat = PL.default_init(21)
    want_losses, want_flat = port_replay("sgnn", flat, ro, B, 2, 7, 0.99, 0.95, DUAL, 0.5, 0.2, True)
    logged = []
    ag = sgnn_agent(dev, 128, 512, flat, logged, num_optim_epoch=2, mini_batch_size=B, lr=LR)
    ctl = use_b200_update(ag, dual_clip=DUAL, huber_delta=0.5, value_clip=0.2, normalize_advantage=True,
                          diagnostics=True)
    assert ctl.updater.engine.dual_clip == DUAL and ctl.updater.engine.huber_delta == 0.5
    batch = types.SimpleNamespace(states=ro[0], actions=ro[1], rewards=ro[2], masks=ro[3], exps=ro[4])
    np.random.seed(7)
    ag.update_params(batch, 0)
    assert np.allclose(update_losses(logged), want_losses, rtol=2e-4, atol=2e-5)
    assert rel(ag.actor_critic_net.flat_parameters(), want_flat) < 5e-5
    tags = {tg for tg, _, _ in logged}
    assert {"diag/dual_clip_fraction", "diag/huber_fraction", "diag/total_huber_fraction"} <= tags
