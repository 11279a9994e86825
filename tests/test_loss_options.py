"""CPU: dual-clip PPO and the Huber value loss -- the kernels' fp32 seed replays against torch fp32 autograd on scalar
grids (exact ties of clip1 with c A, |e| == delta, value clipping), the float64 minibatch oracle against the torch port's
autograd, the argument checks before any CUDA call, and the update's host bookkeeping of statistics slots 15, 20, 21."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import ppo_oracle as PPO
from drl_urban_planning_b200 import _lib, synth
from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.diagnostics import NAMES
from drl_urban_planning_b200.engine import Engine, check_dual_clip, check_huber_delta
from drl_urban_planning_b200.ppo import DUAL_COUNT_SLOT, HUBER_COUNT_SLOT, VCLIP_LOSS_SLOT, PPOUpdater, UpdateLog
from harness import Cfg, rel
from oracle import torch_port as TP

LO_, HI_ = np.float32(0.8), np.float32(1.2)          # clip_range(0.2)
BAD_DUAL = [1.0, 0.5, 0.0, -3.0, 1.00000001, float("nan"), float("inf"), -float("inf"), 1e39, True, np.bool_(True)]
BAD_HUBER = [0.0, -0.5, 1e-50, float("nan"), float("inf"), -float("inf"), 1e39, True, np.bool_(False)]


def torch_dual(r, A, c):
    """Tianshou's surrogate per element in fp32 with r a leaf: (surr, d surr / d log r = grad_r * r)."""
    rt = torch.tensor(np.asarray(r, np.float32), requires_grad=True)
    s = PPO.surrogate(rt, torch.tensor(np.asarray(A, np.float32)), 0.2, c, reduce=False)
    s.sum().backward()
    return s.detach().numpy(), (rt.grad * rt.detach()).numpy()


def dual_grid(c):
    """Ratios and advantages over every branch: inside, outside the clip range, the dual bound active, inactive and on
    an exact tie (r == fp32(c) with r > hi: clip1 = r A == fp32(c) A)."""
    c32 = np.float32(c)
    rs = np.array([0.5, 0.8, 1.0, 1.1, 1.2, 1.5, c32, np.nextafter(c32, np.float32(0)), np.nextafter(c32, np.float32(9)),
                   2 * c32, 10.0], np.float32)
    As = np.array([-2.0, -0.7, -1e-3, 0.0, 0.3, 1.5], np.float32)
    r, A = np.meshgrid(rs, As)
    return r.ravel(), A.ravel()


@pytest.mark.parametrize("c", [1.5, 3.0, 2.7182817, 10.0])
def test_dual_seed_against_autograd(c):
    r, A = dual_grid(c)
    s_ref, g_ref = torch_dual(r, A, c)
    glp, surr, active = PPO.dual_seed32(r, A, LO_, HI_, c)
    assert np.array_equal(surr, s_ref)
    assert np.array_equal(glp, g_ref), np.flatnonzero(glp != g_ref)
    cA = (np.float32(c) * A).astype(np.float32)
    clip1 = np.minimum(r * A, np.minimum(np.maximum(r, LO_), HI_) * A).astype(np.float32)
    tie = (A < 0) & (cA == clip1)
    assert tie.any() and active.any() and (~active & (A < 0)).any()
    # on a tie half the seed without the option; where the bound is active none
    g_off = PPO.dual_seed32(r, A, LO_, HI_, None)[0]
    assert np.array_equal(glp[tie], np.float32(0.5) * g_off[tie]) and (g_off[tie] != 0).all()
    assert not glp[active].any()
    assert np.array_equal(active, (A < 0) & (cA > clip1))
    # float64 away from the ties and the clip range's bounds, where fp32 rounding decides the branch
    s64, gr64, act64 = PPO.surr64(r, A, LO_, HI_, np.float32(c))
    away = (np.abs(cA - clip1) > 1e-5 * np.abs(cA)) & (np.abs(r - LO_) > 1e-6) & (np.abs(r - HI_) > 1e-6)
    assert np.allclose(s64, s_ref, rtol=1e-6, atol=1e-7) and np.array_equal(act64[away], active[away])
    assert np.allclose((gr64 * r)[away], g_ref[away], rtol=1e-6, atol=1e-7)


def test_dual_clip_is_fp32_c_times_A():
    """c * A with a Python float c and an fp32 tensor A is fp32(c) * A (what the Engine passes the library)."""
    A = torch.tensor(np.random.default_rng(0).normal(size=2000).astype(np.float32))
    for c in (1.1, 1.5, 2.0 / 3.0 + 1.0, 3.3, 7.77):
        assert torch.equal(c * A, torch.tensor(np.float32(c)) * A), c


def torch_value(V, R, delta, V_old=None, vclip=None):
    v = torch.tensor(np.asarray(V, np.float32), requires_grad=True)
    ov = None if V_old is None else torch.tensor(np.asarray(V_old, np.float32))
    t = PPO.value_terms(v, torch.tensor(np.asarray(R, np.float32)), delta, ov, vclip)
    t.sum().backward()
    return t.detach().numpy(), v.grad.numpy()


@pytest.mark.parametrize("delta", [0.25, 1.0, 0.3, 1e30])
def test_huber_seed_against_autograd(delta):
    d32 = np.float32(delta)
    e = np.array([0.0, 0.01, -0.2, 0.5, -0.9, 2.0, -7.5, 1e3], np.float32)
    if delta < 1e3:
        e = np.concatenate([e, [d32, -d32, np.nextafter(d32, np.float32(0)), np.nextafter(d32, np.float32(9))]])
    R = np.linspace(-1, 1, e.size).astype(np.float32)
    V = (R + e).astype(np.float32)
    loss_ref, g_ref = torch_value(V, R, delta)
    gv, loss, _, lin = PPO.value_seed32(V, R, delta, c_value=1.0, inv_batch=1.0)
    assert np.array_equal(loss, loss_ref) and np.array_equal(gv, g_ref)
    dv = (V - R).astype(np.float32)
    assert np.array_equal(lin, np.abs(dv) > d32)
    inside = np.abs(dv) < d32
    assert np.array_equal(loss[inside], (dv * dv)[inside])          # the reference's term itself inside delta
    if delta > 1e3:            # beyond every |e|: exactly the step without Huber
        g_off, l_off, _, _ = PPO.value_seed32(V, R, None, c_value=0.5, inv_batch=1.0 / 7)
        g_on, l_on, _, lin_on = PPO.value_seed32(V, R, delta, c_value=0.5, inv_batch=1.0 / 7)
        assert np.array_equal(g_on, g_off) and np.array_equal(l_on, l_off) and not lin_on.any()
    g64, l64, _, lin64 = PPO.value64(V, R, d32)
    away = np.abs(np.abs(dv) - d32) > 1e-5 * d32        # float64's V - R may fall on the other side of delta
    assert np.allclose(g64, g_ref, rtol=1e-6) and np.allclose(l64, loss_ref, rtol=1e-6)
    assert np.array_equal(lin64[away], lin[away])


def test_huber_backward_is_the_fp32_clamp():
    """The backward of 2 huber_loss is exactly 2 clamp(e, -fp32(delta), fp32(delta)), and inside delta the forward is
    e * e, on many values."""
    rng = np.random.default_rng(1)
    V, R = (rng.normal(scale=2, size=5000).astype(np.float32) for _ in range(2))
    for delta in (0.1, 0.7, 1.3):
        loss, g = torch_value(V, R, delta)
        e = (V - R).astype(np.float32)
        d32 = np.float32(delta)
        assert np.array_equal(g, (2 * np.clip(e, -d32, d32)).astype(np.float32))
        inside = np.abs(e) < d32
        assert np.array_equal(loss[inside], (e * e)[inside])


@pytest.mark.parametrize("delta", [0.3, 1e30])
def test_huber_with_value_clip_against_autograd(delta):
    """max(h(V - R), h(Vc - R)) in every branch of the clipped value loss."""
    rng = np.random.default_rng(2)
    R = rng.normal(size=400).astype(np.float32)
    V = (R + rng.normal(scale=0.6, size=400)).astype(np.float32)
    V_old = (V + rng.choice([0.0, 0.05, -0.1, 0.5, -0.5, 2.0], size=400)).astype(np.float32)
    loss_ref, g_ref = torch_value(V, R, delta, V_old, 0.2)
    gv, loss, _, lin = PPO.value_seed32(V, R, delta, c_value=1.0, inv_batch=1.0, V_old=V_old, value_clip=0.2)
    assert np.array_equal(loss, loss_ref)
    assert np.allclose(gv, g_ref, rtol=1e-6, atol=1e-7)
    g64, l64, _, lin64 = PPO.value64(V, R, np.float32(delta), V_old, np.float32(0.2))
    assert np.allclose(l64, loss_ref, rtol=1e-5, atol=1e-7) and np.allclose(g64, g_ref, rtol=1e-5, atol=1e-6)
    if delta < 1:
        assert lin.any() and not lin.all()


def minibatch(seed=3, n=10):
    states, actions = synth.make_states(seed, "small", n, stages=[i % 2 for i in range(n)])
    adv, ret, exps = synth.make_ppo_targets(seed, n)
    exps[1] = 0.0
    adv = np.where(np.arange(n)[:, None] % 3 == 0, np.abs(adv), -np.abs(adv)).astype(np.float32)
    fixed = np.random.default_rng(seed).normal(-3.0, 0.6, size=(n, 1)).astype(np.float32)
    return states, actions, adv, ret, exps, fixed


@pytest.mark.parametrize("opts", [dict(dual_clip=1.3), dict(huber_delta=0.4), dict(dual_clip=1.3, huber_delta=0.4),
                                  dict(dual_clip=1.3, huber_delta=0.4, value_clip=0.2)])
def test_numpy_oracle_matches_the_torch_port(opts):
    states, actions, adv, ret, exps, fixed = minibatch()
    flat = PL.default_init(3)
    b = TP.stack_states(states)
    with torch.no_grad():
        P = TP.params_from_flat(torch.tensor(flat))
        v0 = TP.value(P, b).numpy().reshape(-1)
        lp0, _ = TP.log_prob_entropy(P, b, torch.tensor(actions))
    old = None
    if "value_clip" in opts:
        old = (v0 + np.resize(np.array([0.0, 0.05, -0.5, 0.5, 2.0], np.float32), v0.size)).astype(np.float32)
    # ratios well above c on some exps != 0 graphs with A < 0
    fixed = (lp0.numpy() - np.resize(np.array([0.9, -0.4, 0.6, 0.1, 1.2], np.float32), (10, 1))).astype(np.float32)
    ratio = np.exp(lp0.numpy().reshape(-1) - fixed.reshape(-1))
    want = PPO.sgnn_minibatch(flat.astype(np.float64), states, actions, adv, ret, fixed, exps, old_values=old, **opts)
    agent = PPO.PortAgent(flat, **opts)
    if old is not None:
        agent.old_values = torch.tensor(old).reshape(-1, 1)
    ind = torch.tensor(exps).nonzero(as_tuple=False).squeeze(1)
    losses = agent.backward(b, torch.tensor(actions), torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    assert np.allclose(losses, [want["loss"], want["value_loss"], want["surr_loss"], want["entropy_loss"]],
                       rtol=2e-5, atol=2e-6)
    assert rel(agent.flat_grad(), want["grad"]) < 1e-4
    plain = TP.PortAgent(flat)
    plain.backward(b, torch.tensor(actions), torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    assert rel(plain.flat_grad(), want["grad"]) > 1e-3               # the options change the gradient
    if "dual_clip" in opts:
        assert 0 < want["dual"] < int((exps != 0).sum()), (want["dual"], ratio)
    if "huber_delta" in opts:
        assert 0 < want["linear"] < 10


@pytest.mark.parametrize("bad", BAD_DUAL)
def test_bad_dual_clip_is_refused_before_cuda(monkeypatch, bad):
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("a CUDA call before the argument check"))
    with pytest.raises(ValueError, match="dual_clip"):
        check_dual_clip(bad)
    with pytest.raises(ValueError, match="dual_clip"):
        Engine("cuda:0", 64, 64, dual_clip=bad)
    with pytest.raises(ValueError, match="dual_clip"):
        PPOUpdater(PL.default_init(0), 64, 64, "cuda:0", dual_clip=bad)


@pytest.mark.parametrize("bad", BAD_HUBER)
def test_bad_huber_delta_is_refused_before_cuda(monkeypatch, bad):
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("a CUDA call before the argument check"))
    with pytest.raises(ValueError, match="huber_delta"):
        check_huber_delta(bad)
    with pytest.raises(ValueError, match="huber_delta"):
        Engine("cuda:0", 64, 64, huber_delta=bad)
    with pytest.raises(ValueError, match="huber_delta"):
        PPOUpdater(PL.default_init(0), 64, 64, "cuda:0", huber_delta=bad)


def test_good_values_pass():
    assert check_dual_clip(None) == 0.0 and check_huber_delta(None) == 0.0
    assert check_dual_clip(3) == 3.0 and check_dual_clip(np.float32(1.5)) == 1.5 and check_dual_clip(1e30) == 1e30
    assert check_huber_delta(1) == 1.0 and check_huber_delta(np.float64(0.25)) == 0.25


def fake_agent():
    c = Cfg(64, 64)
    c.agent, c.agent_specs = "rl-sgnn", {}
    for k, v in dict(lr=4e-4, eps=1e-5, clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01, gamma=0.99, tau=0.95,
                     num_optim_epoch=1, mini_batch_size=16).items():
        setattr(c, k, v)
    return types.SimpleNamespace(cfg=c, device=torch.device("cuda", 0))


@pytest.mark.parametrize("kw", [dict(dual_clip=1.0), dict(dual_clip=float("nan")), dict(huber_delta=0.0),
                                dict(huber_delta=True), dict(huber_delta=float("inf"))])
def test_use_b200_update_refuses_before_cuda(monkeypatch, kw):
    from drl_urban_planning_b200.agent import use_b200_update
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("a CUDA call before the argument check"))
    with pytest.raises(ValueError, match=next(iter(kw))):
        use_b200_update(fake_agent(), **kw)


def test_setters_without_a_context():
    L = _lib.lib()
    assert L.upb_set_dual_clip(None, C.c_float(2.0)) == -1 and b"set_dual_clip" in L.upb_last_error()
    assert L.upb_set_huber_delta(None, C.c_float(1.0)) == -1 and b"set_huber_delta" in L.upb_last_error()


def rows(n, seed=0):
    rng = np.random.default_rng(seed)
    st = np.zeros((n, 22))
    st[:, 3], st[:, 4] = 16, 12
    st[:, 0] = rng.random(n) * 10
    st[:, 1], st[:, 2] = rng.normal(size=n), -rng.random(n)
    st[:, VCLIP_LOSS_SLOT] = rng.random(n) * 5
    st[:, DUAL_COUNT_SLOT] = rng.integers(0, 12, n)
    st[:, HUBER_COUNT_SLOT] = rng.integers(0, 16, n)
    return st


@pytest.mark.parametrize("dual,huber", [(False, False), (True, False), (False, True), (True, True)])
def test_update_log_slots(dual, huber):
    st = rows(5)
    diag = {k: np.arange(5, dtype=np.float64) for k in NAMES}
    logged = []
    book = UpdateLog(1, 0.5, 0.01, log_fn=lambda tg, v, s: logged.append((tg, v, s)), dual_clip=dual, huber=huber)
    book.epoch(0, st, diag)
    out = book.finish(True)
    vl = [v for tg, v, _ in logged if tg == "loss/value_loss"]
    want_vl = st[:, VCLIP_LOSS_SLOT if huber else 0] / 16
    assert np.allclose(vl, want_vl)
    tags = {tg for tg, _, _ in logged}
    assert ("diag/dual_clip_fraction" in tags) == dual and ("total_dual_clip_fraction" in out) == dual
    assert ("diag/huber_fraction" in tags) == huber and ("total_huber_fraction" in out) == huber
    if dual:
        assert np.isclose(out["total_dual_clip_fraction"], (st[:, DUAL_COUNT_SLOT] / 12).mean())
    if huber:
        assert np.isclose(out["total_huber_fraction"], (st[:, HUBER_COUNT_SLOT] / 16).mean())
