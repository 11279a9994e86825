"""CPU: the clipped value loss and the per-minibatch advantage normalisation -- the oracles' seed against torch autograd
in every branch, the float64 minibatch oracle against the torch port, the normalisation oracle against torch's fp32
formula, the argument checks and the update's host bookkeeping of statistics slots 15 / 16."""
import os
import types

import numpy as np
import pytest
import torch

import ppo_oracle as PPO
import vclip_oracle as VO
from drl_urban_planning_b200 import _lib, synth
from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.diagnostics import NAMES
from drl_urban_planning_b200.engine import Engine, check_value_clip
from drl_urban_planning_b200.ppo import VCLIP_COUNT_SLOT, VCLIP_LOSS_SLOT, UpdateLog
from fixtures_io import expand_states
from harness import Cfg, load, rel
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP

BAD = [0.0, -0.2, -1e-30, float("nan"), float("inf"), -float("inf")]

# (V, R, V_old, c): one graph in each branch of the seed
BRANCHES = {
    "unclipped_larger": (1.0, 0.0, 0.9, 0.05),          # d = 0.1 > c, Vc = 0.95: a > b
    "clipped_larger": (0.1, 1.0, -0.5, 0.2),            # d = 0.6 > c, Vc = -0.3: b > a, clamp saturated: gradient 0
    "inside_clamp": (0.7, 0.2, 0.65, 0.2),              # |d| < c: Vc = V up to rounding
    "exact_tie": (0.3125, -1.0, 0.3125, 0.2),           # d = 0: a == b
    "saturated_tie": (1.0, 0.0, -1.5, 0.5),             # d = 2.5 > c, Vc = -1: a == b == 1, the clamp passes nothing
    "at_the_bound": (1.5, 0.25, 1.0, 0.5),              # |d| == c exactly: the inclusive clamp passes the gradient
}


def autograd_seed(V, R, V_old, c):
    v = torch.tensor([V], dtype=torch.float32, requires_grad=True)
    loss = VO.clipped_value_loss(v, torch.tensor([R]), torch.tensor([V_old]), c)
    loss.backward()
    return float(v.grad[0]), float(loss.detach())


@pytest.mark.parametrize("case", sorted(BRANCHES))
def test_seed_against_autograd(case):
    V, R, V_old, c = BRANCHES[case]
    g_ref, loss_ref = autograd_seed(V, R, V_old, c)
    g32, l32, clipped, _ = PPO.value_seed32(V, R, c_value=1.0, inv_batch=1.0, V_old=V_old, value_clip=c)
    g64, l64, clipped64, _ = PPO.value64(V, R, V_old=V_old, value_clip=c)
    assert np.float32(g32[0]) == np.float32(g_ref) and np.float32(l32[0]) == np.float32(loss_ref), case
    assert abs(g64[0] - g_ref) <= 1e-6 * max(1.0, abs(g_ref)) and abs(l64[0] - loss_ref) <= 1e-6
    want_clipped = {"clipped_larger": 1.0}.get(case, 0.0)
    assert clipped[0] == want_clipped and clipped64[0] == want_clipped
    if case == "saturated_tie":
        assert g_ref == 1.0          # half of 2 (V - R); the clipped input is cut off by the clamp
    if case == "clipped_larger":
        assert g_ref == 0.0


def test_seed_takes_torchs_branch_inside_the_clamp():
    """V_old + (V - V_old) need not round back to V: across many values the fp32 seed picks the branch torch picks,
    including the graphs where a and b differ only in the last bits."""
    rng = np.random.default_rng(0)
    V = rng.normal(size=4000).astype(np.float32)
    V_old = (V + rng.normal(scale=0.05, size=4000)).astype(np.float32)
    R = rng.normal(size=4000).astype(np.float32)
    v = torch.tensor(V, requires_grad=True)
    loss = VO.clipped_value_loss(v, torch.tensor(R), torch.tensor(V_old), 0.2) * V.size
    loss.backward()
    g32, l32, clipped, _ = PPO.value_seed32(V, R, c_value=1.0, V_old=V_old, value_clip=0.2)
    d = torch.tensor(V) - torch.tensor(V_old)
    vc = torch.tensor(V_old) + torch.clamp(d, -0.2, 0.2)
    a, b = (torch.tensor(V) - torch.tensor(R)).pow(2), (vc - torch.tensor(R)).pow(2)
    assert np.array_equal(clipped, (b > a).numpy().astype(np.float32))
    assert ((a != b) & (d.abs() < 0.2)).any()            # last-bit differences inside the clamp do occur
    assert np.allclose(g32, v.grad.numpy(), rtol=1e-6, atol=1e-7)
    assert np.array_equal(l32, torch.max(a, b).numpy())


def test_clamp_bounds_are_the_fp32_range():
    """torch.clamp(x, -c, c) with a Python float c clamps an fp32 tensor at +-fp32(c) (the Engine passes
    np.float32(c)): values one ulp either side of fp32(c) land where the kernel's fminf / fmaxf put them."""
    for c in (0.1, 0.2, 0.3, 1.0 / 3.0, 0.7):
        c32 = np.float32(c)
        x = np.array([np.nextafter(c32, np.float32(0)), c32, np.nextafter(c32, np.float32(2)),
                      -np.nextafter(c32, np.float32(0)), -c32, -np.nextafter(c32, np.float32(2))], np.float32)
        got = torch.clamp(torch.tensor(x), -c, c).numpy()
        want = np.minimum(np.maximum(x, -c32), c32)
        assert np.array_equal(got, want), c


def test_numpy_oracle_matches_the_torch_port():
    """The float64 minibatch oracle with the clipped seed against the torch port's autograd of the same loss, on a
    mixed-stage minibatch whose old values put graphs in every branch."""
    states, actions = synth.make_states(3, "small", 10, stages=[i % 2 for i in range(10)])
    adv, ret, exps = synth.make_ppo_targets(3, 10)
    exps[1] = 0.0
    fixed = np.random.default_rng(3).normal(-3.0, 0.3, size=(10, 1)).astype(np.float32)
    flat = PL.default_init(3)
    b = TP.stack_states(states)
    with torch.no_grad():
        v0 = TP.value(TP.params_from_flat(torch.tensor(flat)), b).numpy().reshape(-1)
    old = (v0 + np.array([0.0, 0.05, -0.05, 0.5, -0.5, 0.3, -0.3, 0.01, 2.0, -2.0], np.float32)).astype(np.float32)
    c = 0.2
    r = PPO.sgnn_minibatch(flat.astype(np.float64), states, actions, adv, ret, fixed, exps, old_values=old,
                           value_clip=c)
    agent = PPO.PortAgent(flat, value_clip=c)
    agent.old_values = torch.tensor(old).reshape(-1, 1)
    ind = torch.tensor(exps).nonzero(as_tuple=False).squeeze(1)
    losses = agent.backward(b, torch.tensor(actions), torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    assert np.allclose(losses, [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]], rtol=2e-5, atol=2e-6)
    assert rel(agent.flat_grad(), r["grad"]) < 1e-4
    assert 0 < r["clipped"] < 10
    plain = TP.PortAgent(flat)
    plain.backward(b, torch.tensor(actions), torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    assert rel(plain.flat_grad(), r["grad"]) > 1e-3          # the clip changes the gradient


@pytest.mark.parametrize("n_ind", [0, 1, 2, 16])
def test_normalisation_oracle_against_torch(n_ind):
    """|ind| of 0, 1, 2 and B = 16 in the first minibatch, T = 45 (a tail of 13 states the update never steps on)."""
    rng = np.random.default_rng(n_ind)
    T, B = 45, 16
    adv = rng.normal(2.0, 3.0, size=T).astype(np.float32)
    exps = np.ones(T, np.float32)
    order = rng.permutation(T)
    exps[order[:B]] = 0.0
    exps[order[:n_ind]] = 1.0
    got = VO.normalize64(adv, exps, order, B)
    want = VO.normalize_torch(adv, exps, order, B)
    assert np.allclose(got, want, rtol=0, atol=2e-6 * np.abs(want).max())
    tail = order[2 * B:]
    assert np.array_equal(got[tail], adv[tail])
    first = order[:B]
    if n_ind < 2:
        assert np.array_equal(got[first], adv[first])
    else:
        sel = got[first][exps[first] != 0].astype(np.float64)
        assert abs(sel.mean()) < 1e-5 and abs(sel.std(ddof=1) - 1.0) < 1e-5


def test_normalisation_of_constant_advantages():
    adv = np.full(32, 3.25, np.float32)
    exps = np.ones(32, np.float32)
    order = np.arange(32)
    got = VO.normalize64(adv, exps, order, 8)
    assert np.array_equal(got, VO.normalize_torch(adv, exps, order, 8)) and not got.any()


def test_check_value_clip_values():
    assert check_value_clip(None) == 0.0
    assert check_value_clip(0.2) == 0.2 and check_value_clip(np.float32(10.0)) == 10.0
    for bad in BAD:
        with pytest.raises(ValueError):
            check_value_clip(bad)


@pytest.mark.parametrize("bad", BAD)
def test_bad_value_clip_is_rejected_before_any_cuda_call(bad, monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    with pytest.raises(ValueError, match="value_clip"):
        Engine("cuda:0", 16, 16, value_clip=bad)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError, match="value_clip"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", value_clip=bad,
                   normalize_advantage=True)
    from drl_urban_planning_b200.agent import B200Update
    for kind in ("rl-sgnn", "rl-mlp"):
        cfg = Cfg(64, 64)
        cfg.agent, cfg.clip_epsilon = kind, 0.2
        with pytest.raises(ValueError, match="value_clip"):
            B200Update(types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0)), value_clip=bad)


def test_c_entry_points_validate_without_a_context():
    import ctypes as C
    L = _lib.lib()
    assert L.upb_set_value_clip(None, C.c_float(0.2)) == -1 and b"set_value_clip" in L.upb_last_error()
    assert L.upb_normalize_advantages(None, None, None, None, 0, 1, None, None) == -1
    assert b"normalize_advantages" in L.upb_last_error()


def stat_rows(nb, seed):
    rng = np.random.default_rng(seed)
    st = np.zeros((nb, 17))
    st[:, 0] = rng.random(nb) * 4
    st[:, 1] = rng.normal(size=nb)
    st[:, 2] = -rng.random(nb) * 30
    st[:, 3] = 32
    st[:, 4] = 28
    st[:, 8:13] = rng.random((nb, 5))
    st[:, VCLIP_LOSS_SLOT] = st[:, 0] + rng.random(nb)
    st[:, VCLIP_COUNT_SLOT] = rng.integers(0, 33, nb)
    return st


@pytest.mark.parametrize("diag", [False, True])
@pytest.mark.parametrize("value_clip", [False, True])
def test_update_log_takes_the_clipped_value_loss(value_clip, diag):
    VC, EC = 0.5, 0.01
    logged = []
    book = UpdateLog(2, VC, EC, 0, 0, lambda t, v, s: logged.append((t, v, s)), value_clip=value_clip)
    eps = [stat_rows(3, s) for s in range(2)]
    for e, st in enumerate(eps):
        d = {n: np.arange(3, dtype=np.float64) for n in NAMES} if diag else None
        book.epoch(e, st, d)
    out = book.finish(diag)
    st = np.concatenate(eps)
    vl = st[:, VCLIP_LOSS_SLOT if value_clip else 0] / 32
    loss = st[:, 1] / 28 + VC * vl + EC * st[:, 2] / 28
    assert np.allclose([v for t, v, _ in logged if t == "loss/value_loss"], vl)
    assert np.allclose([v for t, v, _ in logged if t == "loss/loss"], loss)
    assert np.isclose(out["total_value_loss"], vl.sum() / 2)
    tags = {t for t, _, _ in logged}
    assert ("diag/value_clip_fraction" in tags) == (value_clip and diag)
    assert ("total_value_clip_fraction" in out) == (value_clip and diag)
    if value_clip and diag:
        frac = [v for t, v, _ in logged if t == "diag/value_clip_fraction"]
        assert np.allclose(frac, st[:, VCLIP_COUNT_SLOT] / 32)
        assert np.isclose(out["total_value_clip_fraction"], (st[:, VCLIP_COUNT_SLOT] / 32).mean())
    if not value_clip:
        ref = []
        plain = UpdateLog(2, VC, EC, 0, 0, lambda t, v, s: ref.append((t, v, s)))
        for e, st_e in enumerate(eps):
            plain.epoch(e, st_e, {n: np.arange(3, dtype=np.float64) for n in NAMES} if diag else None)
        plain.finish(diag)
        assert ref == logged                   # off: the tags and values of a log that never heard of the option


# ---- the golden vectors recorded by the unmodified reference with both options (tests/golden/make_golden_vf.py) ------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    z = load(GOLDEN, name)
    assert float(z["value_clip"]) > 0 and int(z["normalize_advantage"]) == 1
    return z, expand_states(z)


@pytest.mark.parametrize("name", ["small_mixed_vf", "mlp_small_vf"])
def test_normalisation_oracles_reproduce_the_fixture(name):
    z, _ = golden(name)
    B = len(z["exps"])
    for got in (VO.normalize64(z["advantages"], z["exps"], np.arange(B), B),
                VO.normalize_torch(z["advantages"], z["exps"], np.arange(B), B)):
        assert np.allclose(got, z["advantages_normalized"].reshape(-1), rtol=0, atol=1e-6)


def test_numpy_oracle_reproduces_small_mixed_vf():
    """The float64 oracle with the clipped seed: losses, every gradient and the three-step trajectory (first step
    clipped); the oracle at the default settings (raw advantages, no value clipping) misses the fixture."""
    z, states = golden("small_mixed_vf")
    B, c = len(states), float(z["value_clip"])
    adv = VO.normalize64(z["advantages"], z["exps"], np.arange(B), B)
    args = (states, z["actions"], adv, z["returns"], z["fixed_log_probs"], z["exps"])
    live = ON.live_mask(states)
    flat = z["params"].astype(np.float64)
    m = v = tt = np.zeros(PL.NUM_PARAMS)
    for k in range(3):
        r = PPO.sgnn_minibatch(flat, *args, old_values=z["old_values"], value_clip=c)
        got = [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]]
        assert np.allclose(got, z["losses"][k], rtol=2e-5, atol=2e-6), (k, got, z["losses"][k])
        assert rel(r["grad"], z["grads"][k]) < 1e-4, k
        g = ON.clip_groups(r["grad"]) if k == 0 else r["grad"]
        flat, m, v, tt = ON.adam_step(flat, m, v, tt, g, live)
        assert rel(flat, z["params_after"][k]) < 5e-6, k
    r0 = ON.ppo_minibatch(z["params"].astype(np.float64), states, z["actions"], z["advantages"], z["returns"],
                          z["fixed_log_probs"], z["exps"])
    assert rel(r0["grad"], z["grads"][0]) > 1e-2


@pytest.mark.parametrize("name", ["small_mixed_vf", "mlp_small_vf"])
def test_torch_ports_reproduce_the_fixture(name):
    """The torch port (SGNN) or the rl-mlp port with the clipped loss: losses and parameters of three steps, the first
    one clipped; the port at the default settings misses the first step."""
    z, states = golden(name)
    mlp = name.startswith("mlp")
    B, c = len(states), float(z["value_clip"])
    b = (MP.stack_states if mlp else TP.stack_states)(states)
    adv = torch.tensor(VO.normalize_torch(z["advantages"], z["exps"], np.arange(B), B)).reshape(-1, 1)
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    args = (b, torch.tensor(z["actions"]), adv, torch.tensor(z["returns"]), torch.tensor(z["fixed_log_probs"]), ind)
    agent = (PPO.MLPPortAgent if mlp else PPO.PortAgent)(z["params"], value_clip=c)
    agent.old_values = torch.tensor(z["old_values"]).reshape(-1, 1)
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < 5e-6, k
    base = (MP.MLPPortAgent if mlp else TP.PortAgent)(z["params"])
    base.step(b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
              torch.tensor(z["fixed_log_probs"]), ind)
    assert rel(base.flat(), z["params_after"][0]) > 1e-4
