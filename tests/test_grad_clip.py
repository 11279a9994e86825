"""The global gradient-norm clip (`max_grad_norm`) without a GPU: the oracles against the fixtures the unmodified
reference recorded with clip_grad_norm_ on every step (tests/golden/make_golden_gclip.py), the float64 clip against
torch's, the argument checks and the update log's tags."""
import types

import numpy as np
import pytest
import torch

import gclip_oracle as GO
import ppo_oracle as PPO
from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.diagnostics import NAMES, grad_clip_coef
from drl_urban_planning_b200.engine import Engine, check_max_grad_norm
from drl_urban_planning_b200.ppo import GCLIP_NORM_SLOT, KL_STOP_SLOT, UpdateLog
from fixtures_io import expand_states
from harness import Cfg, load, rel
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP
from test_value_clip import GOLDEN

FIXTURES = ["small_mixed_gclip", "mlp_small_gclip"]


def port_args(z, mlp):
    b = (MP.stack_states if mlp else TP.stack_states)(expand_states(z))
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    return (b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
            torch.tensor(z["fixed_log_probs"]), ind)


@pytest.mark.parametrize("name", FIXTURES)
def test_torch_ports_reproduce_the_fixture(name):
    """The torch ports with clip_grad_norm_ on every step: losses, parameters of three steps, torch's norm; the ports
    without the clip (the reference's first-step clip) miss them."""
    z = load(GOLDEN, name)
    mlp = name.startswith("mlp")
    m = float(z["max_grad_norm"])
    assert (z["grad_norms"] > m).all()
    args = port_args(z, mlp)
    agent = (PPO.MLPPortAgent if mlp else PPO.PortAgent)(z["params"], max_grad_norm=m)
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < 5e-6, k
    base = (MP.MLPPortAgent if mlp else TP.PortAgent)(z["params"])
    for k in range(3):
        base.step(*args)
    assert rel(base.flat(), z["params_after"][2]) > 1e-3


@pytest.mark.parametrize("name", FIXTURES)
def test_float64_clip_reproduces_the_fixture(name):
    """The recorded gradients, clipped in float64 and fed to the float64 Adam, give the recorded trajectory; the norms
    are torch's; unclipped they miss it."""
    z = load(GOLDEN, name)
    m = float(z["max_grad_norm"])
    live = np.ones(z["params"].size, bool)
    if not name.startswith("mlp"):
        live = ON.live_mask(expand_states(z))
    flat, plain = z["params"].astype(np.float64), z["params"].astype(np.float64)
    st = [np.zeros(flat.size)] * 3
    sp = [np.zeros(flat.size)] * 3
    for k in range(3):
        g, norm = GO.clip64(z["grads"][k], m)
        assert np.isclose(norm, z["grad_norms"][k], rtol=1e-5)
        flat, *st = ON.adam_step(flat, *st, g, live)
        plain, *sp = ON.adam_step(plain, *sp, z["grads"][k].astype(np.float64), live)
        assert rel(flat, z["params_after"][k]) < 5e-6, k
    assert rel(plain, z["params_after"][2]) > 1e-3


@pytest.mark.parametrize("scale", [1e-3, 1.0, 50.0])
def test_float64_clip_against_clip_grad_norm(scale):
    rng = np.random.default_rng(int(scale * 1000))
    shapes = [(64, 52), (64,), (16, 23), (32, 67), (1,)]
    ts = [torch.tensor(rng.normal(size=s).astype(np.float32) * scale, requires_grad=True) for s in shapes]
    for x in ts:
        x.grad = x.detach().clone()
    flat = np.concatenate([x.grad.numpy().ravel() for x in ts])
    want, norm = GO.clip64(flat, 0.5)
    got = torch.nn.utils.clip_grad_norm_(ts, 0.5)
    assert np.isclose(float(got), norm, rtol=1e-6)
    assert rel(np.concatenate([x.grad.numpy().ravel() for x in ts]), want) < 1e-6


def test_coefficient_is_torchs_fp32():
    """grad_clip_coef is clip_grad_norm_'s fp32 coefficient bit for bit (reciprocal times max_norm, clamped at 1,
    NaN through)."""
    rng = np.random.default_rng(3)
    norms = np.concatenate([rng.random(2000).astype(np.float32) * 3, [0.0, 0.5, 1.0, np.nan, np.inf]]).astype(np.float32)
    for m in (0.5, 0.3, 1.0, 0.1234567):
        want = torch.clamp(m / (torch.tensor(norms) + 1e-6), max=1.0).numpy()
        got = grad_clip_coef(norms, m)
        assert np.array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        assert np.array_equal(got[ok], want[ok])


BAD = [0.0, -1.0, float("nan"), float("inf")]


def test_check_max_grad_norm_values():
    assert check_max_grad_norm(None, _lib.CLIP_REFERENCE) == 0.0
    assert check_max_grad_norm(0.5, _lib.CLIP_NEVER) == 0.5
    for bad in BAD:
        with pytest.raises(ValueError):
            check_max_grad_norm(bad, _lib.CLIP_NEVER)
    for mode in (_lib.CLIP_REFERENCE, _lib.CLIP_ALWAYS):
        with pytest.raises(ValueError, match="clip_mode=CLIP_NEVER"):
            check_max_grad_norm(0.5, mode)


@pytest.mark.parametrize("mode", [_lib.CLIP_REFERENCE, _lib.CLIP_ALWAYS, _lib.CLIP_NEVER])
@pytest.mark.parametrize("bad", BAD + [0.5])
def test_bad_max_grad_norm_is_rejected_before_any_cuda_call(bad, mode, monkeypatch):
    if bad == 0.5 and mode == _lib.CLIP_NEVER:
        return                                  # a valid setting
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    with pytest.raises(ValueError, match="max_grad_norm|CLIP_NEVER"):
        Engine("cuda:0", 16, 16, clip_mode=mode, max_grad_norm=bad)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError, match="max_grad_norm|CLIP_NEVER"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", clip_mode=mode, max_grad_norm=bad)
    from drl_urban_planning_b200.agent import B200Update
    for kind in ("rl-sgnn", "rl-mlp"):
        cfg = Cfg(64, 64)
        cfg.agent, cfg.clip_epsilon = kind, 0.2
        with pytest.raises(ValueError, match="max_grad_norm|CLIP_NEVER"):
            B200Update(types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0)), clip_mode=mode,
                       max_grad_norm=bad)


def test_c_entry_point_validates_without_a_context():
    import ctypes as C
    L = _lib.lib()
    assert L.upb_set_max_grad_norm(None, C.c_float(0.5)) == -1 and b"set_max_grad_norm" in L.upb_last_error()


def rows(nb, seed):
    rng = np.random.default_rng(seed)
    st = np.zeros((nb, 18))
    st[:, 0] = rng.random(nb)
    st[:, 3], st[:, 4] = 32, 28
    st[:, 8:13] = rng.random((nb, 5))
    st[:, GCLIP_NORM_SLOT] = rng.random(nb).astype(np.float32) + 0.2
    return st


@pytest.mark.parametrize("kl_stop", [False, True])
@pytest.mark.parametrize("diag", [False, True])
def test_update_log_reports_the_clip(diag, kl_stop):
    m = 0.6
    logged = []
    book = UpdateLog(2, 0.5, 0.01, 0, 0, lambda t, v, s: logged.append((t, v, s)), kl_stop=kl_stop, max_grad_norm=m)
    eps = [rows(4, s) for s in range(2)]
    if kl_stop:
        eps[1][2, KL_STOP_SLOT] = 1.0            # the step that stopped: logged, no Adam, slot 17 = 0
        eps[1][2, GCLIP_NORM_SLOT] = 0.0
    for e, st in enumerate(eps):
        if book.epoch(e, st, {n: np.arange(4, dtype=np.float64) for n in NAMES} if diag else None):
            break
    out = book.finish(diag)
    applied = np.concatenate([eps[0][:, GCLIP_NORM_SLOT], eps[1][:2 if kl_stop else 4, GCLIP_NORM_SLOT]])
    norms = [v for t, v, _ in logged if t == "diag/grad_norm"]
    fracs = [v for t, v, _ in logged if t == "diag/grad_clip_fraction"]
    if not diag:
        assert not norms and "total_grad_norm" not in out
        return
    assert np.allclose(norms, applied)
    clipped = (np.float32(1) / (applied.astype(np.float32) + np.float32(1e-6))) * np.float32(m) < 1
    assert 0 < clipped.sum() < clipped.size
    assert fracs == clipped.astype(float).tolist()
    assert np.isclose(out["total_grad_norm"], applied.mean())
    assert np.isclose(out["total_grad_clip_fraction"], clipped.mean())
    plain = []
    ref = UpdateLog(2, 0.5, 0.01, 0, 0, lambda t, v, s: plain.append((t, v, s)), kl_stop=kl_stop)
    for e, st in enumerate(eps):
        if ref.epoch(e, st, {n: np.arange(4, dtype=np.float64) for n in NAMES}):
            break
    ref.finish(diag)
    ours = {"diag/grad_norm", "diag/grad_clip_fraction", "diag/total_grad_norm", "diag/total_grad_clip_fraction"}
    assert [x for x in logged if x[0] not in ours] == plain
