"""Value-target normalisation (`value_norm`, upb_set_value_norm) without a GPU: the argument checks, the exported
symbols, the float64 oracle (tests/vnorm_oracle.py) against an independent torch formulation of MAPPO's ValueNorm and
PopArt's identity, the oracle's fp32 fma, and the checkpoint entry of B200Update."""
import ctypes as C
import types
from fractions import Fraction

import numpy as np
import pytest
import torch

import vnorm_oracle as VN
from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.engine import Engine, check_value_norm, value_norm_stats
from harness import Cfg

BAD_SWITCH = [0.5, 2, -1, "yes", None, float("nan")]
BAD_BETA = [0.0, 1.0, -0.5, 1.5, float("nan"), float("inf"), "0.9", None, True]


def test_check_value_norm_values():
    assert check_value_norm(False, 0.99999) == (False, 0.99999)
    assert check_value_norm(True, 0.5) == (True, 0.5)
    assert check_value_norm(1, np.float32(0.25)) == (True, 0.25)
    assert check_value_norm(np.bool_(False), 1e-9)[0] is False
    for bad in BAD_SWITCH:
        with pytest.raises(ValueError, match="value_norm value"):
            check_value_norm(bad, 0.99999)
    for bad in BAD_BETA:
        with pytest.raises(ValueError, match="value_norm_beta"):
            check_value_norm(True, bad)


@pytest.mark.parametrize("kw", [dict(value_norm=b) for b in BAD_SWITCH] +
                         [dict(value_norm=True, value_norm_beta=b) for b in BAD_BETA])
def test_bad_value_norm_is_rejected_before_any_cuda_call(kw, monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    with pytest.raises(ValueError, match="value_norm"):
        Engine("cuda:0", 16, 16, **kw)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError, match="value_norm"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", **kw)
    from drl_urban_planning_b200.agent import B200Update
    for kind in ("rl-sgnn", "rl-mlp"):
        cfg = Cfg(64, 64)
        cfg.agent, cfg.clip_epsilon = kind, 0.2
        with pytest.raises(ValueError, match="value_norm"):
            B200Update(types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0)), **kw)


def test_c_entry_points_are_exported_and_validate_without_a_context():
    L = _lib.lib()
    names = ["upb_set_value_norm"] + [p + n for p in ("upb_", "upb_mlp_") for n in
                                      ("value_norm_denormalize", "value_norm_update", "get_value_norm_state",
                                       "set_value_norm_state")]
    for name in names:
        assert name in _lib.EXPORTED_SYMBOLS
    assert L.upb_set_value_norm(None, 0.5) == -1 and b"set_value_norm" in L.upb_last_error()
    st = (C.c_double * 3)()
    assert L.upb_get_value_norm_state(None, st) == -1
    assert L.upb_mlp_set_value_norm_state(None, st) == -1
    assert L.upb_value_norm_update(None, None, None, 1, None, None, None, None, None) == -1
    assert L.upb_mlp_value_norm_denormalize(None, None, 1, None, None) == -1


# ---- the oracle against MAPPO's ValueNorm ----------------------------------------------------------------------------
class ValueNorm:
    """MAPPO's ValueNorm (per_element_update=False, norm_axes=1, epsilon=1e-5) over a scalar value, in float64 torch."""

    def __init__(self, beta):
        self.beta = beta
        self.running_mean = torch.zeros(1, dtype=torch.float64)
        self.running_mean_sq = torch.zeros(1, dtype=torch.float64)
        self.debiasing_term = torch.tensor(0.0, dtype=torch.float64)

    def running_mean_var(self):
        mean = self.running_mean / self.debiasing_term.clamp(min=1e-5)
        mean_sq = self.running_mean_sq / self.debiasing_term.clamp(min=1e-5)
        return mean, (mean_sq - mean ** 2).clamp(min=1e-2)

    def update(self, x):
        x = torch.as_tensor(x, dtype=torch.float64).reshape(-1, 1)
        w = self.beta
        self.running_mean.mul_(w).add_(x.mean(dim=0) * (1.0 - w))
        self.running_mean_sq.mul_(w).add_((x ** 2).mean(dim=0) * (1.0 - w))
        self.debiasing_term.mul_(w).add_(1.0 * (1.0 - w))

    def denormalize(self, n):
        mean, var = self.running_mean_var()
        return torch.as_tensor(n, dtype=torch.float64) * torch.sqrt(var) + mean


def close(a, b, tol=1e-12):
    return abs(a - b) <= tol * max(abs(b), 1e-300)


@pytest.mark.parametrize("beta", [0.99999, 0.99, 0.5, 1e-3, 1e-9, 1.0 - 1e-12])
def test_oracle_follows_mappo_value_norm(beta):
    rng = np.random.default_rng(int(beta * 1e6) % 1000)
    ref, state = ValueNorm(beta), (0.0, 0.0, 0.0)
    # d == 0 is the identity (MAPPO would give std 0.1 from its variance clamp before any update)
    assert VN.stats(*state) == (0.0, 1.0) == value_norm_stats(*state)
    for k in range(40):
        scale = 10.0 ** rng.uniform(-4, 4)
        n = int(rng.integers(1, 600))
        r = (rng.normal(rng.normal() * scale, scale, n) if k % 5 else np.full(n, scale)).astype(np.float32)
        ref.update(r.astype(np.float64))
        state = VN.update(state, r, beta)
        for got, want in zip(state, (ref.running_mean.item(), ref.running_mean_sq.item(), ref.debiasing_term.item())):
            assert close(got, want), (k, got, want)
        mean, var = ref.running_mean_var()
        mu, sd = VN.stats(*state)
        assert close(mu, mean.item(), 1e-10 if beta < 1e-6 else 1e-12) or abs(mu - mean.item()) < 1e-12 * sd
        assert close(sd, float(np.sqrt(var.item())), 1e-9)
        assert value_norm_stats(*state) == (mu, sd)
    # a constant batch and a tiny spread hit the variance clamp
    st = VN.update((0.0, 0.0, 0.0), np.full(8, 3.0, np.float32), 0.9)
    assert VN.stats(*st) == pytest.approx((3.0, 0.1), rel=1e-12)


def test_non_finite_returns_leave_the_state():
    st = VN.update((0.0, 0.0, 0.0), np.arange(5, dtype=np.float32), 0.9)
    for bad in (np.nan, np.inf, -np.inf):
        r = np.arange(5, dtype=np.float32)
        r[3] = bad
        assert VN.update(st, r, 0.9) == st
        out = VN.step(st, r, None, np.ones(32, np.float32), np.float32(0.5), 0.9)
        assert out["state"] == st and out["b2"] == np.float32(0.5) and (out["w2"] == 1).all()


@pytest.mark.parametrize("seed", range(6))
def test_popart_preserves_the_output(seed):
    """sigma_n (w' h + b') + mu_n == sigma_o (w h + b) + mu_o, to 1e-12 in float64."""
    rng = np.random.default_rng(seed)
    state, beta = (0.0, 0.0, 0.0), [0.99999, 0.9, 0.3][seed % 3]
    w, b = rng.normal(size=32), float(rng.normal())
    h = np.tanh(rng.normal(size=(64, 32)))
    for _ in range(5):
        old = VN.stats(*state)
        state = VN.update(state, rng.normal(rng.normal() * 100, 10.0 ** rng.uniform(-2, 3), 300), beta)
        new = VN.stats(*state)
        w2, b2 = VN.rescale(w, b, old, new, dtype=np.float64)
        before = old[1] * (h @ w + b) + old[0]
        after = new[1] * (h @ w2 + b2) + new[0]
        assert np.abs(after - before).max() <= 1e-12 * max(np.abs(before).max(), 1.0)
        w, b = w2, b2


def test_oracle_fmaf_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a = rng.normal(size=4000).astype(np.float32)
    x = rng.normal(size=4000).astype(np.float32)
    b = (rng.normal(size=4000) * 10.0 ** rng.integers(-6, 6, 4000)).astype(np.float32)
    # exact ties: b = the midpoint's remainder for a * x with an odd 25th bit
    a[:8], x[:8] = np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12)
    b[:8] = np.float32([2 ** -60, -2 ** -60, 0, 2 ** -30, -2 ** -30, 1, -1, 2 ** -24])
    got = VN.fmaf(a, x, b)
    for i in range(a.size):
        exact = Fraction(float(a[i])) * Fraction(float(x[i])) + Fraction(float(b[i]))
        f = np.float32(float(exact))
        cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
        dist = [abs(Fraction(float(c)) - exact) for c in cands]
        best = min(dist)
        ok = [c for c, d in zip(cands, dist) if d == best]
        want = ok[0] if len(ok) == 1 else next(c for c in ok if not (c.view(np.int32) & 1))
        assert got[i] == want, (i, a[i], x[i], b[i], got[i], want)


def test_denormalize_is_the_identity_at_d_zero():
    n = np.float32([-0.0, 0.0, 1.5, -3e-39, np.inf])
    out = VN.denormalize(n, (0.0, 0.0, 0.0))
    assert np.array_equal(out.view(np.int32), n.view(np.int32))


# ---- the checkpoint entry --------------------------------------------------------------------------------------------
class FakeEngine:
    def __init__(self):
        self.state = (0.0, 0.0, 0.0)

    def get_opt_state(self):
        return np.zeros(3, np.float32), np.zeros(3, np.float32), np.zeros(4, np.int64)

    def set_opt_state(self, *a, **k):
        pass

    def get_value_norm_state(self):
        return self.state

    def set_value_norm_state(self, st):
        self.state = tuple(float(x) for x in st)


def controller(value_norm):
    from drl_urban_planning_b200.agent import B200Update
    ctl = object.__new__(B200Update)
    ctl.updater = types.SimpleNamespace(engine=FakeEngine(), kl_coef=None, value_norm=value_norm)
    return ctl


def test_checkpoint_entry_and_value_stats():
    ctl = controller(True)
    assert ctl.value_stats() == (0.0, 1.0)
    ctl.updater.engine.state = (1.0, 5.0, 0.5)
    state = ctl.optimizer_state()
    assert state["value_norm"] == dict(m1=1.0, m2=5.0, d=0.5)
    assert ctl.value_stats() == VN.stats(1.0, 5.0, 0.5) == (2.0, np.sqrt(6.0))
    other = controller(True)
    other.load_optimizer_state(state)
    assert other.updater.engine.state == (1.0, 5.0, 0.5)
    del state["value_norm"]                  # an older checkpoint: the identity
    other.load_optimizer_state(state)
    assert other.updater.engine.state == (0.0, 0.0, 0.0)
    off = controller(False)
    off.updater.engine.state = (1.0, 5.0, 0.5)
    assert "value_norm" not in off.optimizer_state() and off.value_stats() == (0.0, 1.0)
