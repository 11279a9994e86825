"""The per-epoch advantage recomputation (`recompute_advantage`) without a GPU: the switch's checks before any CUDA call,
the four exported C entry points, and the float64 targets oracle (tests/recompute_oracle.py) against an independent torch
formulation."""
import types

import numpy as np
import pytest
import torch

import recompute_oracle as RO
import vnorm_oracle as VN
from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.engine import check_recompute_advantage
from harness import Cfg
from oracle import sgnn_numpy as ON

BAD = [0.5, 2, -1, "yes", None, float("nan")]
SYMBOLS = ("upb_values", "upb_mlp_values", "upb_gae_targets", "upb_mlp_gae_targets")


def test_check_recompute_advantage_values():
    assert check_recompute_advantage(False) is False and check_recompute_advantage(True) is True
    assert check_recompute_advantage(0) is False and check_recompute_advantage(np.bool_(True)) is True
    assert check_recompute_advantage(np.int64(1)) is True
    for bad in BAD:
        with pytest.raises(ValueError, match="recompute_advantage"):
            check_recompute_advantage(bad)


@pytest.mark.parametrize("bad", BAD)
def test_bad_switch_is_rejected_before_any_cuda_call(bad, monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError, match="recompute_advantage"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", recompute_advantage=bad)
    from drl_urban_planning_b200.agent import B200Update
    for kind in ("rl-sgnn", "rl-mlp"):
        cfg = Cfg(64, 64)
        cfg.agent, cfg.clip_epsilon = kind, 0.2
        with pytest.raises(ValueError, match="recompute_advantage"):
            B200Update(types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0)), recompute_advantage=bad)


def test_c_entry_points_are_exported_and_validate_without_a_context():
    L = _lib.lib()
    for name in SYMBOLS:
        assert name in _lib.EXPORTED_SYMBOLS
    x = np.zeros(4, np.float32).ctypes.data
    assert L.upb_values(None, x, None, 1, x, x, None) == -1 and b"values" in L.upb_last_error()
    assert L.upb_mlp_values(None, x, None, 1, x, x, None) == -1 and b"mlp_values" in L.upb_last_error()
    assert L.upb_gae_targets(None, x, x, x, 4, 1.0, 0.0, x, x, x, None) == -1
    assert b"gae_targets" in L.upb_last_error()
    assert L.upb_mlp_gae_targets(None, x, x, x, 4, 1.0, 0.0, x, x, x, None) == -1
    assert b"mlp_gae_targets" in L.upb_last_error()


def rollout(seed, T=2000):
    rng = np.random.default_rng(seed)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 40, replace=False)] = 0.0
    rewards = (rng.standard_normal(T) * 30.0 + 200.0).astype(np.float32)
    head = rng.standard_normal(T).astype(np.float32)
    return rewards, masks, head


def torch_targets(rewards, masks, head, gamma, tau, state=None):
    """The same targets another way: TD errors formed for the whole buffer at once, then A_t = delta_t + gamma tau m_t
    A_{t+1} over the whole buffer (masks == 0 cuts it), the denormalisation an exact float64 affine map."""
    n = torch.tensor(head, dtype=torch.float64)
    if state is not None and state[2] != 0.0:
        mu, sd = VN.stats(*state)
        v = n * float(np.float32(sd)) + float(np.float32(mu))
    else:
        v = n.clone()
    r, m = torch.tensor(rewards, dtype=torch.float64), torch.tensor(masks, dtype=torch.float64)
    v_next = torch.cat([v[1:], torch.zeros(1, dtype=torch.float64)])
    delta = r + gamma * v_next * m - v
    adv = torch.zeros_like(delta)
    acc = torch.zeros((), dtype=torch.float64)
    for i in range(delta.numel() - 1, -1, -1):
        acc = delta[i] + gamma * tau * m[i] * acc
        adv[i] = acc
    ret = v + adv
    if state is not None:
        mu, sd = VN.stats(*state)
        ret = (ret - float(np.float32(mu))) / float(np.float32(sd))
    return adv.numpy(), ret.numpy(), n.numpy()


@pytest.mark.parametrize("gamma,tau", [(1.0, 0.0), (0.99, 0.95)])
@pytest.mark.parametrize("norm", [False, True])
def test_oracle_agrees_with_an_independent_torch_formulation(gamma, tau, norm):
    rewards, masks, head = rollout(3)
    state = VN.update((0.0, 0.0, 0.0), rewards, 0.99) if norm else None
    got = RO.targets(rewards, masks, head, gamma, tau, state)
    want = torch_targets(rewards, masks, head, gamma, tau, state)
    # the oracle's values are the fp32 fmaf the kernel forms; the torch ones are exact: half an fp32 ulp of V apart
    v = VN.denormalize(head, state) if norm else head
    vbar = 64 * np.spacing(np.abs(v).max().astype(np.float32))
    for g, w, name in zip(got, want, ("adv", "ret", "anchor")):
        assert np.abs(g - w).max() <= vbar, name
    assert np.array_equal(got[2], head.astype(np.float64))
    if norm:
        assert abs(np.mean(VN.denormalize(head, state)) - VN.stats(*state)[0]) < 5.0   # the statistics are in play


@pytest.mark.parametrize("gamma,tau", [(1.0, 0.0), (0.99, 0.95)])
def test_oracle_is_the_fp32_reference_gae_up_to_rounding(gamma, tau):
    """Without value normalisation the oracle is estimate_advantages in float64: within fp32 round-off of the
    reference's own fp32 scan, episode by episode."""
    rewards, masks, head = rollout(4, T=800)
    adv, ret, _ = RO.targets(rewards, masks, head, gamma, tau)
    for a, e in RO.episodes(masks):
        a32, r32 = ON.estimate_advantages(rewards[a:e + 1], masks[a:e + 1], head[a:e + 1], gamma, tau)
        # the scan's sums reach thousands of reward units, each step rounded in fp32
        bar = 1e-6 * np.abs(a32).max()
        assert np.abs(adv[a:e + 1] - a32.ravel()).max() <= bar
        assert np.abs(ret[a:e + 1] - r32.ravel()).max() <= bar
