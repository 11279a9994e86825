"""CPU: Adam weight decay (cfg `weightdecay`, torch.optim.Adam(weight_decay=...) at urban_planning_agent.py:145-149):
the oracles against golden vectors recorded by the unmodified reference with weight_decay = 1e-2 (the checks of
tests/cross_path.py), the decayed numpy Adam against torch's, the untouched road head of the land-use-only fixture, and
the argument checks of the host layer that need no device."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL
import cross_path as XP
import decay_oracle as DO
from harness import Cfg, load
from oracle import sgnn_numpy as ON

# fixture recorded with decay -> the fixture of the same seeds and states without it
PAIRS = {"small_mixed_wd": "small_mixed", "hlg_wd": "hlg", "mlp_small_wd": "mlp_small",
         "update_small_wd": "update_small"}
SGNN_STEP_FIXTURES = ["small_mixed_wd", "hlg_wd"]


@pytest.mark.parametrize("name", SGNN_STEP_FIXTURES)
def test_torch_port_steps_match_reference_with_weight_decay(name, golden_dir):
    XP.check_torch_port_steps(load(golden_dir, name))


@pytest.mark.parametrize("name", SGNN_STEP_FIXTURES)
def test_numpy_oracle_steps_match_reference_with_weight_decay(name, golden_dir):
    XP.check_numpy_oracle_steps(load(golden_dir, name))


def test_mlp_port_matches_reference_with_weight_decay(golden_dir):
    XP.check_mlp_port(load(golden_dir, "mlp_small_wd"))


def test_torch_port_update_policy_matches_reference_with_weight_decay(golden_dir):
    XP.check_torch_port_update(load(golden_dir, "update_small_wd"))


@pytest.mark.parametrize("name", sorted(PAIRS))
def test_decay_moves_the_trajectory(name, golden_dir):
    XP.check_away_from_shipped(golden_dir, name, PAIRS[name])


def test_skipped_road_head_is_not_decayed(golden_dir):
    """hlg_wd is land-use only: the road head has grad None, so Adam skips it and its weights never decay."""
    z = load(golden_dir, "hlg_wd")
    assert (z["stage"][:, :2].argmax(1) == 0).all()
    road = slice(PL.SLOTS["road_w0"].offset, PL.POLICY_END)
    for k in range(3):
        assert np.array_equal(z["params_after"][k][road], z["params"][road]), k
    lu = slice(PL.SLOTS["lu_w0"].offset, PL.SLOTS["road_w0"].offset)
    assert not np.array_equal(z["params_after"][0][lu], z["params"][lu])


def test_decayed_numpy_adam_step_matches_torch_on_live_entries_only():
    p = np.array([1.0, -2.0, 3.0, 0.5])
    g = np.array([0.0, 0.0, 0.1, 0.0])
    live = np.array([True, True, True, False])
    z = np.zeros(4)
    a, m, v, t = DO.adam_step(p, z, z, z, g, live, 0.1)
    ref = torch.tensor(p[:3], requires_grad=True)
    opt = torch.optim.Adam([ref], lr=4e-4, eps=1e-5, weight_decay=0.1)
    ref.grad = torch.tensor(g[:3])
    opt.step()
    assert np.allclose(a[:3], ref.detach().numpy(), rtol=0, atol=1e-12)
    assert a[3] == p[3] and m[3] == 0.0 and v[3] == 0.0 and t[3] == 0.0
    a0 = ON.adam_step(p, z, z, z, g, live)[0]
    assert np.array_equal(a0, DO.adam_step(p, z, z, z, g, live, 0.0)[0])
    assert a0[0] == p[0]                                      # zero gradient, no decay: no movement


@pytest.mark.parametrize("bad", [-1e-3, float("nan"), float("inf"), -float("inf")])
def test_engine_rejects_invalid_weight_decay(bad):
    """Checked before any device is touched, as torch.optim.Adam raises ValueError("Invalid weight_decay value")."""
    from drl_urban_planning_b200.engine import Engine, check_weight_decay
    with pytest.raises(ValueError, match="weight_decay"):
        check_weight_decay(bad)
    for model in ("sgnn", "mlp"):
        with pytest.raises(ValueError, match="weight_decay"):
            Engine("cuda:0", 64, 64, weight_decay=bad, model=model)


def test_check_weight_decay_accepts_the_adam_range():
    from drl_urban_planning_b200.engine import check_weight_decay
    assert check_weight_decay(0) == 0.0 and check_weight_decay(1e-2) == 1e-2 and check_weight_decay(np.float32(2.0)) == 2.0


@pytest.mark.parametrize("kind", ["rl-sgnn", "rl-mlp"])
@pytest.mark.parametrize("bad", [-1e-2, float("nan")])
def test_b200_update_rejects_invalid_weightdecay(kind, bad):
    """use_b200_update honours cfg.weightdecay for both agents and refuses what torch's Adam refuses, before building a
    CUDA context."""
    import types
    from drl_urban_planning_b200.agent import B200Update
    cfg = Cfg(64, 64)
    cfg.agent, cfg.weightdecay = kind, bad
    agent = types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0))
    with pytest.raises(ValueError, match="weight_decay"):
        B200Update(agent)
