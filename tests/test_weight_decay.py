"""CPU: Adam weight decay (cfg `weightdecay`, torch.optim.Adam(weight_decay=...) at urban_planning_agent.py:145-149) in
the oracles against golden vectors recorded by the unmodified reference with weight_decay = 1e-2, and the argument
checks of the host layer that need no device."""
import math
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL
from fixtures_io import expand_states
import decay_oracle as DO
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP

# fixture recorded with decay -> the fixture of the same seeds and states without it
PAIRS = {"small_mixed_wd": "small_mixed", "hlg_wd": "hlg", "mlp_small_wd": "mlp_small",
         "update_small_wd": "update_small"}
SGNN_STEP_FIXTURES = ["small_mixed_wd", "hlg_wd"]


def rel(a, b, floor=1e-9):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


def load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def wd_of(z):
    wd = float(z["weight_decay"])
    assert wd > 0.0
    return wd


@pytest.mark.parametrize("name", SGNN_STEP_FIXTURES)
def test_torch_port_steps_match_reference_with_weight_decay(name, golden_dir):
    """Three steps, the first one clipped by the reference's clip_policy_grad, then Adam with coupled decay."""
    z = load(golden_dir, name)
    agent = DO.port_agent(z["params"], wd_of(z))
    b = TP.stack_states(expand_states(z))
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    args = (b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
            torch.tensor(z["fixed_log_probs"]), ind)
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < 5e-6, k


@pytest.mark.parametrize("name", SGNN_STEP_FIXTURES)
def test_numpy_oracle_steps_match_reference_with_weight_decay(name, golden_dir):
    """The float64 oracle: first-step clip, then decay on the live entries only, over all three steps."""
    z = load(golden_dir, name)
    wd = wd_of(z)
    states = expand_states(z)
    live = ON.live_mask(states)
    flat = z["params"].astype(np.float64)
    m = v = t = np.zeros(PL.NUM_PARAMS)
    for k in range(3):
        r = ON.ppo_minibatch(flat, states, z["actions"], z["advantages"], z["returns"], z["fixed_log_probs"], z["exps"])
        g = ON.clip_groups(r["grad"]) if k == 0 else r["grad"]
        flat, m, v, t = DO.adam_step(flat, m, v, t, g, live, wd)
        assert rel(flat, z["params_after"][k]) < 5e-6, k
    assert np.array_equal(flat[~live].astype(np.float32), z["params"][~live])


def test_mlp_port_matches_reference_with_weight_decay(golden_dir):
    z = load(golden_dir, "mlp_small_wd")
    b = MP.stack_states(expand_states(z))
    agent = DO.mlp_port_agent(z["params"], wd_of(z))
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    args = (b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
            torch.tensor(z["fixed_log_probs"]), ind)
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < 5e-6, k


def test_torch_port_update_policy_matches_reference_with_weight_decay(golden_dir):
    """The reference's whole update_params iteration with decay, driven through the oracle port the same way."""
    z = load(golden_dir, "update_small_wd")
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    states = expand_states(z)
    agent = DO.port_agent(z["params"], wd_of(z))
    b_all = TP.stack_states(states)
    act = torch.tensor(z["actions"])
    with torch.no_grad():
        values = TP.value(agent.params(), b_all)
    adv, ret = TP.estimate_advantages(torch.tensor(z["rewards"]), torch.tensor(z["masks"]), values,
                                      float(z["gamma_tau"][0]), float(z["gamma_tau"][1]))
    with torch.no_grad():
        fixed, _ = TP.log_prob_entropy(agent.params(), b_all, act)
    exps_t = torch.tensor(z["exps"])
    np.random.seed(np_seed)
    order, losses = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(int(math.floor(T / B))):
            idx = order[i * B:(i + 1) * B]
            b = TP.stack_states([states[j] for j in idx])
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(agent.step(b, act[idx], adv[idx], ret[idx], fixed[idx], ind))
    assert np.allclose(np.array(losses), z["losses"], rtol=2e-5, atol=2e-6)
    assert rel(agent.flat(), z["params_after"]) < 5e-6


@pytest.mark.parametrize("name", sorted(PAIRS))
def test_decay_moves_the_trajectory(name, golden_dir):
    """Each decayed fixture starts where its undecayed counterpart does and ends far outside the parity bars (5e-6 on
    the CPU, 1e-4 per tensor on the GPU), so a path that ignored the decay could not match it."""
    z, base = load(golden_dir, name), load(golden_dir, PAIRS[name])
    assert np.array_equal(z["params"], base["params"]) and np.array_equal(z["actions"], base["actions"])
    a, b = z["params_after"], base["params_after"]
    assert a.shape == b.shape
    assert rel(a.reshape(-1, a.shape[-1])[-1], b.reshape(-1, b.shape[-1])[-1]) > 10 * 1e-4


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
    from test_model_dropin import Cfg
    cfg = Cfg(64, 64)
    cfg.agent, cfg.weightdecay = kind, bad
    agent = types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0))
    with pytest.raises(ValueError, match="weight_decay"):
        B200Update(agent)
