"""CPU: the PPO loss coefficients, clip range and Adam settings away from the shipped values (clip_epsilon 0.2,
value_pred_coef 0.5, entropy_coef 0.01, lr 4e-4, eps 1e-5).

References: golden vectors recorded by the unmodified reference at other settings (tests/golden/*_hp*.npz,
make_golden_hp.py), pinned to the float64 numpy oracle, the torch port and the rl-mlp port (the checks of
tests/cross_path.py); torch.clamp's clip bounds; and UpdateLog's loss composition."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.engine import Engine, check_clip_epsilon, clip_range
from drl_urban_planning_b200.ppo import UpdateLog
import cross_path as XP
from harness import Cfg, load

# fixture at other settings -> the fixture of the same seeds and states recorded at the shipped ones
PAIRS = {"small_mixed_hp": "small_mixed", "small_mixed_hp0": "small_mixed", "mlp_small_hp": "mlp_small",
         "update_small_hp": "update_small"}
EPSILONS = [k / 100 for k in range(1, 100)]
VALUE_HEAD = slice(PL.POLICY_END, PL.NUM_PARAMS)


def fp32_formed(eps):
    """The bounds formed in fp32 from the fp32 epsilon (what the step kernels computed before upb_set_clip_range)."""
    e = np.float32(eps)
    return np.float32(np.float32(1) - e), np.float32(np.float32(1) + e)


def test_torch_clamp_rounds_each_bound_once_from_the_double():
    """The reference's torch.clamp(ratio, 1.0 - eps, 1.0 + eps) on fp32 ratios far outside the range returns
    np.float32(1.0 - eps) and np.float32(1.0 + eps) for every eps = k/100; clip_range gives exactly those."""
    r = torch.tensor([0.0, 1e-3, 0.5 ** 30, 50.0, 1e30], dtype=torch.float32)
    for eps in EPSILONS:
        lo, hi = np.float32(1.0 - eps), np.float32(1.0 + eps)
        got = torch.clamp(r, 1.0 - eps, 1.0 + eps).numpy()
        assert got.dtype == np.float32
        assert np.array_equal(got, [lo, lo, lo, hi, hi]), eps
        assert clip_range(eps) == (float(lo), float(hi)), eps


def test_fp32_formed_clip_range_is_off_for_47_epsilons():
    """Why the kernels must receive the double's bounds: forming them in fp32, even 1 -/+ (double)fp32(eps), misses the
    reference's bound (by one ulp of 1.0 at most) for 47 of the 99 values, though not for the shipped 0.2."""
    off = []
    for eps in EPSILONS:
        want = (np.float32(1.0 - eps), np.float32(1.0 + eps))
        got = fp32_formed(eps)
        e64 = float(np.float32(eps))
        assert (np.float32(1.0 - e64), np.float32(1.0 + e64)) == got, eps       # the tie is already in fp32(eps)
        if got != want:
            assert max(abs(float(g) - float(w)) for g, w in zip(got, want)) <= float(np.spacing(np.float32(1))), eps
            off.append(eps)
    assert len(off) == 47
    assert {0.09, 0.16, 0.18, 0.29, 0.32, 0.33} <= set(off) and 0.2 not in off
    assert fp32_formed(0.18)[1] == np.float32(1.1800001) and np.float32(1.0 + 0.18) == np.float32(1.18)
    assert fp32_formed(0.33)[0] == np.float32(0.66999996) and np.float32(1.0 - 0.33) == np.float32(0.67)


def test_check_clip_epsilon_values():
    assert check_clip_epsilon(0) == 0.0 and check_clip_epsilon(0.2) == 0.2 and check_clip_epsilon(np.float32(1.5)) == 1.5
    for bad in (-1e-3, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="clip_epsilon"):
            check_clip_epsilon(bad)


@pytest.mark.parametrize("bad", [-0.1, float("nan"), float("inf")])
def test_engine_and_updater_reject_a_bad_clip_epsilon_before_any_cuda_call(bad, monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    for model in ("sgnn", "mlp"):
        with pytest.raises(ValueError, match="clip_epsilon"):
            Engine("cuda:0", 16, 16, clip_epsilon=bad, model=model)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError, match="clip_epsilon"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", clip_epsilon=bad)


@pytest.mark.parametrize("kind", ["rl-sgnn", "rl-mlp"])
def test_b200_update_rejects_a_bad_cfg_clip_epsilon(kind):
    import types
    from drl_urban_planning_b200.agent import B200Update
    cfg = Cfg(64, 64)
    cfg.agent, cfg.clip_epsilon = kind, -0.2
    agent = types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0))
    with pytest.raises(ValueError, match="clip_epsilon"):
        B200Update(agent)


def test_set_clip_range_validates_without_a_context():
    import ctypes as C
    L = _lib.lib()
    assert L.upb_set_clip_range(None, C.c_float(0.8), C.c_float(1.2)) == -1
    assert b"set_clip_range" in L.upb_last_error()


# ---- the fixtures (the checks of tests/cross_path.py) ------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PAIRS))
def test_fixture_settings_are_away_from_the_defaults(name, golden_dir):
    XP.check_away_from_shipped(golden_dir, name, PAIRS[name])


@pytest.mark.parametrize("name", ["small_mixed_hp", "small_mixed_hp0"])
def test_numpy_oracle_steps_match_reference_at_other_settings(name, golden_dir):
    XP.check_numpy_oracle_steps(load(golden_dir, name))


@pytest.mark.parametrize("name", ["small_mixed_hp", "small_mixed_hp0"])
def test_torch_port_steps_match_reference_at_other_settings(name, golden_dir):
    XP.check_torch_port_steps(load(golden_dir, name))


def test_zero_value_coefficient_gives_the_value_head_a_zero_gradient(golden_dir):
    """value_pred_coef = 0: the reference's value-head parameters get a zero .grad, not None, so its Adam counts their
    steps (3) while their moments stay zero and they never move; entropy_coef = 0 adds nothing to the policy head."""
    z = load(golden_dir, "small_mixed_hp0")
    assert float(z["value_pred_coef"]) == 0.0 and float(z["entropy_coef"]) == 0.0
    assert bool(z["value_grad_zero"]) and z["value_adam_steps"].tolist() == [3] * len(z["value_adam_steps"])
    for k in range(3):
        assert not z["grads"][k][VALUE_HEAD].any(), k
        assert np.array_equal(z["params_after"][k][VALUE_HEAD], z["params"][VALUE_HEAD]), k
        assert z["losses"][k][0] == pytest.approx(z["losses"][k][2], rel=1e-6)     # loss == surr


def test_mlp_port_matches_reference_at_other_settings(golden_dir):
    XP.check_mlp_port(load(golden_dir, "mlp_small_hp"))


def test_torch_port_update_params_matches_reference_at_other_settings(golden_dir):
    """The reference's whole update_params iteration at gamma 1, tau 0 and non-default coefficients, lr and clip range,
    driven through the torch port."""
    z = load(golden_dir, "update_small_hp")
    assert z["gamma_tau"].tolist() == [float(z["gamma"]), float(z["tau"])] == [1.0, 0.0]
    XP.check_torch_port_update(z)


# ---- UpdateLog's loss composition ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["update_small_hp", "update_small"])
def test_update_log_composes_the_reference_loss_with_the_given_coefficients(name, golden_dir):
    """Statistics rows holding the reference's value / surrogate / entropy losses as sums: UpdateLog logs the reference's
    loss/* tags, its total loss being surr + value_pred_coef * value + entropy_coef * entropy with the coefficients it
    was given, and the reference's loss/total_* tags."""
    z = load(golden_dir, name)
    vc, ec = (float(z["value_pred_coef"]), float(z["entropy_coef"])) if "value_pred_coef" in z else (0.5, 0.01)
    T, B, epochs, _ = (int(x) for x in z["cfg"])
    nb = T // B
    L = z["losses"].reshape(epochs, nb, 4)
    logged = []
    book = UpdateLog(epochs, vc, ec, 0, 0, lambda t, v, s: logged.append((t, v, s)))
    for e in range(epochs):
        st = np.zeros((nb, 16))
        st[:, 3], st[:, 4] = B, B - 1
        st[:, 0], st[:, 1], st[:, 2] = L[e, :, 1] * B, L[e, :, 2] * (B - 1), L[e, :, 3] * (B - 1)
        book.epoch(e, st)
    out = book.finish(False)
    got = np.array([[v for t, v, s in logged if t == k] for k in
                    ("loss/loss", "loss/value_loss", "loss/surr_loss", "loss/entropy_loss")]).T
    assert np.allclose(got, z["losses"], rtol=1e-6, atol=1e-7)
    assert np.allclose([out["total_loss"], out["total_value_loss"], out["total_surr_loss"], out["total_entropy_loss"]],
                       z["totals"], rtol=1e-6, atol=1e-7)
    if name == "update_small_hp":          # the shipped coefficients would not give the reference's loss
        wrong = UpdateLog(epochs, 0.5, 0.01)
        for e in range(epochs):
            st = np.zeros((nb, 16))
            st[:, 3], st[:, 4] = B, B - 1
            st[:, 0], st[:, 1], st[:, 2] = L[e, :, 1] * B, L[e, :, 2] * (B - 1), L[e, :, 3] * (B - 1)
            wrong.epoch(e, st)
        assert not np.isclose(wrong.finish(False)["total_loss"], z["totals"][0], rtol=1e-3)
