"""CPU: Adam options (use_b200_update(adam_options=True)): betas, eps, amsgrad and decoupled_weight_decay read from
agent.optimizer's param_groups.  Every refusal comes before the library or the device is touched, the switch off keeps
the old ValueErrors, the float64 oracle (tests/adamw_oracle.py) is torch.optim.Adam / AdamW run in float64, the fp32
replay in the kernels' operation order stays within a few ulps of torch's fp32 step, and the new C entry points
validate without a context."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.agent import B200Update, live_hyperparameters, live_param_groups
from drl_urban_planning_b200.engine import check_adam, check_adam_options
from drl_urban_planning_b200.ppo import PPOUpdater
import adamw_oracle as AO
from test_param_groups import RecordingUpdater, agent, null_engine


# ---- checks before any call --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("betas, eps, match", [
    ((torch.tensor(0.9), 0.999), 1e-8, "not tensors"),
    ((0.9, 0.999), torch.tensor(1e-8), "not tensors"),
    ((-0.1, 0.999), 1e-8, "beta parameter at index 0"),
    ((0.9, 1.0), 1e-8, "beta parameter at index 1"),
    ((0.9, 0.99999999), 1e-8, "beta parameter at index 1"),      # 1.0 once rounded to fp32
    ((0.9, float("nan")), 1e-8, "beta parameter at index 1"),
    ((0.9, 0.999), -1e-8, "epsilon"),
    ((0.9, 0.999), float("inf"), "epsilon"),
    ((0.9, 0.999), float("nan"), "epsilon"),
])
def test_check_adam_refuses(betas, eps, match):
    with pytest.raises(ValueError, match=match):
        check_adam(betas, eps)


def test_check_adam_options_switch():
    assert check_adam_options(True) is True and check_adam_options(0) is False
    for bad in (0.5, 2, "yes", None):
        with pytest.raises(ValueError, match="adam_options"):
            check_adam_options(bad)


def test_engine_checks_adam_before_the_library():
    n = len(PL.SGNN.slots)
    eng = null_engine()
    eng.adam = (0.9, 0.999, 1e-5, False, False)
    with pytest.raises(ValueError, match="beta parameter"):
        eng.set_adam((1.0, 0.999), 1e-8)
    with pytest.raises(ValueError, match="epsilon"):
        eng.set_param_groups([4e-4] * n, [0.0] * n, [True] * n, adam=[(0.9, 0.999, -1.0, False, False)] * n)
    with pytest.raises(ValueError, match="need 32 Adam settings"):
        eng.set_param_groups([4e-4] * n, [0.0] * n, [True] * n, adam=[(0.9, 0.999, 1e-8, False, False)])
    with pytest.raises(_lib.UpbError, match="null context"):         # a valid setting reaches the library
        eng.set_adam((0.8, 0.99), 1e-8, amsgrad=True)
    assert eng.adam == (0.9, 0.999, 1e-5, False, False)
    eng.param_groups = ((4e-4,) * n, (0.0,) * n, (True,) * n)
    with pytest.raises(ValueError, match="parameter groups"):
        eng.set_adam((0.9, 0.999), 1e-8)


def _options_update(ag):
    ctl = B200Update.__new__(B200Update)
    ctl.agent, ctl.updater, ctl.layout = ag, RecordingUpdater(), PL.SGNN
    ctl.param_groups, ctl.adam_options = False, True
    ctl.updater.engine = types.SimpleNamespace(betas=(0.9, 0.999), eps=1e-5)
    ctl.push_weights = lambda: pytest.fail("the update touched the device before checking its optimizer")
    return ctl


def _set_all(key, value):
    return lambda ag: [g.__setitem__(key, value) for g in ag.optimizer.param_groups]


def _sgd(ag):
    ag.optimizer = torch.optim.SGD(ag.actor_critic_net.parameters(), lr=1e-3)


def _two_groups(key, a, b):
    def mutate(ag):
        ps = list(ag.actor_critic_net.parameters())
        ag.optimizer = torch.optim.Adam([dict(params=ps[:4], **{key: a}), dict(params=ps[4:], **{key: b})], lr=1e-3)
    return mutate


REFUSED = [
    (_sgd, "torch.optim.Adam or AdamW, not SGD"),
    (_set_all("maximize", True), "maximize=True"),
    (_set_all("betas", (torch.tensor(0.9), 0.999)), "not tensors"),
    (_set_all("eps", torch.tensor(1e-8)), "not tensors"),
    (_set_all("betas", (0.9, 1.0)), "beta parameter at index 1"),
    (_set_all("eps", -1.0), "epsilon"),
    (_set_all("eps", float("nan")), "epsilon"),
    (_two_groups("betas", (0.9, 0.999), (0.8, 0.999)), "disagree on betas"),
    (_two_groups("eps", 1e-8, 1e-6), "disagree on eps"),
    (_two_groups("amsgrad", False, True), "disagree on amsgrad"),
]


@pytest.mark.parametrize("groups", [False, True])
@pytest.mark.parametrize("mutate, match", REFUSED)
def test_update_params_refuses_before_cuda(mutate, match, groups):
    if groups and "disagree" in match:
        pytest.skip("with param_groups each group keeps its own value")
    ag = agent("sgnn")
    mutate(ag)
    ctl = _options_update(ag)
    ctl.param_groups = groups
    with pytest.raises(ValueError, match=match):
        ctl.update_params(types.SimpleNamespace(), 0)


def test_the_switch_off_keeps_the_old_refusals():
    for key, value in (("betas", (0.8, 0.999)), ("eps", 1e-8), ("amsgrad", True), ("decoupled_weight_decay", True)):
        ag = agent("sgnn")
        _set_all(key, value)(ag)
        with pytest.raises(ValueError, match=f"{key} is"):
            live_hyperparameters(ag, (0.9, 0.999), 1e-5)
    ag = agent("sgnn")
    _sgd(ag)
    assert live_hyperparameters(ag, (0.9, 0.999), 1e-5)["lr"] == 1e-3       # unchanged: another optimizer passes


def test_adamw_and_amsgrad_are_read_live():
    ag = agent("sgnn")
    ag.optimizer = torch.optim.AdamW(ag.actor_critic_net.parameters(), lr=3e-4)
    got = live_hyperparameters(ag, (0.9, 0.999), 1e-5, adam_options=True)
    assert (got["lr"], got["weight_decay"], got["eps"]) == (3e-4, 0.01, 1e-8)
    assert got["betas"] == (0.9, 0.999) and got["decoupled_weight_decay"] is True and got["amsgrad"] is False
    ag.optimizer = torch.optim.Adam(ag.actor_critic_net.parameters(), lr=3e-4, betas=(0.8, 0.99), amsgrad=True)
    got = live_hyperparameters(ag, (0.9, 0.999), 1e-5, adam_options=True)
    assert got["betas"] == (0.8, 0.99) and got["amsgrad"] is True and got["decoupled_weight_decay"] is False
    enc = {id(p) for p in ag.actor_critic_net.actor_net.shared_net.parameters()}
    ps = list(ag.actor_critic_net.parameters())
    ag.optimizer = torch.optim.AdamW([dict(params=[p for p in ps if id(p) in enc], betas=(0.5, 0.9), eps=1e-6),
                                      dict(params=[p for p in ps if id(p) not in enc], amsgrad=True)], lr=1e-3)
    groups = live_param_groups(ag, PL.SGNN, (0.9, 0.999), 1e-5, adam_options=True)
    assert groups[0]["betas"] == (0.5, 0.9) and groups[0]["eps"] == 1e-6 and groups[0]["decoupled_weight_decay"]
    assert groups[1]["amsgrad"] and groups[1]["betas"] == (0.9, 0.999) and groups[1]["eps"] == 1e-8


class RecordingEngine:
    def __init__(self):
        self.lr, self.weight_decay, self.clip_epsilon = 4e-4, 0.0, 0.2
        self.betas, self.eps, self.adam = (0.9, 0.999), 1e-5, (0.9, 0.999, 1e-5, False, False)
        self.param_groups, self.param_group_adam, self.layout = None, None, PL.SGNN
        self.calls = []

    def set_adam(self, betas, eps, amsgrad=False, decoupled_weight_decay=False):
        self.calls.append(("adam", tuple(betas), eps, amsgrad, decoupled_weight_decay))
        self.adam = (*betas, eps, amsgrad, decoupled_weight_decay)

    def set_param_groups(self, lr, wd, trained, adam=None):
        self.calls.append(("groups", lr, wd, trained, adam))
        self.param_groups, self.param_group_adam = (lr, wd, trained), adam


def recording_updater(options=True, groups=False):
    up = PPOUpdater.__new__(PPOUpdater)
    up.engine, up.param_groups, up.adam_options = RecordingEngine(), groups, options
    up.value_pred_coef, up.entropy_coef, up.gamma, up.tau = 0.5, 0.01, 1.0, 0.0
    up.opt_num_epochs, up.mini_batch_size = 4, 256
    return up


def test_updater_issues_one_call_per_change():
    up = recording_updater()
    up.set_hyperparameters(betas=(0.9, 0.999), eps=1e-5)             # the defaults: no call
    assert up.engine.calls == []
    up.set_hyperparameters(eps=1e-8, decoupled_weight_decay=True)
    up.set_hyperparameters(eps=1e-8, decoupled_weight_decay=True)
    assert up.engine.calls == [("adam", (0.9, 0.999), 1e-8, False, True)]
    with pytest.raises(ValueError, match="beta parameter"):
        up.set_hyperparameters(betas=(0.9, 1.5))
    assert len(up.engine.calls) == 1
    with pytest.raises(ValueError, match="adam_options=True"):
        recording_updater(options=False).set_hyperparameters(amsgrad=True)
    grouped = recording_updater(groups=True)
    with pytest.raises(ValueError, match="Adam settings come from set_param_groups"):
        grouped.set_hyperparameters(amsgrad=True)
    names = list(PL.SGNN.slots)
    grouped.set_param_groups([dict(params=names[:20], lr=1e-3, betas=(0.8, 0.99), amsgrad=True),
                              dict(params=names[20:], lr=1e-3, weight_decay=0.01, decoupled_weight_decay=True)])
    adam = grouped.engine.calls[-1][4]
    assert adam[0] == (0.8, 0.99, 1e-5, True, False) and adam[20] == (0.9, 0.999, 1e-5, False, True)
    grouped.set_param_groups([dict(params=names[:20], lr=1e-3, betas=(0.8, 0.99), amsgrad=True),
                              dict(params=names[20:], lr=1e-3, weight_decay=0.01, decoupled_weight_decay=True)])
    assert len(grouped.engine.calls) == 1


def test_c_entry_points_validate_without_a_context():
    L = _lib.lib()
    x = C.c_void_p(0)
    assert L.upb_set_adam(None, 0.9, 0.999, 1e-8, 0, 1) == -1 and b"set_adam" in L.upb_last_error()
    for name in ("upb_set_param_groups_adam", "upb_mlp_set_param_groups_adam"):
        assert getattr(L, name)(None, x, x, x, x, x, x, x, x, 32) == -1
        assert name[4:].encode() in L.upb_last_error()
    assert L.upb_set_weight_decay_double(None, 0.01) == -1 and b"set_weight_decay_double" in L.upb_last_error()
    for name in ("upb_get_amsgrad_state", "upb_mlp_get_amsgrad_state"):        # the existence query too
        assert getattr(L, name)(None, None, 10) == -1
    for name in ("upb_get_amsgrad_state", "upb_mlp_get_amsgrad_state", "upb_set_amsgrad_state",
                 "upb_mlp_set_amsgrad_state"):
        assert getattr(L, name)(None, x, 10) == -1
        assert name[4:].encode() in L.upb_last_error()


# ---- the float64 oracle and the fp32 replay --------------------------------------------------------------------------
SETTINGS = [
    dict(lr=3e-3, weight_decay=0.05, betas=(0.9, 0.999), eps=1e-8, amsgrad=False, decoupled_weight_decay=True),
    dict(lr=1e-3, weight_decay=0.02, betas=(0.8, 0.99), eps=1e-6, amsgrad=True, decoupled_weight_decay=False),
    dict(lr=2e-3, weight_decay=0.0, betas=(0.5, 0.9), eps=1e-5, amsgrad=True, decoupled_weight_decay=True),
    dict(lr=5e-4, weight_decay=0.01, betas=(0.95, 0.9995), eps=1e-7, amsgrad=True, decoupled_weight_decay=True),
]


def _run_torch(dtype, steps=50, seed=3):
    """Four groups of two tensors (one more tensor frozen), AdamW / Adam per group, foreach=False; each step a random
    gradient, with one group skipped (grad None) on every fifth step.  Returns the trajectory of every tensor's
    (param, exp_avg, exp_avg_sq, max_exp_avg_sq, count) and the gradients fed."""
    rng = np.random.default_rng(seed)
    ps = [torch.tensor(rng.normal(0, 1, 7), dtype=dtype, requires_grad=True) for _ in range(9)]
    ps[8].requires_grad_(False)
    groups = [dict(params=ps[2 * k:2 * k + 2], **s) for k, s in enumerate(SETTINGS)]
    opt = torch.optim.Adam(groups, foreach=False)
    trace = []
    for it in range(steps):
        grads = []
        for k, p in enumerate(ps[:8]):
            skip = it % 5 == 4 and k // 2 == it % 4
            g = None if skip else torch.tensor(rng.normal(0, 0.3, 7) * (1 + (it % 3)), dtype=dtype)
            p.grad = g
            grads.append(None if g is None else g.clone())
        snap = lambda: [(p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items()}) for p in ps]
        before = snap()
        opt.step()
        trace.append((grads, before, snap()))
    return trace


def _state(st, n, key, dtype):
    return st[key].numpy() if key in st else np.zeros(n, dtype)


@pytest.mark.parametrize("_", [0])
def test_float64_oracle_matches_torch_adam_and_adamw(_):
    trace = _run_torch(torch.float64)
    for it, (grads, before, after) in enumerate(trace):
        for k in range(9):
            (p0, st0), (p1, st1) = before[k], after[k]
            if k == 8 or grads[k] is None:                # frozen / skipped: nothing moves
                assert torch.equal(p0, p1)
                continue
            s = SETTINGS[k // 2]
            step = int(st1["step"])
            got = AO.adam64(p0.numpy(), grads[k].numpy(), _state(st0, 7, "exp_avg", np.float64),
                            _state(st0, 7, "exp_avg_sq", np.float64), _state(st0, 7, "max_exp_avg_sq", np.float64),
                            step, s["lr"], s["weight_decay"], *s["betas"], s["eps"], s["amsgrad"],
                            s["decoupled_weight_decay"])
            want = (p1.numpy(), st1["exp_avg"].numpy(), st1["exp_avg_sq"].numpy())
            for a, b in zip(got[:3], want):
                np.testing.assert_allclose(a, b, rtol=1e-13, atol=1e-300)
            if s["amsgrad"]:
                np.testing.assert_allclose(got[3], st1["max_exp_avg_sq"].numpy(), rtol=1e-13)


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def test_fp32_replay_stays_with_torch_fp32():
    """Teacher-forced per step: from torch's own fp32 state, the replay's parameter lands within 4 ulps of torch's, and
    its moments and max within 1e-4 of the tensor's largest.  They are not bit-identical because the kernels keep the
    library's arithmetic: moment weights 1.f - fp32(beta) (torch: fp32(1 - beta), 1.3e-5 apart at beta2 = 0.999),
    the bias corrections from fp32(beta), and an unfused lerp."""
    trace = _run_torch(torch.float32)
    for grads, before, after in trace:
        for k in range(8):
            if grads[k] is None:
                continue
            (p0, st0), (p1, st1) = before[k], after[k]
            s = SETTINGS[k // 2]
            got = AO.adam32(p0.numpy(), grads[k].numpy(), _state(st0, 7, "exp_avg", np.float32),
                            _state(st0, 7, "exp_avg_sq", np.float32), _state(st0, 7, "max_exp_avg_sq", np.float32),
                            int(st1["step"]), s["lr"], s["weight_decay"], *s["betas"], s["eps"], s["amsgrad"],
                            s["decoupled_weight_decay"])
            assert _ulps(got[0], p1.numpy()).max() <= 4
            want = [st1["exp_avg"].numpy(), st1["exp_avg_sq"].numpy()]
            if s["amsgrad"]:
                want.append(st1["max_exp_avg_sq"].numpy())
            for a, b in zip(got[1:], want):
                assert np.abs(a.astype(np.float64) - b).max() <= 1e-4 * np.abs(b).max()


def test_fp32_replay_decoupled_decay_is_torchs_mul():
    """With the moments' arithmetic out of the way (g = 0, m = v = 0), the decoupled step is torch's param.mul_ bit for
    bit: p * fp32(1 - lr * wd) with lr * wd formed in double."""
    rng = np.random.default_rng(9)
    p = rng.normal(0, 1, 64).astype(np.float32)
    for lr, wd in ((3e-4, 0.01), (1e-3, 0.1), (0.1, 0.3)):
        t = torch.tensor(p.copy(), requires_grad=True)
        opt = torch.optim.AdamW([t], lr=lr, weight_decay=wd, foreach=False)
        t.grad = torch.zeros(64)
        opt.step()
        got = AO.adam32(p, np.zeros(64, np.float32), np.zeros(64, np.float32), np.zeros(64, np.float32),
                        np.zeros(64, np.float32), 1, lr, wd, 0.9, 0.999, 1e-8, False, True)[0]
        assert np.array_equal(got, t.detach().numpy())


def test_fma32_rounds_once():
    a, b, c = np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12), np.float32(-1)
    assert AO.fma32(a, b, c)[()] == np.float32(2 ** -11 + 2 ** -24)      # the product's low bits survive
    assert AO.fma32(np.float32(2), np.float32(3), np.float32(np.nan)).item() != AO.fma32(1, 1, 1).item()
