"""CPU: the KL-adaptive learning rate (desired_kl) -- the argument checks before any CUDA call, the float64 host mirror
(adaptive_lr_oracle) on hand-built statistics rows, the update's host bookkeeping of slot 22 (diag/lr, lr_changes),
and a multi-epoch update of the torch port with RSL-RL's rule against the mirror's decision sequence."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import adaptive_lr_oracle as AO
from drl_urban_planning_b200 import _lib, synth
from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.engine import LR_BOUNDS, Engine, adapt_lr, check_adaptive_lr
from drl_urban_planning_b200.ppo import LR_DECISION_SLOT, PPOUpdater, UpdateLog
from harness import Cfg, reproducible_states
from oracle import torch_port as TP

BAD_KL = [0.0, -0.01, float("nan"), float("inf"), -float("inf"), 1e-50, 1e39, True, np.bool_(False), "0.01", [0.01]]
BAD_BOUNDS = [(0.0, 1e-2), (-1e-5, 1e-2), (1e-2, 1e-5), (1e-5, float("inf")), (float("nan"), 1e-2), (1e-5,),
              (1e-5, 1e-3, 1e-2), 1e-5, (True, 1e-2), ("1e-5", 1e-2), (None, None)]


def no_cuda(monkeypatch):
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("a CUDA call before the argument check"))


@pytest.mark.parametrize("bad", BAD_KL)
def test_bad_desired_kl_is_refused_before_cuda(monkeypatch, bad):
    no_cuda(monkeypatch)
    with pytest.raises(ValueError, match="desired_kl"):
        check_adaptive_lr(bad)
    with pytest.raises(ValueError, match="desired_kl"):
        Engine("cuda:0", 64, 64, desired_kl=bad)
    with pytest.raises(ValueError, match="desired_kl"):
        PPOUpdater(PL.default_init(0), 64, 64, "cuda:0", desired_kl=bad)


@pytest.mark.parametrize("bad", BAD_BOUNDS)
def test_bad_lr_bounds_are_refused_before_cuda(monkeypatch, bad):
    no_cuda(monkeypatch)
    with pytest.raises(ValueError, match="lr_bounds"):
        check_adaptive_lr(0.01, bad)
    with pytest.raises(ValueError, match="lr_bounds"):
        Engine("cuda:0", 64, 64, desired_kl=0.01, lr_bounds=bad)
    with pytest.raises(ValueError, match="lr_bounds"):
        PPOUpdater(PL.default_init(0), 64, 64, "cuda:0", desired_kl=0.01, lr_bounds=bad)


def fake_agent():
    c = Cfg(64, 64)
    c.agent, c.agent_specs = "rl-sgnn", {}
    for k, v in dict(lr=4e-4, eps=1e-5, clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01, gamma=0.99, tau=0.95,
                     num_optim_epoch=1, mini_batch_size=16).items():
        setattr(c, k, v)
    return types.SimpleNamespace(cfg=c, device=torch.device("cuda", 0))


@pytest.mark.parametrize("kw", [dict(desired_kl=0.0), dict(desired_kl=float("nan")), dict(desired_kl=True),
                                dict(desired_kl=0.01, lr_bounds=(1e-2, 1e-5)), dict(desired_kl=0.01, lr_bounds=(0, 1))])
def test_use_b200_update_refuses_before_cuda(monkeypatch, kw):
    from drl_urban_planning_b200.agent import use_b200_update
    no_cuda(monkeypatch)
    with pytest.raises(ValueError, match="desired_kl|lr_bounds"):
        use_b200_update(fake_agent(), **kw)


def test_good_values_pass():
    assert check_adaptive_lr(None) == (0.0, *LR_BOUNDS) == (0.0, 1e-5, 1e-2)
    assert check_adaptive_lr(0.01) == (0.01, 1e-5, 1e-2)
    assert check_adaptive_lr(np.float32(0.02), (1e-4, 1e-4)) == (float(np.float32(0.02)), 1e-4, 1e-4)
    assert check_adaptive_lr(1, [np.float64(1e-6), 3]) == (1.0, 1e-6, 3.0)
    # None is the default bounds on every entry point (Engine and PPOUpdater pass it to check_adaptive_lr as given)
    assert check_adaptive_lr(0.01, None) == (0.01, *LR_BOUNDS) and check_adaptive_lr(None, None) == (0.0, *LR_BOUNDS)


def test_setters_without_a_context():
    L = _lib.lib()
    assert L.upb_set_adaptive_lr(None, 0.01, 1e-5, 1e-2) == -1 and b"set_adaptive_lr" in L.upb_last_error()
    buf = (C.c_double * 1)()
    assert L.upb_get_lr_state(None, buf, 1, None) == -1 and b"get_lr_state" in L.upb_last_error()
    assert L.upb_mlp_set_lr_state(None, buf, 1, None) == -1 and b"mlp_set_lr_state" in L.upb_last_error()


# ---- the mirror on hand-built rows -------------------------------------------------------------------------------------
DKL = 0.01
UP32, DOWN32 = np.float32(DKL / 2), np.float32(2 * DKL)


@pytest.mark.parametrize("s4", [0.0, 1.0, 12.0, 255.0])
def test_decision_at_the_thresholds(s4):
    n = np.float32(max(s4, 1.0))
    down = np.float32(DOWN32 * n)
    up = np.float32(UP32 * n)
    assert AO.decision(down, s4, DKL) == 0                                   # equal to 2 desired_kl: no change
    assert AO.decision(np.nextafter(down, np.float32(np.inf)), s4, DKL) == -1
    assert AO.decision(up, s4, DKL) == 0                                     # equal to desired_kl / 2: no change
    assert AO.decision(np.nextafter(up, np.float32(0)), s4, DKL) == 1
    assert AO.decision(np.float32(1e-30), s4, DKL) == 1
    assert AO.decision(0.0, s4, DKL) == 0                                    # s8 = 0: no change (RSL-RL's kl > 0)
    assert AO.decision(-1e-6, s4, DKL) == 0
    assert AO.decision(float("nan"), s4, DKL) == 0
    assert AO.decision(float("inf"), s4, DKL) == -1


def test_decision_without_an_exps_graph():
    # s4 = 0 and s8 = 0: a minibatch without an exps != 0 graph keeps the lr
    assert AO.decision(0.0, 0.0, DKL) == 0
    assert AO.decision(0.0, float("nan"), DKL) == 0


def test_decision_matches_the_mean_rule_away_from_the_thresholds():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        s4 = float(rng.integers(1, 300))
        kl = float(np.exp(rng.uniform(np.log(1e-4), np.log(1.0))))
        if min(abs(kl - 2 * DKL), abs(kl - DKL / 2)) < 1e-5:
            continue
        s8 = np.float32(kl * s4)
        want = -1 if kl > 2 * DKL else (1 if 0 < kl < DKL / 2 else 0)
        assert AO.decision(s8, s4, DKL) == want


def test_new_lr_in_double_and_saturation():
    lo, hi = 1e-5, 1e-2
    assert adapt_lr(4e-4, -1, lo, hi) == 4e-4 / 1.5
    assert adapt_lr(4e-4, 1, lo, hi) == 4e-4 * 1.5
    assert adapt_lr(4e-4, 0, lo, hi) == 4e-4
    assert adapt_lr(1.2e-5, -1, lo, hi) == lo and adapt_lr(lo, -1, lo, hi) == lo
    assert adapt_lr(8e-3, 1, lo, hi) == hi and adapt_lr(hi, 1, lo, hi) == hi
    # a start outside the bounds: no decision keeps it; a decision moves it and clamps
    assert adapt_lr(5e-2, 0, lo, hi) == 5e-2 and adapt_lr(5e-2, -1, lo, hi) == 5e-2 / 1.5
    assert adapt_lr(5e-2, 1, lo, hi) == hi
    assert adapt_lr(1e-6, 0, lo, hi) == 1e-6 and adapt_lr(1e-6, -1, lo, hi) == lo and adapt_lr(1e-6, 1, lo, hi) == 1.5e-6
    lr = 4e-4
    for _ in range(40):
        lr = adapt_lr(lr, 1, lo, hi)
    assert lr == hi
    for _ in range(40):
        lr = adapt_lr(lr, -1, lo, hi)
    assert lr == lo


def test_per_group_clamping_and_frozen_tensors():
    bounds = (1e-4, 1e-3)
    lrs = [9e-4, 1.2e-4, 5e-3, 5e-5]
    trained = [True, True, True, False]
    assert AO.step(lrs, 1, bounds, trained) == [1e-3, 1.2e-4 * 1.5, 1e-3, 5e-5]
    assert AO.step(lrs, -1, bounds, trained) == [9e-4 / 1.5, 1e-4, 5e-3 / 1.5, 5e-5]
    assert AO.step(lrs, 0, bounds, trained) == lrs


def test_replay_skips_steps_that_apply_nothing():
    rows = [(0.0, 10), (10.0, 10), (1e-4, 10), (10.0, 10), (1e-4, 10)]
    decs, per_step, final = AO.replay([4e-4], rows, DKL, LR_BOUNDS, applied=[True, True, False, False, True])
    assert decs == [0, -1, 0, 0, 1]
    assert per_step[1] == per_step[2] == per_step[3] == [4e-4 / 1.5]
    assert final == [4e-4 / 1.5 * 1.5]


# ---- the update's bookkeeping of slot 22 -------------------------------------------------------------------------------
def test_update_log_logs_diag_lr_on_the_rows_it_logs():
    st = np.zeros((4, 23))
    st[:, 3], st[:, 4] = 16, 12
    st[2, 13] = 1                     # the step that stopped on target_kl; row 3 was skipped after it
    st[3, 14] = 1
    lr = np.array([1.0, 2.0, 2.0, 2.0])
    logged = []
    book = UpdateLog(1, 0.5, 0.01, log_fn=lambda tg, v, s: logged.append((tg, v, s)), kl_stop=True)
    book.epoch(0, st, None, lr)
    got = [(v, s) for tg, v, s in logged if tg == "diag/lr"]
    assert got == [(1.0, 0), (2.0, 1), (2.0, 2)]


# ---- RSL-RL's rule on the torch port, several epochs --------------------------------------------------------------------
def rsl_rl_update(agent, b, actions, adv, ret, fixed, ind, batches, epochs, desired_kl, bounds):
    """RSL-RL's PPO.update with schedule="adaptive": before each optimizer.step the KL at the parameters the step starts
    from decides the new lr of every param group, which that step applies.  Returns (decisions, fp32 row sums)."""
    decs, rows = [], []
    for _ in range(epochs):
        for sel in batches:
            sb = {k: v[sel] for k, v in b.items()}
            idx = ind[sel]
            with torch.no_grad():
                lp, _ = TP.log_prob_entropy(agent.P, sb, actions[sel])
                d = (lp[idx] - fixed[sel][idx]).double()
                kl_terms = torch.expm1(d) - d
                s8, s4 = np.float32(kl_terms.float().sum().item()), float(idx.sum().item())
                kl = kl_terms.mean().item()
            lr = agent.opt.param_groups[0]["lr"]
            if kl > 2 * desired_kl:
                lr, dec = max(bounds[0], lr / 1.5), -1
            elif 0 < kl < desired_kl / 2:
                lr, dec = min(bounds[1], lr * 1.5), 1
            else:
                dec = 0
            for g in agent.opt.param_groups:
                g["lr"] = lr
            agent.step(sb, actions[sel], adv[sel], ret[sel], fixed[sel], idx)
            decs.append(dec)
            rows.append((s8, s4))
    return decs, rows


def test_torch_port_update_against_the_mirror():
    torch.manual_seed(0)
    states, act = reproducible_states(3, 24)
    b = TP.stack_states(states)
    actions = torch.as_tensor(act)
    rng = np.random.default_rng(1)
    adv = torch.as_tensor(rng.normal(size=(24, 1)).astype(np.float32))
    ret = torch.as_tensor(rng.normal(size=(24, 1)).astype(np.float32))
    ind = torch.ones(24, dtype=torch.bool)
    ind[5] = False
    agent = TP.PortAgent(PL.default_init(3), lr=3e-3, reference_clip=False)
    with torch.no_grad():        # old log-probs a little off the current ones: the KL starts small and grows
        lp, _ = TP.log_prob_entropy(agent.P, b, actions)
    assert lp.shape == (24, 1)
    fixed = (lp + torch.as_tensor(rng.normal(0.0, 0.02, size=(24, 1)).astype(np.float32))).float()
    d = (lp - fixed)[ind].double()
    desired_kl, bounds = 3 * float((torch.expm1(d) - d).mean()), (1e-4, 1e-2)
    batches = [np.arange(i * 8, (i + 1) * 8) for i in range(3)]
    decs, rows = rsl_rl_update(agent, b, actions, adv, ret, fixed, ind, batches, 4, desired_kl, bounds)
    mirror, per_step, final = AO.replay([3e-3], rows, desired_kl, bounds)
    assert mirror == decs
    assert final[0] == agent.opt.param_groups[0]["lr"]
    assert len(set(decs)) >= 2, decs             # the run moves the lr
