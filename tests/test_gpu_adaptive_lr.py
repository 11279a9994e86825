"""GPU (H100): the KL-adaptive learning rate decided inside the step kernels (upb_set_adaptive_lr), both models.

1. Replay: a run with desired_kl equals, bit for bit, the same steps run with the option off and the mirror's lr
   (adaptive_lr_oracle, on the adaptive run's own statistics rows) set before every step -- parameters, moments, step
   counts, AMSGrad state and every statistics slot but 22 -- on the fused step, on the k_apply path (CLIP_REFERENCE's
   first step, the two-call path with max_grad_norm) and with two parameter groups at different lrs under AdamW.
2. Each decision (up, down, none, saturation at either bound) forced, slot 22 against the mirror.
3. Steps that apply nothing (a target_kl stop and the steps skipped after it, a skip_nonfinite step) keep the lr.
4. End to end: use_b200_update writes the lr back to agent.optimizer, logs diag/lr and survives a checkpoint round trip,
   with parameter groups too (the next update resumes at the restored lrs); update_params reports one lr per group.
5. Off: desired_kl=None is a run without the keyword: launches and outputs."""
import numpy as np
import pytest
import torch

import adaptive_lr_oracle as AO
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.agent import use_b200_update
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from harness import dev, reproducible_states, t
from test_gpu_live_hyperparams import E_CAP, N_CAP, batch, flat_init, make_agent

pytestmark = pytest.mark.gpu

DEC = 22
LR = 3e-3
BOUNDS = (1e-4, 1e-2)


class Case:
    """One minibatch of B graphs whose old log-probs are a little off the log-probs at the start (the KL starts small
    and grows as the steps move the policy), as the KL stop's tests build it."""

    def __init__(self, model, dev, B=96, seed=5):
        if model == "sgnn":
            states, actions = synth.make_states(seed, "small", B)
            self.flat = PL.default_init(seed)
        else:
            states, actions = reproducible_states(seed, B)
            self.flat = PL.MLP.default_init(seed)
        self.model, self.dev, self.B = model, dev, B
        self.layout = PL.MLP if model == "mlp" else PL.SGNN
        self.blob = pack_states(states).to(dev)
        adv, ret, exps = synth.make_ppo_targets(seed, B)
        exps[::5] = 0.0
        probe = Engine(dev, self.blob.n_cap, self.blob.e_cap, model=model)
        _, lp, _ = probe.forward(self.blob, t(self.flat, dev), t(actions, dev))
        probe.close()
        lp = lp.cpu().numpy().reshape(B, 1)
        flp = (lp + np.random.default_rng(seed).normal(0.0, 0.02, (B, 1))).astype(np.float32)
        self.adv = adv
        self.args = [t(x, dev) for x in (actions, adv, ret, flp, exps)]
        self.n_ind = int((exps != 0).sum())

    def engine(self, clip_mode=_lib.CLIP_NEVER, **kw):
        kw.setdefault("lr", LR)
        return Engine(self.dev, self.blob.n_cap, self.blob.e_cap, model=self.model, clip_mode=clip_mode,
                      diagnostics=True, **kw)

    def step(self, eng, p, grad, two_call=False, args=None):
        a = (self.blob, p) + tuple(args or self.args) + (1.0 / self.B, 1.0 / self.n_ind)
        if two_call:
            eng.ppo_grad(*a, out=grad)
            eng.apply(p, grad)
        else:
            eng.ppo_step(*a, out=grad)


def run(case, eng, n, two_call=False, before=None, args_of=None):
    """n steps; before(k) runs ahead of step k; returns the statistics rows and the parameters."""
    p = t(case.flat, case.dev).clone()
    rows = []
    for k in range(n):
        if before is not None:
            before(k)
        g = eng.new_grad_buffer()
        case.step(eng, p, g, two_call, None if args_of is None else args_of(k))
        torch.cuda.synchronize()
        rows.append(g.cpu().numpy()[eng.stat_offset:eng.stat_offset + 28].copy())
    return np.stack(rows), p


def same_optimiser(e1, p1, e2, p2, what):
    torch.cuda.synchronize()
    assert np.array_equal(p1.cpu().numpy(), p2.cpu().numpy()), what
    for a, b in zip(e1.get_opt_state(), e2.get_opt_state()):
        assert np.array_equal(a, b), what
    v1, v2 = e1.get_amsgrad_state(), e2.get_amsgrad_state()
    assert (v1 is None) == (v2 is None) and (v1 is None or np.array_equal(v1, v2)), what
    if e1.param_groups is not None:
        assert np.array_equal(e1.get_tensor_steps(), e2.get_tensor_steps()), what


def two_groups(layout, lr_enc, lr_rest):
    names = list(layout.slots)
    enc = [n for n in names if layout.slots[n].owner == "enc"]
    lrs = [lr_enc if n in enc else lr_rest for n in names]
    return lrs, [1e-2] * len(names), [True] * len(names)


VARIANTS = {
    "fused": dict(),
    "reference_first_step": dict(clip_mode=_lib.CLIP_REFERENCE),
    "two_call_max_grad_norm": dict(max_grad_norm=0.5, two_call=True),
    "groups_adamw": dict(groups=True),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_replay_against_the_option_off(model, variant, dev):
    case = Case(model, dev)
    v = dict(VARIANTS[variant])
    two_call, groups = v.pop("two_call", False), v.pop("groups", False)
    probe = case.engine()
    rows0, _ = run(case, probe, 1)
    probe.close()
    n, dkl = 10, float(3 * rows0[0, 8] / rows0[0, 4])     # the first steps go up, the KL grows as the lr does
    adam = None
    if groups:
        lrs0, wd, trained = two_groups(case.layout, 2e-3, 5e-3)
        adam = [(0.9, 0.999, 1e-5, True, True)] * len(lrs0)         # AdamW with AMSGrad, decoupled decay
    else:
        lrs0, trained = [LR], [True]
    on = case.engine(desired_kl=dkl, lr_bounds=BOUNDS, **v)
    off = case.engine(**v)
    if groups:
        on.set_param_groups(lrs0, wd, trained, adam=adam)
        off.set_param_groups(lrs0, wd, trained, adam=adam)
    rows_on, p_on = run(case, on, n, two_call)
    decs = [AO.decision(r[8], r[4], dkl) for r in rows_on]
    assert rows_on[:, DEC].tolist() == decs, (rows_on[:, DEC], decs)
    assert any(decs), decs
    _, per_step, final = AO.replay(list(lrs0), rows_on[:, [8, 4]], dkl, BOUNDS)

    def before(k):
        if groups:
            off.set_param_groups(per_step[k], wd, trained, adam=adam)
        else:
            off.set_lr(per_step[k][0])
    rows_off, p_off = run(case, off, n, two_call, before)
    assert np.array_equal(np.delete(rows_on, DEC, 1), np.delete(rows_off, DEC, 1))
    assert not rows_off[:, DEC].any()
    same_optimiser(on, p_on, off, p_off, variant)
    assert on.get_lr_state().tolist() == (final if groups else final[:1])


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_each_decision_and_saturation(model, dev):
    case = Case(model, dev)
    probe = case.engine()
    rows, _ = run(case, probe, 1)
    kl0 = rows[0, 8] / rows[0, 4]
    assert kl0 > 0
    for dkl, bounds, want in ((1e3, (1e-4, 1e-2), {1}),            # always up: saturates at lr_max
                              (1e-9, (1e-3, 1e-2), {-1}),          # always down: saturates at lr_min
                              (float(kl0), BOUNDS, {0})):          # the first step inside [dkl / 2, 2 dkl]
        eng = case.engine(desired_kl=dkl, lr_bounds=bounds)
        n = 8 if want != {0} else 1
        rows, _ = run(case, eng, n)
        decs = [AO.decision(r[8], r[4], dkl) for r in rows]
        assert rows[:, DEC].tolist() == decs and set(decs) == want, (dkl, decs)
        _, per_step, final = AO.replay([LR], rows[:, [8, 4]], dkl, bounds)
        assert eng.get_lr_state().tolist() == final
        if want == {1}:
            assert final == [bounds[1]]
        if want == {-1}:
            assert final == [bounds[0]]
        eng.close()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
@pytest.mark.parametrize("two_call", [False, True])
def test_a_target_kl_stop_keeps_the_lr(model, two_call, dev):
    case = Case(model, dev)
    eng = case.engine(desired_kl=1e3, lr_bounds=BOUNDS, target_kl=1e-12)
    rows, _ = run(case, eng, 3, two_call)
    assert rows[0, 13] == 1 and rows[1:, 14].all()
    assert not rows[:, DEC].any()
    assert eng.get_lr_state().tolist() == [LR]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
@pytest.mark.parametrize("two_call", [False, True])
def test_a_skipped_nonfinite_step_keeps_the_lr(model, two_call, dev):
    case = Case(model, dev)
    eng = case.engine(desired_kl=1e3, lr_bounds=BOUNDS, skip_nonfinite=True)
    bad = list(case.args)
    adv = case.adv.copy()
    adv[1] = np.nan
    bad[1] = t(adv, dev)
    rows, _ = run(case, eng, 3, two_call, args_of=lambda k: bad if k == 1 else None)
    assert rows[1, 19] == 1 and rows[1, DEC] == 0
    assert rows[0, DEC] == 1 and rows[2, DEC] == 1
    assert eng.get_lr_state().tolist() == [LR * 1.5 * 1.5]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_end_to_end_write_back_log_and_checkpoint(model, dev):
    flat = flat_init(model, 3)
    logged = []
    ag = make_agent(model, dev, flat, logged, lr=3e-3, num_optim_epoch=2, mini_batch_size=16)
    ctl = use_b200_update(ag, clip_mode=_lib.CLIP_NEVER, desired_kl=1e-3, lr_bounds=(1e-4, 1e-2))
    b = batch(4)
    ag.update_params(b, 0)
    lr_logged = [v for tg, v, _ in logged if tg == "diag/lr"]
    assert len(lr_logged) == 2 * (48 // 16)
    state = ctl.updater.engine.get_lr_state().tolist()
    assert ag.optimizer.param_groups[0]["lr"] == state[0] == lr_logged[-1] == ctl.updater.engine.lr
    assert state[0] != 3e-3
    # a scheduler that multiplies lr composes with the adapted value
    for g in ag.optimizer.param_groups:
        g["lr"] = g["lr"] * 0.5
    ag.update_params(b, 1)
    lr_logged2 = [v for tg, v, _ in logged if tg == "diag/lr"][len(lr_logged):]
    first = AO.step([state[0] * 0.5], 0, (1e-4, 1e-2))
    assert lr_logged2[0] in (AO.step(first, 1, (1e-4, 1e-2))[0], AO.step(first, -1, (1e-4, 1e-2))[0], first[0])
    # checkpoint round trip: a fresh controller restores the lr state and writes it back
    st = ctl.optimizer_state()
    assert st["lr_state"].tolist() == [ag.optimizer.param_groups[0]["lr"]]
    ag2 = make_agent(model, dev, flat, [], lr=3e-3, num_optim_epoch=2, mini_batch_size=16)
    ctl2 = use_b200_update(ag2, clip_mode=_lib.CLIP_NEVER, desired_kl=1e-3, lr_bounds=(1e-4, 1e-2))
    ctl2.load_optimizer_state(st)
    assert ctl2.updater.engine.get_lr_state().tolist() == st["lr_state"].tolist()
    assert ag2.optimizer.param_groups[0]["lr"] == st["lr_state"][0]
    # without the entry the run starts from the optimizer's lr
    ag3 = make_agent(model, dev, flat, [], lr=3e-3, num_optim_epoch=2, mini_batch_size=16)
    ctl3 = use_b200_update(ag3, clip_mode=_lib.CLIP_NEVER, desired_kl=1e-3, lr_bounds=(1e-4, 1e-2))
    ctl3.load_optimizer_state({k: v for k, v in st.items() if k != "lr_state"})
    assert ctl3.updater.engine.get_lr_state().tolist() == [3e-3]


def grouped_agent(model, dev, flat, logged):
    """An agent whose optimizer holds two groups at different lrs (the first six tensors, the rest)."""
    ag = make_agent(model, dev, flat, logged, lr=3e-3, num_optim_epoch=2, mini_batch_size=16)
    ps = list(ag.actor_critic_net.parameters())
    ag.optimizer = torch.optim.Adam([dict(params=ps[:6], lr=2e-3), dict(params=ps[6:], lr=5e-3)], eps=ag.cfg.eps)
    return ag


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_param_groups_checkpoint_resumes_at_the_restored_lrs(model, dev):
    """A fresh controller that loads a param_groups checkpoint writes the restored lrs into its optimizer's groups, and
    its next update is the update the original controller runs from the same state, bit for bit."""
    flat = flat_init(model, 3)
    # a desired_kl no step reaches: every step goes down, so the groups' lrs move and stay apart
    kw = dict(clip_mode=_lib.CLIP_NEVER, param_groups=True, desired_kl=1e-9, lr_bounds=(1e-4, 1e-2))
    log1, log2 = [], []
    ag = grouped_agent(model, dev, flat, log1)
    ctl = use_b200_update(ag, **kw)
    b = batch(4)
    np.random.seed(11)
    ag.update_params(b, 0)
    lrs = [g["lr"] for g in ag.optimizer.param_groups]
    # the update's first step starts at the pre-pass parameters (KL exactly 0: no change), the other five go down
    rows = [(0.0, 1)] + [(1.0, 1)] * 5
    assert lrs == [AO.replay([x], rows, 1e-9, (1e-4, 1e-2))[2][0] for x in (2e-3, 5e-3)]
    st = ctl.optimizer_state()
    state = st["lr_state"].tolist()
    assert len(state) == len(ctl.layout.slots) and [state[0], state[6]] == lrs
    ag2 = grouped_agent(model, dev, flat, log2)
    ag2.actor_critic_net.load_state_dict(ag.actor_critic_net.state_dict())
    ctl2 = use_b200_update(ag2, **kw)
    ctl2.load_optimizer_state(st)
    assert [g["lr"] for g in ag2.optimizer.param_groups] == lrs
    assert ctl2.updater.engine.get_lr_state().tolist() == state
    n1 = len(log1)
    for a in (ag, ag2):
        np.random.seed(12)
        a.update_params(b, 1)
    first = [v for tg, v, _ in log2 if tg == "diag/lr"][0]
    assert first in (AO.step(lrs[:1], d, (1e-4, 1e-2))[0] for d in (-1, 0, 1))      # resumed from the restored lr
    assert [(tg, v) for tg, v, _ in log1[n1:]] == [(tg, v) for tg, v, _ in log2]
    assert np.array_equal(ctl.updater.flat_params(), ctl2.updater.flat_params())
    assert ctl.updater.engine.get_lr_state().tolist() == ctl2.updater.engine.get_lr_state().tolist()
    assert [g["lr"] for g in ag.optimizer.param_groups] == [g["lr"] for g in ag2.optimizer.param_groups]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_update_returns_one_lr_per_group(model, dev):
    """With parameter groups update_params returns each group's lr (a group without a tensor keeps its own), diag/lr is
    the first group's, and a frozen tensor's lr does not move.  lr_bounds=None is the default bounds."""
    from drl_urban_planning_b200.engine import LR_BOUNDS
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat = flat_init(model, 3)
    b = batch(4)
    up = PPOUpdater(flat, N_CAP, E_CAP, dev, lr=3e-3, clip_mode=_lib.CLIP_NEVER, opt_num_epochs=3, mini_batch_size=16,
                    model=model, param_groups=True, desired_kl=1e-3, lr_bounds=None)
    assert up.lr_bounds == LR_BOUNDS
    names = list(up.engine.layout.slots)
    up.set_param_groups([dict(params=names[:6], lr=2e-3), dict(params=[], lr=7e-3),
                         dict(params=names[6:-1], lr=5e-3)])               # the last tensor is frozen
    logged = []
    np.random.seed(13)
    out = up.update_params(b.states, b.actions, b.rewards, b.masks, b.exps,
                           log_fn=lambda tg, v, s: logged.append((tg, v)))
    state = up.engine.get_lr_state().tolist()
    assert out["lr"] == [state[0], 7e-3, state[6]]
    assert state[-1] == 0.0 and len(set(state[:6])) == 1 and len(set(state[6:-1])) == 1
    assert [v for tg, v in logged if tg == "diag/lr"][-1] == out["lr"][0]
    assert out["lr_changes"]["up"] + out["lr_changes"]["down"] >= 1


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_update_returns_lr_and_changes(model, dev):
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat = flat_init(model, 3)
    b = batch(4)
    up = PPOUpdater(flat, N_CAP, E_CAP, dev, lr=3e-3, clip_mode=_lib.CLIP_NEVER, opt_num_epochs=3, mini_batch_size=16,
                    model=model, desired_kl=1e-3, lr_bounds=(1e-4, 1e-2))
    out = up.update_params(b.states, b.actions, b.rewards, b.masks, b.exps)
    assert out["lr"] == up.engine.get_lr_state()[0] == up.engine.lr
    ch = out["lr_changes"]
    assert ch["up"] + ch["down"] >= 1 and ch["up"] + ch["down"] <= 9


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_a_run_without_the_keyword(model, dev):
    flat = flat_init(model, 3)
    b = batch(4)
    from drl_urban_planning_b200.ppo import PPOUpdater
    ups = [PPOUpdater(flat, N_CAP, E_CAP, dev, lr=3e-3, opt_num_epochs=2, mini_batch_size=16, model=model, **kw)
           for kw in (dict(), dict(desired_kl=None))]
    outs = []
    for u in ups:
        np.random.seed(7)                          # the epochs' permutations
        outs.append(u.update_params(b.states, b.actions, b.rewards, b.masks, b.exps))
    assert outs[0].keys() == outs[1].keys() and "lr" not in outs[0]
    assert all(np.array_equal(outs[0][k], outs[1][k]) for k in outs[0])
    assert ups[0].engine.launches == ups[1].engine.launches
    assert np.array_equal(ups[0].flat_params(), ups[1].flat_params())
    assert np.array_equal(ups[0]._grad_ring.cpu().numpy(), ups[1]._grad_ring.cpu().numpy())
    for a, c in zip(ups[0].engine.get_opt_state(), ups[1].engine.get_opt_state()):
        assert np.array_equal(a, c)
