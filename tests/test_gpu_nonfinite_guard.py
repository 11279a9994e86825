"""H100: the non-finite guard (upb_set_nonfinite_guard; tail_gclip's decision in the fused tails, k_apply's branch) on
both models.  Bad inputs are data: a NaN or an infinity written into a parameter, an advantage, a return or an old
log-prob.

  * off (never set, set to 0, set and reset) is bit-identical to a context without the option, slot 19 stays 0;
  * on, a finite step is bit-identical to off at every fused-tail grid size, with the global clip, weight decay and an
    armed KL stop; one launch per fused step;
  * each cause makes the step skip: slot 19 set, nothing else on the device changed, the buffer still shows the
    non-finite entries, and the next clean step is bit for bit the step of a context without the guard;
  * the decision is the host replay of the norm on the step's own buffer, and upb_apply on that buffer takes it too;
  * an absent head cannot make a step bad; the KL stop wins over the guard; the two-group clip modes;
  * PPOUpdater / use_b200_update finish an update with one poisoned sample and equal a hand-stepped update without the
    minibatches that held it."""
import copy
import types

import numpy as np
import pytest
import torch

import gclip_oracle as GO
from cross_path import MLP_GRIDS, SGNN_GRIDS, hlg_case
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.ppo import (GCLIP_NORM_SLOT, KL_SKIP_SLOT, KL_STOP_SLOT, NONFINITE_COUNT_SLOT,
                                         NONFINITE_SLOT, PPOUpdater)
from harness import (Case, assert_same_state, dev, fused_step, heads, nan_buffer, per_tensor_rel, rel,
                     reproducible_states, sgnn_agent, t, two_call_step)

pytestmark = pytest.mark.gpu
NEVER = _lib.CLIP_NEVER
M = 1e-3              # below every step's norm on these cases: every step clips
CAUSES = ["param", "ratio", "adv", "ret"]
BAD = 0               # the poisoned graph: exps != 0 in every case below


def mixed_case(dev, model, seed=5, count=12):
    states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    return Case(dev, model, states, actions, seed, zero_exps=(1,))


def initial_log_probs(c):
    if not hasattr(c, "logp0"):
        c.logp0 = c.engine().forward(c.blob, t(c.flat, c.dev), c.dev_args[0])[1].cpu().numpy()
    return c.logp0


def poisoned(c, cause, g=BAD):
    """The case with graph g's inputs made bad: an old log-prob of -200 under a negative advantage (the ratio
    overflows to inf and the unclipped branch wins), an infinite advantage at a ratio inside the clip range (old
    log-prob = the initial policy's; outside the range the clipped branch wins, the graph's policy gradient is 0 and the
    step is rightly applied), or a NaN return."""
    adv, ret, fixed = c.adv.copy(), c.ret.copy(), c.fixed.copy()
    if cause == "ratio":
        fixed[g], adv[g] = -200.0, -1.0
    elif cause == "adv":
        fixed[g], adv[g] = initial_log_probs(c)[g], np.inf
    elif cause == "ret":
        ret[g] = np.nan
    p = copy.copy(c)
    p.adv, p.ret, p.fixed = adv, ret, fixed
    p.dev_args = (c.dev_args[0], t(adv, c.dev), t(ret, c.dev), t(fixed, c.dev), c.dev_args[4])
    return p


def stats(g, eng):
    return g.cpu().numpy()[eng.stat_offset:]


def device_state(eng, p):
    torch.cuda.synchronize()
    return (p.cpu().numpy().copy(),) + eng.get_opt_state()


def assert_untouched(before, after, what):
    for a, b in zip(before, after):
        assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                              b.view(np.uint32) if b.dtype == np.float32 else b), what


def bad_step(run, eng, c, p, cause, sel=None):
    """One step on bad data (for "param", a NaN in the value head's output bias for the duration of the step).  The
    step must be skipped: slot 19 set, slot 17 clear, non-finite entries in the buffer, the device state untouched."""
    bias = c.layout.slots["val_b2"].offset
    if cause == "param":
        keep = p[bias].clone()
        p[bias] = float("nan")
    before = device_state(eng, p)
    g = run(eng, poisoned(c, cause) if cause != "param" else c, p, sel)
    after = device_state(eng, p)
    buf = g.cpu().numpy()
    st = buf[eng.stat_offset:]
    assert st[NONFINITE_SLOT] == 1 and st[GCLIP_NORM_SLOT] == 0 and st[KL_STOP_SLOT] == 0, (cause, st[:20])
    assert not np.isfinite(buf).all(), cause
    if cause == "param":
        assert st[NONFINITE_COUNT_SLOT] > 0
        p[bias] = keep
    else:
        assert st[NONFINITE_COUNT_SLOT] == 0, (cause, st[:8])
    assert_untouched(before, after, cause)
    return g


# ---- 1. off ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_untouched(dev, model, fused):
    c = mixed_case(dev, model)
    never, zero, reset = c.engine(clip_mode=NEVER), c.engine(clip_mode=NEVER), c.engine(clip_mode=NEVER,
                                                                                        skip_nonfinite=True)
    _lib.check(_lib.lib().upb_set_nonfinite_guard(zero._ctx, 0))
    _lib.check(_lib.lib().upb_set_nonfinite_guard(reset._ctx, 0))
    ps = [t(c.flat, dev).clone() for _ in range(3)]
    run = fused_step if fused else two_call_step
    for k in range(3):
        b = [e.launches for e in (never, zero, reset)]
        gs = [run(e, c, p) for e, p in zip((never, zero, reset), ps)]
        for e, p, g, b0 in zip((zero, reset), ps[1:], gs[1:], b[1:]):
            assert_same_state(never, ps[0], gs[0], e, p, g, (model, k))
            assert e.launches - b0 == never.launches - b[0] == (1 if fused else 3)
        assert stats(gs[0], never)[NONFINITE_SLOT] == 0


# ---- 2. on, finite steps ---------------------------------------------------------------------------------------------
SETTINGS = {"plain": {}, "gclip": dict(max_grad_norm=M), "wd": dict(weight_decay=1e-2),
            "kl_armed": dict(target_kl=1e6), "gclip_wd": dict(max_grad_norm=M, weight_decay=1e-2)}


def check_on_equals_off(c, grid, kw, sels):
    """guard on against guard off on the fused path, bit for bit; the two-call path with the guard on against the fused
    one (the rl-mlp bit for bit, the SGNN within the cross-path bars)."""
    off = c.engine(grid_limit=grid, clip_mode=NEVER, **kw)
    on = c.engine(grid_limit=grid, clip_mode=NEVER, skip_nonfinite=True, **kw)
    two = c.engine(grid_limit=grid, clip_mode=NEVER, skip_nonfinite=True, **kw)
    p0, p1, p2 = (t(c.flat, c.dev).clone() for _ in range(3))
    for k, sel in enumerate(sels):
        assert on.next_step_fused() and off.next_step_fused()
        g0 = fused_step(off, c, p0, sel)
        before = on.launches
        g1 = fused_step(on, c, p1, sel)
        assert on.launches - before == 1
        assert_same_state(off, p0, g0, on, p1, g1, (grid, k))
        assert stats(g1, on)[NONFINITE_SLOT] == 0
        g2 = two_call_step(two, c, p2, sel)
        if c.model == "mlp":
            assert_same_state(on, p1, g1, two, p2, g2, (grid, k, "two-call"))
        else:
            torch.cuda.synchronize()
            worst, where = per_tensor_rel(g1.cpu().numpy()[:PL.NUM_PARAMS], g2.cpu().numpy()[:PL.NUM_PARAMS])
            assert worst < 1e-5, (k, worst, where)
            assert rel(p1.cpu().numpy(), p2.cpu().numpy()) < 1e-6, k
            assert stats(g2, two)[NONFINITE_SLOT] == 0
            assert two.get_opt_state()[2].tolist() == on.get_opt_state()[2].tolist()
    assert on.peer_timeouts() == 0


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_on_is_bit_identical_on_finite_steps(dev, model, setting):
    c = mixed_case(dev, model)
    lu = np.flatnonzero(c.stage == 0)
    check_on_equals_off(c, 0, SETTINGS[setting], [None, lu, None])


@pytest.mark.parametrize("gclip", [False, True])
@pytest.mark.parametrize("grid", MLP_GRIDS)
def test_mlp_on_is_bit_identical_at_every_grid(dev, grid, gclip):
    states, actions = reproducible_states(5, 24)
    c = Case(dev, "mlp", states, actions, 5)
    lu, allg = np.flatnonzero(c.stage == 0), np.arange(c.count)
    check_on_equals_off(c, grid, SETTINGS["gclip" if gclip else "plain"], [allg, lu, allg])


@pytest.mark.parametrize("grid", SGNN_GRIDS)
def test_sgnn_on_is_bit_identical_at_every_grid(dev, grid):
    c = hlg_case(dev, 7)
    check_on_equals_off(c, grid, SETTINGS["gclip" if grid % 2 else "plain"], [None, None, None])


# ---- 3. each cause skips ---------------------------------------------------------------------------------------------
def check_skip_sequence(c, cause, run, grid=0, sel=None, **kw):
    """clean, bad, clean: the bad step changes nothing, and the clean step after it is the step a context without the
    guard takes from the same state."""
    off, on = c.engine(grid_limit=grid, **kw), c.engine(grid_limit=grid, skip_nonfinite=True, **kw)
    p0, p1 = t(c.flat, c.dev).clone(), t(c.flat, c.dev).clone()
    assert_same_state(off, p0, run(off, c, p0, sel), on, p1, run(on, c, p1, sel), (cause, 0))
    before = on.launches
    bad_step(run, on, c, p1, cause, sel)
    launches = on.launches - before
    assert_same_state(off, p0, run(off, c, p0, sel), on, p1, run(on, c, p1, sel), (cause, 2))
    assert on.peer_timeouts() == 0
    return launches


@pytest.mark.parametrize("gclip", [False, True])
@pytest.mark.parametrize("cause", CAUSES)
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_each_cause_skips_the_step(dev, model, fused, cause, gclip):
    c = mixed_case(dev, model)
    kw = dict(max_grad_norm=M) if gclip else {}
    launches = check_skip_sequence(c, cause, fused_step if fused else two_call_step, clip_mode=NEVER, **kw)
    assert launches == (1 if fused else 3)


@pytest.mark.parametrize("grid", SGNN_GRIDS)
def test_sgnn_ratio_overflow_skips_at_every_grid(dev, grid):
    check_skip_sequence(hlg_case(dev, 7), "ratio", fused_step, grid=grid, clip_mode=NEVER)


@pytest.mark.parametrize("grid", MLP_GRIDS)
def test_mlp_ratio_overflow_skips_at_every_grid(dev, grid):
    states, actions = reproducible_states(5, 24)
    check_skip_sequence(Case(dev, "mlp", states, actions, 5), "ratio", fused_step, grid=grid, clip_mode=NEVER)


# ---- 4. the decision is the host replay's ----------------------------------------------------------------------------
def host_bad(buf, eng, model):
    return bool(buf[eng.stat_offset + NONFINITE_COUNT_SLOT] != 0) or not np.isfinite(GO.replay_norm(buf, model))


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_decision_matches_the_host_replay(dev, model, fused):
    """Clean, and one bad graph of either stage through its advantage (that stage's policy head and the encoder) or
    its return (the value head, the encoder and the SGNN's chained attention tensors)."""
    c = mixed_case(dev, model)
    eng = c.engine(clip_mode=NEVER, skip_nonfinite=True)
    p = t(c.flat, dev).clone()
    lu, rd = int(np.flatnonzero(c.stage == 0)[0]), int(np.flatnonzero(c.stage == 1)[1])
    assert c.exps[lu] != 0 and c.exps[rd] != 0
    seen = set()
    for cause, g in [(None, 0), ("adv", lu), ("adv", rd), ("ret", lu), (None, 0), ("ratio", rd)]:
        case = c if cause is None else poisoned(c, cause, g)
        buf = (fused_step if fused else two_call_step)(eng, case, p).cpu().numpy()
        bad = host_bad(buf, eng, model)
        assert bad == (cause is not None) and buf[eng.stat_offset + NONFINITE_SLOT] == float(bad), (cause, g)
        if cause == "adv":
            grads = buf[:c.layout.num_params]
            other = heads(c.layout)[1 if g == lu else 0]
            assert np.isfinite(grads[other]).all() and not np.isfinite(grads[heads(c.layout)[0 if g == lu else 1]]).all()
        if cause == "ret" and model == "sgnn":
            assert not np.isfinite(buf[GO._sgnn_chain()[0]]).all()
        seen.add(bad)
    assert seen == {False, True} and np.isfinite(p.cpu().numpy()).all()
    assert eng.get_opt_state()[2][0] == 2


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_apply_decides_on_the_real_parameter_columns(dev, model):
    """upb_apply on a finite gradient buffer with one infinity planted: in the value head, in one policy head, in a
    chained attention tensor (the SGNN) or in a plain encoder tensor the step is skipped; in a pad word or a statistic
    that is not slot 7 it is not."""
    c = mixed_case(dev, model)
    eng = c.engine(clip_mode=NEVER, skip_nonfinite=True)
    p = t(c.flat, dev).clone()
    clean = eng.ppo_grad(c.blob, p, *c.step_args(), out=nan_buffer(eng))
    s, n, so = c.layout.slots, c.layout.num_params, eng.stat_offset
    plant = {"value head": s["val_w1"].offset + 3, "road head": s["road_w0"].offset + 5, "encoder": s["enc_w"].offset,
             "pad": n, "statistic": so, "count": so + NONFINITE_COUNT_SLOT}
    if model == "sgnn":
        plant["chain"] = s["att_k_w"].offset + 17
        plant["chain bias"] = s["mha_in_b"].offset + 40
    for where, col in plant.items():
        for value in (float("inf"), float("nan")) if where != "count" else (1.0, float("nan")):
            g = clean.clone()
            g[col] = value
            before = device_state(eng, p)
            eng.apply(p, g)
            after = device_state(eng, p)
            buf = g.cpu().numpy()
            want = where not in ("pad", "statistic")
            assert host_bad(buf, eng, model) == want, where
            assert buf[so + NONFINITE_SLOT] == float(want), (where, value)
            if want:
                assert_untouched(before, after, where)
                # the cause gone, the same buffer applies and loses the mark it carried
                g[col] = clean[col]
                eng.apply(p, g)
                assert stats(g, eng)[NONFINITE_SLOT] == 0 and eng.get_opt_state()[2][0] == before[3][0] + 1
            else:
                assert after[3][0] == before[3][0] + 1 and np.isfinite(after[0]).all()


# ---- 5. an absent head -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_absent_head_cannot_make_a_step_bad(dev, model, fused):
    """Land-use graphs only: the road head's gradient is 0, the head is skipped as absent and the step applies.  Then
    the same with a NaN in a road-head parameter, which no land-use graph evaluates: the row stays finite."""
    c = mixed_case(dev, model)
    lu = np.flatnonzero(c.stage == 0)
    road = heads(c.layout)[1]
    eng = c.engine(clip_mode=NEVER, skip_nonfinite=True)
    p = t(c.flat, dev).clone()
    run = fused_step if fused else two_call_step
    for k in range(2):
        buf = run(eng, c, p, lu).cpu().numpy()
        assert buf[eng.stat_offset + NONFINITE_SLOT] == 0 and not buf[road].any()
    assert np.array_equal(p.cpu().numpy()[road], c.flat[road])
    m, v, steps = eng.get_opt_state()
    assert not m[road].any() and not v[road].any() and steps.tolist() == [2, 2, 2, 0]
    poison = c.layout.slots["road_w1"].offset + 4
    p[poison] = float("nan")
    buf = run(eng, c, p, lu).cpu().numpy()
    assert np.isfinite(buf).all() and buf[eng.stat_offset + NONFINITE_SLOT] == 0
    assert eng.get_opt_state()[2].tolist() == [3, 3, 3, 0]
    after = p.cpu().numpy()
    assert np.isnan(after[poison]) and np.isfinite(np.delete(after, poison)).all()
    assert np.array_equal(np.delete(after[road], poison - road.start), np.delete(c.flat[road], poison - road.start))


# ---- 6. upb_apply on the fused step's own buffer ---------------------------------------------------------------------
@pytest.mark.parametrize("gclip", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_apply_on_the_fused_buffer_takes_the_same_decision(dev, model, gclip):
    c = mixed_case(dev, model)
    kw = dict(clip_mode=NEVER, skip_nonfinite=True, **(dict(max_grad_norm=M) if gclip else {}))
    e1, e2 = c.engine(**kw), c.engine(**kw)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for k, cause in enumerate([None, "ratio", None, "ret"]):
        m, v, s = e1.get_opt_state()
        e2.set_opt_state(m, v, s)
        p2.copy_(p1)
        g = fused_step(e1, c if cause is None else poisoned(c, cause), p1)
        g2 = g.clone()
        g2[e2.stat_offset + GCLIP_NORM_SLOT] = 0.0          # written by upb_apply only while the global clip is on
        g2[e2.stat_offset + NONFINITE_SLOT] = 1.0 - float(cause is not None)     # upb_apply must write it either way
        e2.apply(p2, g2)
        torch.cuda.synchronize()
        assert stats(g, e1)[NONFINITE_SLOT] == stats(g2, e2)[NONFINITE_SLOT] == float(cause is not None), k
        assert stats(g, e1)[GCLIP_NORM_SLOT] == stats(g2, e2)[GCLIP_NORM_SLOT]
        assert (stats(g, e1)[GCLIP_NORM_SLOT] > 0) == (gclip and cause is None)
        assert np.array_equal(p1.cpu().numpy(), p2.cpu().numpy()), k
        for a, b in zip(e1.get_opt_state(), e2.get_opt_state()):
            assert np.array_equal(a, b), k
    assert e1.get_opt_state()[2][0] == 2


# ---- 7. the KL stop comes first --------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_kl_stop_on_a_nonfinite_step(dev, model, fused):
    """Old log-probs far from the policy's and a NaN return: the step passes the KL criterion, which is decided first.
    Slot 13 set, slot 19 clear, nothing applied, and the word is set: the next step is skipped with slot 14."""
    c = mixed_case(dev, model)
    eng = c.engine(clip_mode=NEVER, skip_nonfinite=True, target_kl=1e-6)
    p = t(c.flat, dev).clone()
    run = fused_step if fused else two_call_step
    before = device_state(eng, p)
    st = stats(run(eng, poisoned(c, "ret"), p), eng)
    assert st[KL_STOP_SLOT] == 1 and st[NONFINITE_SLOT] == 0 and not np.isfinite(st[0])
    st = stats(run(eng, c, p), eng)
    assert st[KL_SKIP_SLOT] == 1 and st[NONFINITE_SLOT] == 0
    assert_untouched(before, device_state(eng, p), model)


def test_kl_stop_row_that_counts_a_nonfinite_result_still_raises(dev):
    """A NaN in the value head's output bias with finite log-probs far from the old ones: slot 8 is finite, the first
    step stops on the KL criterion (slot 13) before the guard decides, and its row counts every graph in slot 7 with
    slot 19 clear.  Its losses would be logged and are not finite, so the update raises as it does without the guard."""
    spec = synth.COMMUNITIES["small"]
    n, batch = 64, 32
    states, actions = synth.make_states(23, "small", n)
    up = PPOUpdater(PL.default_init(3), spec.max_num_nodes, spec.max_num_edges, dev, opt_num_epochs=1,
                    mini_batch_size=batch, clip_mode=NEVER, skip_nonfinite=True, target_kl=1e-6)
    up.load_states(states, actions, np.ones(n, np.float32))
    _, logp, _ = up.forward_all()
    up.fixed_log_probs = logp - 1.0
    adv, ret, _ = synth.make_ppo_targets(23, n)
    up.advantages, up.returns = t(adv.ravel(), dev), t(ret.ravel(), dev)
    before = up.flat_params()
    up.params[PL.SGNN.slots["val_b2"].offset] = float("nan")
    np.random.seed(NP_SEED)
    with pytest.raises(FloatingPointError):
        up.update_policy()
    st = up._grad_ring[:n // batch, up.engine.stat_offset:].cpu().numpy()
    assert st[0, KL_STOP_SLOT] == 1 and st[0, NONFINITE_COUNT_SLOT] == batch and st[0, NONFINITE_SLOT] == 0
    assert st[1, KL_SKIP_SLOT] == 1
    after = up.flat_params()
    assert np.array_equal(np.delete(after, PL.SGNN.slots["val_b2"].offset),
                          np.delete(before, PL.SGNN.slots["val_b2"].offset))


# ---- 8. the two-group clip modes -------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [_lib.CLIP_REFERENCE, _lib.CLIP_ALWAYS])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_two_group_clip_modes(dev, model, mode):
    """clean (clips: the two-call path inside ppo_step), bad, clean.  CLIP_ALWAYS decides in k_apply before its two-group
    coefficients are used; CLIP_REFERENCE's later steps are fused."""
    c = mixed_case(dev, model)
    launches = check_skip_sequence(c, "adv", fused_step, clip_mode=mode)
    assert launches == (3 if mode == _lib.CLIP_ALWAYS else 1)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_bad_first_step_of_clip_reference(dev, model):
    """The first step of CLIP_REFERENCE takes the two-group clip in k_apply; bad, it is skipped there."""
    c = mixed_case(dev, model)
    eng = c.engine(clip_mode=_lib.CLIP_REFERENCE, skip_nonfinite=True)
    p = t(c.flat, dev).clone()
    before = eng.launches
    bad_step(fused_step, eng, c, p, "ret")
    assert eng.launches - before == 3


# ---- 9. a whole update with one poisoned sample ----------------------------------------------------------------------
T, B, EPOCHS, POISON, NP_SEED = 1024, 64, 2, 336, 11        # POISON: the first step of its episode


def rollout():
    spec = synth.COMMUNITIES["small"]
    states, actions = synth.make_states(21, "small", T)
    rng = np.random.default_rng(21)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[15::16] = 0.0
    exps = np.ones(T, np.float32)
    exps[::37] = 0.0
    exps[POISON] = 1.0
    rewards[POISON] = np.inf          # the backward scan of its episode ends here: an infinite advantage and return
                                      # for this sample alone
    return spec, states, actions, rewards, masks, exps


def hand_stepped(dev, spec, states, actions, rewards, masks, exps):
    """A PPOUpdater without the guard, stepped over the same permutations with the minibatches that hold the poisoned
    sample left out; its parameters and the number of minibatches left out."""
    up = PPOUpdater(PL.default_init(3), spec.max_num_nodes, spec.max_num_edges, dev, opt_num_epochs=EPOCHS,
                    mini_batch_size=B, clip_mode=NEVER)
    up.load_states(states, actions, exps)
    values, up.fixed_log_probs, _ = up.forward_all()
    up.advantages, up.returns = up.engine.gae(t(rewards, dev), t(masks, dev), values, up.gamma, up.tau)
    adv = up.advantages.cpu().numpy()
    assert np.flatnonzero(~np.isfinite(adv)).tolist() == [POISON]
    np.random.seed(NP_SEED)
    order, left_out = np.arange(T), 0
    for _ in range(EPOCHS):
        order = up._epoch_order(order)
        for i in range(T // B):
            mb = order[i * B:(i + 1) * B]
            if POISON in mb:
                left_out += 1
                continue
            ids = t(up.engine.balance_ids(mb, up._cost).astype(np.int32), dev)
            up.minibatch_step(ids, B, int((exps[mb] != 0).sum()))
    return up.flat_params(), left_out


@pytest.mark.parametrize("entry", ["updater", "agent"])
def test_update_survives_one_poisoned_sample(dev, entry):
    from drl_urban_planning_b200.agent import use_b200_update
    spec, states, actions, rewards, masks, exps = rollout()
    want, left_out = hand_stepped(dev, spec, states, actions, rewards, masks, exps)
    assert 1 <= left_out <= EPOCHS and np.isfinite(want).all()
    logged = []
    np.random.seed(NP_SEED)
    if entry == "updater":
        up = PPOUpdater(PL.default_init(3), spec.max_num_nodes, spec.max_num_edges, dev, opt_num_epochs=EPOCHS,
                        mini_batch_size=B, clip_mode=NEVER, skip_nonfinite=True, diagnostics=True)
        out = up.update_params(states, actions, rewards, masks, exps, log_fn=lambda *a: logged.append(a))
        flat = up.flat_params()
        assert out["nonfinite_skips"] == left_out and np.isfinite(out["total_loss"])
        assert np.isfinite(out["total_approx_kl"])
    else:
        ag = sgnn_agent(dev, spec.max_num_nodes, spec.max_num_edges, PL.default_init(3), logged, gamma=1.0, tau=0.0,
                        num_optim_epoch=EPOCHS, mini_batch_size=B)
        ctl = use_b200_update(ag, clip_mode=NEVER, skip_nonfinite=True)
        ag.update_params(types.SimpleNamespace(states=states, actions=actions, rewards=rewards, masks=masks, exps=exps), 0)
        flat = ctl.updater.flat_params()
        assert rel(ag.actor_critic_net.flat_parameters(), flat) == 0
    assert [v for tag, v, s in logged if tag == "diag/nonfinite_skips"] == [float(left_out)]
    assert len([1 for tag, v, s in logged if tag == "loss/loss"]) == EPOCHS * (T // B) - left_out
    assert all(np.isfinite(v) for tag, v, s in logged if tag.startswith("loss/"))
    assert np.array_equal(flat, want)


def test_update_without_the_guard_is_poisoned(dev):
    """skip_nonfinite=False on the same rollout: slot 7 does not count the sample (its value, log-prob and entropy are
    finite), so its step applies the infinite gradient.  The later steps of the epoch then see NaN parameters, slot 7
    counts their graphs, and the update raises after the epoch, with the parameters and moments already lost."""
    spec, states, actions, rewards, masks, exps = rollout()
    np.random.seed(NP_SEED)
    up = PPOUpdater(PL.default_init(3), spec.max_num_nodes, spec.max_num_edges, dev, opt_num_epochs=EPOCHS,
                    mini_batch_size=B, clip_mode=NEVER)
    with pytest.raises(FloatingPointError):
        up.update_params(states, actions, rewards, masks, exps)
    assert not np.isfinite(up.flat_params()).all() and not np.isfinite(up.engine.get_opt_state()[0]).all()
