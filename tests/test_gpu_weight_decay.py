"""GPU (H100): what Adam weight decay (cfg `weightdecay`; torch.optim.Adam(weight_decay=...) at
urban_planning_agent.py:145-149) does alone: the attention-chain CTA's zero-gradient biases, the absent policy head on
both models, the C entry point's argument check, and the checks of tests/cross_path.py at weight_decay = 1e-2 (the
`wd` row of cross_path.SETTINGS; golden vectors recorded by the unmodified reference with it, tests/golden/*_wd.npz)."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.engine import Engine
import cross_path as XP
import decay_oracle as DO
from harness import Case, assert_same_state, dev, fused_step, heads, load, rel, reproducible_states, t, two_call_step
from oracle import sgnn_numpy as ON

pytestmark = pytest.mark.gpu

WD = 1e-2
SGNN_HEADS = heads(PL.SGNN)


@pytest.fixture(scope="module")
def sgnn_batch(dev):
    return XP.hlg_case(dev, 17)


@pytest.fixture(scope="module")
def mlp_case(dev):
    states, actions = reproducible_states(23, 150)
    stage = np.array([int(s[8].argmax()) for s in states])
    return Case(dev, "mlp", states, actions, 23, zero_exps=(int(np.flatnonzero(stage == 0)[1]),))


# ---- the checks of every optimiser setting -----------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("name", ["small_mixed_wd", "hlg_wd"])
def test_steps_match_reference_golden_with_weight_decay(name, fused, golden_dir, dev):
    """Three steps: the first one clips (k_apply after the clip, on both paths), the next two run through upb_apply or
    through the fused tail.  hlg_wd is land-use only: the road head must stay untouched."""
    XP.check_golden_trajectory(load(golden_dir, name), name, fused, dev)


def test_update_params_matches_reference_with_weight_decay(golden_dir, dev):
    """The reference's whole update_params iteration with decay (update_small_wd) through PPOUpdater(weight_decay=...)."""
    XP.check_update_params(load(golden_dir, "update_small_wd"), dev)


def test_use_b200_update_honours_cfg_weightdecay(golden_dir, dev):
    """use_b200_update on a reference-shaped agent whose cfg sets `weightdecay: 1.0e-2`."""
    XP.check_use_b200_update(load(golden_dir, "update_small_wd"), dev)


@pytest.mark.parametrize("grid", XP.SGNN_GRIDS)
def test_sgnn_fused_step_matches_two_call_path_with_weight_decay(grid, sgnn_batch, dev):
    XP.check_sgnn_fused_against_two_call(sgnn_batch, "wd", grid)


@pytest.mark.parametrize("grid", XP.MLP_GRIDS)
def test_mlp_fused_step_is_bit_identical_to_two_call_path_with_weight_decay(grid, mlp_case, dev):
    XP.check_mlp_fused_bit_identical(mlp_case, "wd", grid)


# ---- the zero-gradient attention biases ------------------------------------------------------------------------------
@pytest.mark.parametrize("wd", [0.0, WD])
def test_zero_gradient_attention_biases_move_by_decay_alone(wd, sgnn_batch, dev):
    """attention_key_layer.bias and the k-slice of in_proj_bias have an exactly zero gradient (softmax shift invariance,
    SURVEY A.7), and the attention-chain CTA writes them.  After one fused step from m = v = 0, Adam sees g = wd * p0 and
    gives p1 = p0 - lr * g / (|g| + eps); at wd = 0 they do not move at all."""
    b = sgnn_batch
    flat = b.flat.copy()
    kb = np.r_[PL.SLOTS["att_k_b"].offset:PL.SLOTS["att_k_b"].offset + 16,
               PL.SLOTS["mha_in_b"].offset + 16:PL.SLOTS["mha_in_b"].offset + 32]
    flat[kb] = np.random.default_rng(5).uniform(-0.5, 0.5, kb.size).astype(np.float32)   # in_proj_bias starts at zero
    eng = b.engine(clip_mode=_lib.CLIP_NEVER, weight_decay=wd)
    params = t(flat, dev).clone()
    before = eng.launches
    grad = eng.ppo_step(b.blob, params, *b.step_args())
    torch.cuda.synchronize()
    assert eng.launches - before == 1
    assert not grad.cpu().numpy()[kb].any()
    p0 = flat[kb].astype(np.float64)
    p1 = params.cpu().numpy()[kb].astype(np.float64)
    if wd == 0.0:
        assert np.array_equal(p1, p0)
        return
    g = np.float32(wd) * flat[kb].astype(np.float64)
    want = p0 - 4e-4 * g / (np.abs(g) + 1e-5)
    assert rel(p1, want) < 1e-6
    assert rel(p1 - p0, want - p0) < 1e-3                    # the step itself, not just the parameter it moved
    m, v, _ = eng.get_opt_state()
    w1, w2 = float(np.float32(1) - np.float32(0.9)), float(np.float32(1) - np.float32(0.999))   # 1 - beta in fp32
    assert rel(m[kb], w1 * g) < 1e-6 and rel(v[kb], w2 * g * g) < 1e-6


# ---- absent policy heads ---------------------------------------------------------------------------------------------
def test_absent_head_is_not_decayed_on_either_path(sgnn_batch, dev):
    """Minibatches mixed -> mixed -> land-use only -> road only -> land-use only -> road only -> mixed with decay: the
    absent head's parameters, moments and step counter stay untouched on the fused and the two-call path, and both follow
    the float64 oracle's trajectory (clip on the first step, decay on the live entries)."""
    b = sgnn_batch
    allg = np.arange(48)                                      # the first 48 graphs keep the float64 oracle quick
    lu, rd = allg[b.stage[allg] == 0], allg[b.stage[allg] == 1]
    plan = [allg, allg, lu, rd, lu, rd, allg]
    ef, et = b.engine(weight_decay=WD), b.engine(weight_decay=WD)
    pf, pt = t(b.flat, dev).clone(), t(b.flat, dev).clone()
    f64, m, v, tt = b.flat.astype(np.float64), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS)
    for step, sel in enumerate(plan):
        sub = [b.states[i] for i in sel]
        ref = ON.ppo_minibatch(f64, sub, b.actions[sel], b.adv[sel], b.ret[sel], b.fixed[sel], b.exps[sel])
        g = ON.clip_groups(ref["grad"]) if step == 0 else ref["grad"]
        f64, m, v, tt = DO.adam_step(f64, m, v, tt, g, ON.live_mask(sub), WD)
        olds = [(p.cpu().numpy(), *e.get_opt_state()) for e, p in ((ef, pf), (et, pt))]
        before = ef.launches
        ef.ppo_step(b.blob, pf, *b.step_args(sel), ids=b.ids(sel))
        gt = et.ppo_grad(b.blob, pt, *b.step_args(sel), ids=b.ids(sel))
        et.apply(pt, gt)
        torch.cuda.synchronize()
        assert (ef.launches - before == 1) == (step > 0), step
        for (e, p), (p_old, m_old, v_old, _) in zip(((ef, pf), (et, pt)), olds):
            p_now = p.cpu().numpy()
            assert rel(p_now, f64) < 1e-5, step
            m_now, v_now, steps = e.get_opt_state()
            for s, sl in SGNN_HEADS.items():
                if not (b.stage[sel] == s).any():
                    assert np.array_equal(p_now[sl], p_old[sl]), (step, s)
                    assert np.array_equal(m_now[sl], m_old[sl]) and np.array_equal(v_now[sl], v_old[sl]), (step, s)
            assert steps.tolist() == [step + 1, tt[0], tt[SGNN_HEADS[0].start], tt[SGNN_HEADS[1].start]], step
    assert steps.tolist() == [7, 7, 5, 5]


def test_mlp_absent_head_is_not_decayed(mlp_case, dev):
    """The rl-mlp counterpart, fused against two-call bit for bit, with the absent head untouched."""
    c = mlp_case
    lu, rd, allg = np.flatnonzero(c.stage == 0), np.flatnonzero(c.stage == 1), np.arange(c.count)
    e1, e2 = c.engine(weight_decay=WD), c.engine(weight_decay=WD)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for step, sel in enumerate([allg, allg, lu, rd, lu, rd, allg]):
        p_before = p2.cpu().numpy()
        m_before, v_before, _ = e2.get_opt_state()
        g1 = two_call_step(e1, c, p1, sel)
        g2 = fused_step(e2, c, p2, sel)
        steps = assert_same_state(e1, p1, g1, e2, p2, g2, step)
        p_now = p2.cpu().numpy()
        m_now, v_now, _ = e2.get_opt_state()
        for s, sl in heads(PL.MLP).items():
            if not (c.stage[sel] == s).any():
                assert np.array_equal(p_now[sl], p_before[sl]), (step, s)
                assert np.array_equal(m_now[sl], m_before[sl]) and np.array_equal(v_now[sl], v_before[sl]), (step, s)
    assert steps.tolist() == [7, 7, 5, 5]


def test_set_weight_decay_rejects_invalid_values(dev):
    """The C entry point itself refuses what torch's Adam refuses."""
    eng = Engine(dev, 64, 64)
    L = _lib.lib()
    for bad in (-1e-3, float("nan"), float("inf")):
        assert L.upb_set_weight_decay(eng._ctx, bad) == -1                      # UPB_ERR_ARG
        assert b"weight_decay" in L.upb_last_error()
    assert L.upb_set_weight_decay(eng._ctx, 0.0) == 0 and L.upb_set_weight_decay(eng._ctx, WD) == 0
