"""GPU (H100): Adam weight decay (cfg `weightdecay`; torch.optim.Adam(weight_decay=...) at urban_planning_agent.py:145-149)
on every optimiser path of both models: k_apply (clipping steps and every two-call step), the SGNN fused tail (per-slice
Adam and the attention-chain CTA) and the rl-mlp fused tail.

References: golden vectors recorded by the unmodified reference with weight_decay = 1e-2 (tests/golden/*_wd.npz), the
float64 oracle with decay, and the two-call path against the fused step at the grid sizes where the tails own their
gradient slices differently."""
import os
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
import decay_oracle as DO
from fixtures_io import expand_states
from oracle import sgnn_numpy as ON
from test_gpu_mlp_step import Case, assert_same_state, fused_step, reproducible_states, two_call_step
from test_gpu_parity import per_tensor_rel, rel, t

pytestmark = pytest.mark.gpu

WD = 1e-2
TOL = 1e-4
SGNN_HEADS = {0: slice(PL.SLOTS["lu_w0"].offset, PL.SLOTS["road_w0"].offset),
              1: slice(PL.SLOTS["road_w0"].offset, PL.POLICY_END)}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need an H100"
    return torch.device("cuda", 0)


def load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    assert float(z["weight_decay"]) == WD
    return z


# ---- golden trajectories of the reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("name", ["small_mixed_wd", "hlg_wd"])
def test_steps_match_reference_golden_with_weight_decay(name, fused, golden_dir, dev):
    """Three steps: the first one clips (k_apply after the clip, on both paths), the next two run through upb_apply or
    through the fused tail.  hlg_wd is land-use only: the road head must stay untouched."""
    z = load(golden_dir, name)
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE, weight_decay=WD)
    params = t(z["params"], dev).clone()
    n_ind = int((z["exps"] != 0).sum())
    args = (t(z["actions"], dev), t(z["advantages"], dev), t(z["returns"], dev), t(z["fixed_log_probs"], dev),
            t(z["exps"], dev))
    for k in range(3):
        before = eng.launches
        if fused:
            grad = eng.ppo_step(blob, params, *args, 1.0 / B, 1.0 / n_ind)
        else:
            grad = eng.ppo_grad(blob, params, *args, 1.0 / B, 1.0 / n_ind)
            eng.apply(params, grad)
        torch.cuda.synchronize()
        if fused:
            assert (eng.launches - before == 1) == (k > 0), k
        assert np.allclose(eng.read_losses(grad), z["losses"][k], rtol=1e-4, atol=1e-5), k
        worst, where = per_tensor_rel(grad.cpu().numpy()[:PL.NUM_PARAMS], z["grads"][k])     # the undecayed gradient
        assert worst < TOL, (k, worst, where)
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k      # test_gpu_parity.py's bar
    if name == "hlg_wd":
        road = SGNN_HEADS[1]
        assert np.array_equal(params.cpu().numpy()[road], z["params"][road])
        m, v, steps = eng.get_opt_state()
        assert not m[road].any() and not v[road].any() and steps.tolist() == [3, 3, 3, 0]


def update_losses(logged):
    return np.array([[v for tag, v, s in logged if tag == k] for k in
                     ("loss/loss", "loss/value_loss", "loss/surr_loss", "loss/entropy_loss")]).T


def test_update_params_matches_reference_with_weight_decay(golden_dir, dev):
    """The reference's whole update_params iteration with decay (update_small_wd) through PPOUpdater(weight_decay=...)."""
    from drl_urban_planning_b200.ppo import PPOUpdater
    z = load(golden_dir, "update_small_wd")
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    states = expand_states(z)
    up = PPOUpdater(z["params"], int(z["n_cap"]), int(z["e_cap"]), dev, gamma=float(z["gamma_tau"][0]),
                    tau=float(z["gamma_tau"][1]), opt_num_epochs=epochs, mini_batch_size=B,
                    clip_mode=_lib.CLIP_REFERENCE, weight_decay=WD)
    assert up.engine.weight_decay == WD
    logged = []
    np.random.seed(np_seed)
    out = up.update_params(states, z["actions"], z["rewards"], z["masks"], z["exps"],
                           log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    got = update_losses(logged)
    assert got.shape == z["losses"].shape == (epochs * (T // B), 4)
    assert np.allclose(got, z["losses"], rtol=2e-4, atol=2e-5), np.abs(got - z["losses"]).max()
    totals = np.array([out["total_loss"], out["total_value_loss"], out["total_surr_loss"], out["total_entropy_loss"]])
    assert np.allclose(totals, z["totals"], rtol=2e-4, atol=2e-5)
    assert rel(up.flat_params(), z["params_after"]) < 2e-5


def test_use_b200_update_honours_cfg_weightdecay(golden_dir, dev):
    """use_b200_update on a reference-shaped agent whose cfg sets `weightdecay: 1.0e-2` runs and reproduces the
    reference's update_params with that cfg."""
    from drl_urban_planning_b200.agent import use_b200_update
    from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
    from test_model_dropin import Agent, Cfg
    z = load(golden_dir, "update_small_wd")
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    cfg = Cfg(int(z["n_cap"]), int(z["e_cap"]))
    cfg.lr, cfg.eps, cfg.clip_epsilon, cfg.value_pred_coef, cfg.entropy_coef = 4e-4, 1e-5, 0.2, 0.5, 0.01
    cfg.gamma, cfg.tau = float(z["gamma_tau"][0]), float(z["gamma_tau"][1])
    cfg.num_optim_epoch, cfg.mini_batch_size, cfg.weightdecay = epochs, B, WD
    cfg.agent_specs, cfg.agent = {}, "rl-sgnn"
    ag = Agent()
    ag.cfg, ag.device, ag.loss_iter = cfg, dev, 0
    logged = []
    ag.tb_logger = types.SimpleNamespace(add_scalar=lambda tag, v, s: logged.append((tag, v, s)))
    torch.manual_seed(0)
    p, v = create_sgnn_model(cfg, ag)
    ag.policy_net, ag.value_net, ag.actor_critic_net = p, v, ActorCritic(p, v)
    ag.actor_critic_net.load_flat_parameters(z["params"])
    ctl = use_b200_update(ag)
    assert ctl.updater.engine.weight_decay == WD
    batch = types.SimpleNamespace(states=expand_states(z), actions=z["actions"], rewards=z["rewards"], masks=z["masks"],
                                  exps=z["exps"])
    np.random.seed(np_seed)
    ag.update_params(batch, 0)
    assert np.allclose(update_losses(logged), z["losses"], rtol=2e-4, atol=2e-5)
    assert rel(ctl.updater.flat_params(), z["params_after"]) < 2e-5
    assert rel(ag.actor_critic_net.flat_parameters(), z["params_after"]) < 2e-5       # written back into the modules


# ---- fused tail vs two-call path -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sgnn_batch(dev):
    """140 hlg-sized graphs of both stages (one in three a road graph): more than the 132 CTAs of a full grid."""
    count = 140
    states, actions = synth.make_states(17, "hlg", count, stages=[int(i % 3 == 1) for i in range(count)])
    adv, ret, exps = synth.make_ppo_targets(17, count)
    exps[7] = 0.0
    fixed = np.random.default_rng(17).normal(-3.0, 0.3, size=(count, 1)).astype(np.float32)
    blob = pack_states(states).to(dev)
    return types.SimpleNamespace(states=states, count=count, blob=blob, stage=blob.info[:, 3].astype(np.int64),
                                 args=tuple(t(x, dev) for x in (actions, adv, ret, fixed, exps)), exps=exps,
                                 actions=actions, adv=adv, ret=ret, fixed=fixed, flat=PL.default_init(17))


@pytest.mark.parametrize("grid", [1, 2, 3, 57, 113, 114, 115, 132])
def test_sgnn_fused_step_matches_two_call_path_with_weight_decay(grid, sgnn_batch, dev):
    """4 steps (the first clips and takes the two-call path inside upb_ppo_step) at grids where one CTA owns all 114
    slices, several reload later slices, one each with idle CTAs, and the full grid; tolerances of
    test_fused_step_matches_two_call_path.  One launch per fused step."""
    b = sgnn_batch
    n_ind = int((b.exps != 0).sum())
    e1 = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid, weight_decay=WD)
    e2 = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid, weight_decay=WD)
    e0 = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid)                 # undecayed, for contrast
    p1, p2, p0 = (t(b.flat, dev).clone() for _ in range(3))
    for step in range(4):
        g1 = e1.ppo_grad(b.blob, p1, *b.args, 1.0 / b.count, 1.0 / n_ind)
        e1.apply(p1, g1)
        before = e2.launches
        g2 = e2.ppo_step(b.blob, p2, *b.args, 1.0 / b.count, 1.0 / n_ind)
        e0.ppo_step(b.blob, p0, *b.args, 1.0 / b.count, 1.0 / n_ind)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (step > 0), step
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (step, worst, where)
        assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, step
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    assert s1.tolist() == s2.tolist() == [4, 4, 4, 4]
    assert rel(m2, m1) < 1e-5 and rel(v2, v1) < 1e-5
    assert rel(p2.cpu().numpy(), p0.cpu().numpy()) > 1e-3                        # the decay did move the trajectory


@pytest.fixture(scope="module")
def mlp_case(dev):
    states, actions = reproducible_states(23, 150)
    stage = np.array([int(s[8].argmax()) for s in states])
    return Case(dev, states, actions, 23, zero_exps=(int(np.flatnonzero(stage == 0)[1]),))


@pytest.mark.parametrize("grid", [1, 2, 3, 80, 81, 82, 132])
def test_mlp_fused_step_is_bit_identical_to_two_call_path_with_weight_decay(grid, mlp_case, dev):
    """Decay in mlp_fused_tail and in k_apply is the same fused multiply-add on the same old parameter, so on
    reproducible batches the two paths stay bit-identical: parameters, gradient buffer, moments, step counters."""
    c = mlp_case
    lu, allg = np.flatnonzero(c.stage == 0), np.arange(c.count)
    e1 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid, weight_decay=WD)
    e2 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid, weight_decay=WD)
    e0 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid)
    p1, p2, p0 = (t(c.flat, dev).clone() for _ in range(3))
    for step, sel in enumerate([allg, allg, lu, allg]):
        g1 = two_call_step(e1, c, p1, sel)
        before = e2.launches
        g2 = fused_step(e2, c, p2, sel)
        fused_step(e0, c, p0, sel)
        assert e2.launches - before == (3 if step == 0 else 1), step
        steps = assert_same_state(e1, p1, g1, e2, p2, g2, (grid, step))
    assert steps.tolist() == [4, 4, 4, 3]
    assert rel(p2.cpu().numpy(), p0.cpu().numpy()) > 1e-3


# ---- the zero-gradient attention biases --------------------------------------------------------------------------------
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
    eng = Engine(dev, b.blob.n_cap, b.blob.e_cap, clip_mode=_lib.CLIP_NEVER, weight_decay=wd)
    params = t(flat, dev).clone()
    before = eng.launches
    grad = eng.ppo_step(b.blob, params, *b.args, 1.0 / b.count, 1.0 / int((b.exps != 0).sum()))
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
    ef = Engine(dev, b.blob.n_cap, b.blob.e_cap, weight_decay=WD)
    et = Engine(dev, b.blob.n_cap, b.blob.e_cap, weight_decay=WD)
    pf, pt = t(b.flat, dev).clone(), t(b.flat, dev).clone()
    f64, m, v, tt = b.flat.astype(np.float64), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS)
    for step, sel in enumerate(plan):
        sub = [b.states[i] for i in sel]
        ref = ON.ppo_minibatch(f64, sub, b.actions[sel], b.adv[sel], b.ret[sel], b.fixed[sel], b.exps[sel])
        g = ON.clip_groups(ref["grad"]) if step == 0 else ref["grad"]
        f64, m, v, tt = DO.adam_step(f64, m, v, tt, g, ON.live_mask(sub), WD)
        ids = t(sel.astype(np.int32), dev)
        args = b.args + (1.0 / len(sel), 1.0 / max(int((b.exps[sel] != 0).sum()), 1))
        olds = [(p.cpu().numpy(), *e.get_opt_state()) for e, p in ((ef, pf), (et, pt))]
        before = ef.launches
        ef.ppo_step(b.blob, pf, *args, ids=ids)
        gt = et.ppo_grad(b.blob, pt, *args, ids=ids)
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
    from test_gpu_mlp_step import HEADS
    c = mlp_case
    lu, rd, allg = np.flatnonzero(c.stage == 0), np.flatnonzero(c.stage == 1), np.arange(c.count)
    e1 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", weight_decay=WD)
    e2 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", weight_decay=WD)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for step, sel in enumerate([allg, allg, lu, rd, lu, rd, allg]):
        p_before = p2.cpu().numpy()
        m_before, v_before, _ = e2.get_opt_state()
        g1 = two_call_step(e1, c, p1, sel)
        g2 = fused_step(e2, c, p2, sel)
        steps = assert_same_state(e1, p1, g1, e2, p2, g2, step)
        p_now = p2.cpu().numpy()
        m_now, v_now, _ = e2.get_opt_state()
        for s, sl in HEADS.items():
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
