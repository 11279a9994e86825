"""H100: the global gradient-norm clip (upb_set_max_grad_norm; tail_gclip in the fused tails, k_apply's branch) on
both models.

  * off: a context that set the option and turned it off again is bit-identical to one that never set it;
  * both paths reproduce the reference's clip_grad_norm_ fixtures, one launch per fused step;
  * slot 17 is, bit for bit, the host replay of the defined order on the step's own reduced gradient, and upb_apply on
    the fused step's own buffer from the same Adam state reproduces its parameters and moments: the in-kernel coef is
    k_apply's;
  * fused against two-call at every fused-tail grid size (the rl-mlp bit for bit), no peer give-ups;
  * a max_grad_norm above the norm is CLIP_NEVER, decay after the clip, an absent head untouched, the KL stop;
  * PPOUpdater / use_b200_update against a torch-port replay with clip_grad_norm_."""
import types

import numpy as np
import pytest
import torch

import gclip_oracle as GO
import ppo_oracle as PPO
from cross_path import MLP_GRIDS, SGNN_GRIDS, TOL, hlg_case
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from drl_urban_planning_b200.ppo import GCLIP_NORM_SLOT, KL_STOP_SLOT, PPOUpdater
from fixtures_io import expand_states
from harness import (Case, assert_same_state, dev, fused_step, heads, load, per_tensor_rel, rel, reproducible_states,
                     sgnn_agent, t, two_call_step, update_losses)
from oracle import torch_port as TP
from test_value_clip import GOLDEN

pytestmark = pytest.mark.gpu
NEVER = _lib.CLIP_NEVER
M = 1e-3              # below every step's norm on these cases: every step clips


def mixed_case(dev, model, seed=5, count=12):
    states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    return Case(dev, model, states, actions, seed, zero_exps=(1,))


def norm_of(g, eng):
    return g.cpu().numpy()[eng.stat_offset + GCLIP_NORM_SLOT]


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_bit_identical(dev, model, fused):
    c = mixed_case(dev, model)
    never, off = c.engine(clip_mode=NEVER), c.engine(clip_mode=NEVER, max_grad_norm=0.5)
    _lib.check(_lib.lib().upb_set_max_grad_norm(off._ctx, 0.0))
    p0, p1 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    run = fused_step if fused else two_call_step
    for k in range(3):
        b0, b1 = never.launches, off.launches
        g0, g1 = run(never, c, p0), run(off, c, p1)
        assert_same_state(never, p0, g0, off, p1, g1, (model, k))
        assert never.launches - b0 == off.launches - b1 == (1 if fused else 3)
        assert norm_of(g0, never) == 0


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("name", ["small_mixed_gclip", "mlp_small_gclip"])
def test_golden_trajectory(dev, name, fused):
    z = load(GOLDEN, name)
    mlp = name.startswith("mlp")
    layout = PL.MLP if mlp else PL.SGNN
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=NEVER, model="mlp" if mlp else "sgnn",
                 max_grad_norm=float(z["max_grad_norm"]))
    params = t(z["params"], dev).clone()
    n_ind = int((z["exps"] != 0).sum())
    args = tuple(t(z[k], dev) for k in ("actions", "advantages", "returns", "fixed_log_probs", "exps"))
    for k in range(3):
        assert eng.next_step_fused()
        before = eng.launches
        if fused:
            grad = eng.ppo_step(blob, params, *args, 1.0 / B, 1.0 / n_ind)
        else:
            grad = eng.ppo_grad(blob, params, *args, 1.0 / B, 1.0 / n_ind)
            eng.apply(params, grad)
        torch.cuda.synchronize()
        assert eng.launches - before == (1 if fused else 3)
        assert np.allclose(eng.read_losses(grad), z["losses"][k], rtol=1e-4, atol=1e-5)
        worst, where = per_tensor_rel(grad.cpu().numpy()[:layout.num_params], z["grads"][k], layout)
        # the value head's one-element bias is the sum of the graphs' value seeds, which cancel: its relative error is
        # that of a difference (2.2e-4 on both paths at the SGNN fixture's last step); every other tensor keeps TOL
        g = grad.cpu().numpy()[:layout.num_params].copy()
        bias = layout.slots["val_b2"].offset
        g[bias] = z["grads"][k][bias]
        assert per_tensor_rel(g, z["grads"][k], layout)[0] < TOL, k
        assert worst < 5e-4, (k, worst, where)
        assert rel(grad.cpu().numpy()[:layout.num_params], z["grads"][k]) < TOL, k
        assert np.isclose(norm_of(grad, eng), z["grad_norms"][k], rtol=1e-4)
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k


@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_norm_slot_and_coef_are_k_applys(dev, model, fused, wd):
    """Slot 17 equals the host replay of the defined order on the step's own buffer; apply on that buffer, from the
    same prior Adam state, reproduces the step's parameters and moments bit for bit; the decay comes after the clip."""
    c = mixed_case(dev, model)
    e1, e2 = c.engine(clip_mode=NEVER, max_grad_norm=M, weight_decay=wd), c.engine(clip_mode=NEVER, max_grad_norm=M,
                                                                                   weight_decay=wd)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for k in range(3):
        m, v, s = e1.get_opt_state()
        e2.set_opt_state(m, v, s)
        p2.copy_(p1)
        before = p1.cpu().numpy().astype(np.float64)
        g = (fused_step if fused else two_call_step)(e1, c, p1)
        torch.cuda.synchronize()
        buf = g.cpu().numpy()
        norm = GO.replay_norm(buf, model)
        assert norm == norm_of(g, e1), (k, norm, norm_of(g, e1))
        assert GO.coef(norm, M) < 1
        g2 = g.clone()
        g2[e2.stat_offset + GCLIP_NORM_SLOT] = 0.0
        e2.apply(p2, g2)
        torch.cuda.synchronize()
        assert np.array_equal(p1.cpu().numpy(), p2.cpu().numpy()), k
        for a, b in zip(e1.get_opt_state(), e2.get_opt_state()):
            assert np.array_equal(a, b), k
        if k == 0:
            # from zero moments m = 0.1 g: the clipped gradient plus the decay term of the old parameter (the decay
            # before the clip would give a different m wherever wd != 0)
            m1 = e1.get_opt_state()[0].astype(np.float64)
            coef = float(GO.coef(norm, M))
            want = 0.1 * (buf[:c.layout.num_params].astype(np.float64) * coef + wd * before)
            assert rel(m1, want) < 1e-5
            if wd:
                dec = buf[:c.layout.num_params].astype(np.float64) + wd * before
                assert rel(m1, 0.1 * dec * min(M / np.linalg.norm(dec), 1.0)) > 1e-2


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_unreached_max_norm_is_clip_never(dev, model):
    c = mixed_case(dev, model)
    e0, e1 = c.engine(clip_mode=NEVER), c.engine(clip_mode=NEVER, max_grad_norm=1e6)
    p0, p1 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for k in range(3):
        g0, g1 = fused_step(e0, c, p0), fused_step(e1, c, p1)
        torch.cuda.synchronize()
        assert norm_of(g1, e1) > 0
        g1[e1.stat_offset + GCLIP_NORM_SLOT] = 0.0
        assert_same_state(e0, p0, g0, e1, p1, g1, (model, k))


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_land_use_only_batch_leaves_the_road_head(dev, model):
    c = mixed_case(dev, model)
    lu = np.flatnonzero(c.stage == 0)
    eng = c.engine(clip_mode=NEVER, max_grad_norm=M)
    p = t(c.flat, dev).clone()
    road = heads(c.layout)[1]
    for k in range(2):
        fused_step(eng, c, p, lu)
    torch.cuda.synchronize()
    assert np.array_equal(p.cpu().numpy()[road], c.flat[road])
    m, v, steps = eng.get_opt_state()
    assert not m[road].any() and not v[road].any() and steps.tolist() == [2, 2, 2, 0]


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_kl_stop_step_applies_nothing(dev, model, fused):
    """Old log-probs far from the policy's: the first step passes the KL criterion.  It writes slot 13, leaves slot 17
    at 0 and changes no parameter, moment or counter."""
    c = mixed_case(dev, model)
    eng = c.engine(clip_mode=NEVER, max_grad_norm=M, target_kl=1e-6)
    p = t(c.flat, dev).clone()
    g = (fused_step if fused else two_call_step)(eng, c, p)
    torch.cuda.synchronize()
    st = g.cpu().numpy()[eng.stat_offset:]
    assert st[KL_STOP_SLOT] == 1 and st[GCLIP_NORM_SLOT] == 0
    assert np.array_equal(p.cpu().numpy(), c.flat)
    m, v, steps = eng.get_opt_state()
    assert not m.any() and not v.any() and steps.tolist() == [0, 0, 0, 0]


@pytest.mark.parametrize("grid", MLP_GRIDS)
def test_mlp_fused_bit_identical_at_every_grid(dev, grid):
    states, actions = reproducible_states(5, 24)
    c = Case(dev, "mlp", states, actions, 5)
    lu, allg = np.flatnonzero(c.stage == 0), np.arange(c.count)
    e1 = c.engine(grid_limit=grid, clip_mode=NEVER, max_grad_norm=M)
    e2 = c.engine(grid_limit=grid, clip_mode=NEVER, max_grad_norm=M)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for step, sel in enumerate([allg, allg, lu, allg]):
        assert e2.next_step_fused()
        g1 = two_call_step(e1, c, p1, sel)
        before = e2.launches
        g2 = fused_step(e2, c, p2, sel)
        assert e2.launches - before == 1
        assert_same_state(e1, p1, g1, e2, p2, g2, (grid, step))
    assert e2.peer_timeouts() == 0


@pytest.mark.parametrize("grid", SGNN_GRIDS)
def test_sgnn_fused_against_two_call_at_every_grid(dev, grid):
    c = hlg_case(dev, 7)
    e1 = c.engine(grid_limit=grid, clip_mode=NEVER, max_grad_norm=M)
    e2 = c.engine(grid_limit=grid, clip_mode=NEVER, max_grad_norm=M)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for step in range(4):
        g1 = two_call_step(e1, c, p1)
        before = e2.launches
        g2 = fused_step(e2, c, p2)
        torch.cuda.synchronize()
        assert e2.launches - before == 1
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (step, worst, where)
        n1, n2 = norm_of(g1, e1), norm_of(g2, e2)
        assert n2 == GO.replay_norm(g2.cpu().numpy(), "sgnn") and np.isclose(n1, n2, rtol=1e-5)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, step
    assert e2.peer_timeouts() == 0


def port_replay(z, m, B, epochs, np_seed):
    """The reference's update_params iteration at the shipped settings with clip_grad_norm_(all, m) on every step."""
    import math
    T = len(z["exps"])
    agent = PPO.PortAgent(z["params"], max_grad_norm=m)
    states = expand_states(z)
    b_all = TP.stack_states(states)
    act = torch.tensor(z["actions"])
    with torch.no_grad():
        values = TP.value(agent.params(), b_all)
    adv, ret = TP.estimate_advantages(torch.tensor(z["rewards"]), torch.tensor(z["masks"]), values,
                                      *(float(x) for x in z["gamma_tau"]))
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
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(agent.step(TP.stack_states([states[j] for j in idx]), act[idx], adv[idx], ret[idx],
                                     fixed[idx], ind))
    return np.array(losses), agent.flat()


@pytest.mark.parametrize("entry", ["updater", "agent"])
def test_update_matches_the_port_replay(dev, entry):
    from drl_urban_planning_b200.agent import use_b200_update
    z = load(GOLDEN, "update_small")
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    gamma, tau = (float(x) for x in z["gamma_tau"])
    m = 0.05
    want_losses, want_params = port_replay(z, m, B, epochs, np_seed)
    logged = []
    np.random.seed(np_seed)
    if entry == "updater":
        up = PPOUpdater(z["params"], int(z["n_cap"]), int(z["e_cap"]), dev, gamma=gamma, tau=tau,
                        opt_num_epochs=epochs, mini_batch_size=B, clip_mode=NEVER, max_grad_norm=m, diagnostics=True)
        out = up.update_params(expand_states(z), z["actions"], z["rewards"], z["masks"], z["exps"],
                               log_fn=lambda tag, v, s: logged.append((tag, v, s)))
        flat = up.flat_params()
        assert out["total_grad_clip_fraction"] == 1.0 and out["total_grad_norm"] > m
    else:
        ag = sgnn_agent(dev, int(z["n_cap"]), int(z["e_cap"]), z["params"], logged, gamma=gamma, tau=tau,
                        num_optim_epoch=epochs, mini_batch_size=B)
        ctl = use_b200_update(ag, clip_mode=NEVER, max_grad_norm=m)
        batch = types.SimpleNamespace(states=expand_states(z), actions=z["actions"], rewards=z["rewards"],
                                      masks=z["masks"], exps=z["exps"])
        ag.update_params(batch, 0)
        flat = ctl.updater.flat_params()
        assert rel(ag.actor_critic_net.flat_parameters(), flat) == 0
    assert np.allclose(update_losses(logged), want_losses, rtol=2e-4, atol=2e-5)
    assert rel(flat, want_params) < 2e-5
    assert rel(flat, z["params_after"]) > 1e-3
