"""H100: the clipped value loss (upb_set_value_clip, the *_vclip entry points) and the per-minibatch advantage
normalisation (upb_normalize_advantages, k_adv_norm) on both models.

  * off: a context that never set the option, one that set it and turned it off again, and old_values passed to a
    context without it give bit-identical steps (parameters, moments, counters, the whole gradient / statistics buffer,
    launch counts), fused and two-call;
  * the per-graph value seeds (read through the value-head bias gradient of one-graph steps) and statistics slots 15 /
    16 against the fp32 replay of the seed, in all four branches; the whole gradient against the float64 oracle (SGNN)
    and the torch port (rl-mlp);
  * fused against two-call with clipping on at the fused-tail grid sizes, the rl-mlp bit for bit;
  * k_adv_norm against float64 and bit-identical from run to run;
  * PPOUpdater / use_b200_update with both options against a torch-port replay of the same permutations, combined with
    target_kl."""
import os
import types

import numpy as np
import pytest
import torch

import ppo_oracle as PPO
import vclip_oracle as VO
from cross_path import MLP_GRIDS, SGNN_GRIDS, hlg_case
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from drl_urban_planning_b200.ppo import VCLIP_COUNT_SLOT, VCLIP_LOSS_SLOT, PPOUpdater
from harness import (Case, assert_same_state, dev, load, nan_buffer, per_tensor_rel, rel, reproducible_states,
                     sgnn_agent, spawn, t, update_losses)
from oracle import mlp_port as MP
from oracle import torch_port as TP

pytestmark = pytest.mark.gpu
C = 0.2
# offsets V_old - V per graph: exact tie, inside the clamp, clipped branch larger or smaller (both signs), far out
OFFSETS = np.array([0.0, 0.05, -0.07, 0.5, -0.5, 0.35, -0.35, 0.01, 2.0, -2.0, 0.0, 0.12], np.float32)


def mixed_case(dev, model, seed=5, count=12):
    states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    return Case(dev, model, states, actions, seed, zero_exps=(1,))


def old_values(eng, c, params, offsets=OFFSETS):
    v, _, _ = eng.forward(c.blob, params, c.dev_args[0])
    torch.cuda.synchronize()
    v = v.cpu().numpy()
    return v, (v + np.resize(offsets, v.shape)).astype(np.float32)


def split_inside(V, R, ov, c, offsets):
    """Moves the old value of every graph inside the clamp (0 < |offset| < c) by up to 10 % of its offset to where, in
    fp32, V_old + (V - V_old) does not round back to V, so that the two terms differ in the last bits: alternately one
    where the clipped term is the larger and one where the unclipped is.  (V_old + (V - V_old) == V whenever |V| is not
    small against the offset, so this needs offsets well above |V|: a wide clip range.)  Graphs with no such point keep
    their old value."""
    f = np.float32
    ov = ov.copy()
    inside = np.flatnonzero((np.abs(offsets) > 0) & (np.abs(offsets) < c))
    for j, i in enumerate(inside):
        cand = (V[i] + offsets[i] * np.linspace(0.9, 1.1, 4001)).astype(f)
        d = (V[i] - cand).astype(f)
        vc = (cand + np.minimum(np.maximum(d, -f(c)), f(c))).astype(f)
        la, lb = f(f(V[i] - R[i]) ** 2), ((vc - R[i]) * (vc - R[i])).astype(f)
        split = (vc != V[i]) & (la != lb)
        want = split & ((lb > la) if j % 2 else (la > lb))
        pick = np.flatnonzero(want if want.any() else split)
        if pick.size:
            ov[i] = cand[pick[0]]
    return ov


def step(eng, c, params, fused, ov=None, sel=None):
    g = nan_buffer(eng)
    fn = eng.ppo_step if fused else eng.ppo_grad
    fn(c.blob, params, *c.step_args(sel), ids=c.ids(sel), out=g, old_values=None if ov is None else t(ov, c.dev))
    if not fused:
        eng.apply(params, g)
    return g


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_bit_identical(dev, model, fused):
    c = mixed_case(dev, model)
    never, off = c.engine(), c.engine(value_clip=0.3)
    _lib.check(_lib.lib().upb_set_value_clip(off._ctx, 0.0))
    ignored = c.engine()
    ps = [t(c.flat, dev).clone() for _ in range(3)]
    _, ov = old_values(never, c, ps[0])
    for k in range(3):
        before = [e.launches for e in (never, off, ignored)]
        g0 = step(never, c, ps[0], fused)
        g1 = step(off, c, ps[1], fused, ov)
        g2 = step(ignored, c, ps[2], fused, ov)
        assert_same_state(never, ps[0], g0, off, ps[1], g1, (model, k))
        assert_same_state(never, ps[0], g0, ignored, ps[2], g2, (model, k))
        assert [e.launches - b for e, b in zip((never, off, ignored), before)].count(never.launches - before[0]) == 3
        assert not g0.cpu().numpy()[never.stat_offset + VCLIP_LOSS_SLOT:never.stat_offset + VCLIP_COUNT_SLOT + 1].any()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_clipping_on_requires_old_values(dev, model):
    c = mixed_case(dev, model)
    eng = c.engine(value_clip=C)
    p = t(c.flat, dev).clone()
    for fn in (eng.ppo_grad, eng.ppo_step):
        with pytest.raises(_lib.UpbError, match="old_values"):
            fn(c.blob, p, *c.step_args(), out=eng.new_grad_buffer())


@pytest.mark.parametrize("clip", [C, 4.0])
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_per_graph_seeds_and_slots(dev, model, fused, clip):
    """One-graph steps (B = 1): the value-head bias gradient is the graph's seed g_V, bit for bit the fp32 replay of
    torch's operations on the kernel's own inputs (V from the forward kernel, R, V_old), and so are slots 0, 15 and 16.
    The wide clip range puts graphs inside the clamp where V_old + (V - V_old) != V and the two terms differ in the last
    bits, the clipped one larger on some and smaller on others: there the branch must be the one torch takes.  Then
    the whole minibatch: slot 16 exact, slot 15 the sum."""
    c = mixed_case(dev, model)
    b2 = c.layout.slots["val_b2"].offset
    eng = c.engine(value_clip=clip, clip_mode=_lib.CLIP_NEVER)
    p0 = t(c.flat, dev)
    offsets = np.resize(OFFSETS * np.float32(clip / C), c.count)
    V, ov = old_values(eng, c, p0, offsets)
    R = c.ret.reshape(-1)
    ov = split_inside(V, R, ov, clip, offsets)
    _, _, cl, _ = PPO.value_seed32(V, R, V_old=ov, value_clip=clip)
    if clip > 1.0:
        d = (V - ov).astype(np.float32)
        split = (np.abs(d) < clip) & ((ov + d).astype(np.float32) != V)
        assert cl[split].any() and not cl[split].all(), (V, ov)
    for i in range(c.count):
        g = step(eng, c, p0.clone(), fused, ov, sel=[i])
        want, loss, clipped, _ = PPO.value_seed32(V[i], R[i], c_value=0.5, inv_batch=1.0, V_old=ov[i], value_clip=clip)
        st = g.cpu().numpy()[eng.stat_offset:]
        assert g.cpu().numpy()[b2] == want[0], (i, g.cpu().numpy()[b2], want[0])
        assert st[VCLIP_LOSS_SLOT] == loss[0] and st[VCLIP_COUNT_SLOT] == clipped[0], (i, st[15:17], loss, clipped)
        assert st[0] == np.float32(V[i] - R[i]) ** 2, i
    g = step(eng, c, p0.clone(), fused, ov)
    st = g.cpu().numpy()[eng.stat_offset:]
    _, loss, clipped, _ = PPO.value_seed32(V, R, V_old=ov, value_clip=clip)
    assert clipped.any() and not clipped.all()
    assert st[VCLIP_COUNT_SLOT] == clipped.sum()
    assert np.isclose(st[VCLIP_LOSS_SLOT], loss.astype(np.float64).sum(), rtol=1e-5)
    assert np.isclose(eng.read_losses(g)[1], st[VCLIP_LOSS_SLOT] / c.count, rtol=1e-6)


def test_sgnn_gradient_against_the_float64_oracle(dev):
    c = mixed_case(dev, "sgnn")
    eng = c.engine(value_clip=C)
    p = t(c.flat, dev).clone()
    _, ov = old_values(eng, c, p)
    g = eng.ppo_grad(c.blob, p, *c.step_args(), old_values=t(ov, dev))
    r = PPO.sgnn_minibatch(c.flat.astype(np.float64), c.states, c.actions, c.adv, c.ret, c.fixed, c.exps, old_values=ov,
                           value_clip=C)
    worst, where = per_tensor_rel(g.cpu().numpy()[:PL.NUM_PARAMS], r["grad"])
    assert worst < 1e-4, (worst, where)
    assert np.allclose(eng.read_losses(g), [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]],
                       rtol=1e-4, atol=1e-5)
    plain = Engine(dev, c.blob.n_cap, c.blob.e_cap).ppo_grad(c.blob, p, *c.step_args())
    assert per_tensor_rel(plain.cpu().numpy()[:PL.NUM_PARAMS], r["grad"])[0] > 1e-3


def test_mlp_trajectory_against_the_torch_port(dev):
    """Three steps (the first clipped) of the rl-mlp model against MLPPortAgent with the clipped loss."""
    c = mixed_case(dev, "mlp")
    eng = c.engine(value_clip=C)
    p = t(c.flat, dev).clone()
    _, ov = old_values(eng, c, p)
    agent = PPO.MLPPortAgent(c.flat, value_clip=C)
    agent.old_values = torch.tensor(ov).reshape(-1, 1)
    b = MP.stack_states(c.states)
    ind = torch.tensor(c.exps).nonzero(as_tuple=False).squeeze(1)
    for k in range(3):
        want = agent.step(b, torch.tensor(c.actions), torch.tensor(c.adv), torch.tensor(c.ret), torch.tensor(c.fixed),
                          ind)
        g = step(eng, c, p, True, ov)
        torch.cuda.synchronize()
        assert np.allclose(eng.read_losses(g), want, rtol=1e-4, atol=1e-5), k
        assert rel(p.cpu().numpy(), agent.flat()) < 2e-5, k


@pytest.mark.parametrize("grid", MLP_GRIDS)
def test_mlp_fused_bit_identical_with_clipping(dev, grid):
    states, actions = reproducible_states(11, 40)
    c = Case(dev, "mlp", states, actions, 11)
    e1, e2 = c.engine(grid_limit=grid, value_clip=C), c.engine(grid_limit=grid, value_clip=C)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    _, ov = old_values(e1, c, p1, OFFSETS * 0.5)
    for k in range(3):
        g1 = step(e1, c, p1, False, ov)
        g2 = step(e2, c, p2, True, ov)
        assert_same_state(e1, p1, g1, e2, p2, g2, (grid, k))
    assert g2.cpu().numpy()[e2.stat_offset + VCLIP_COUNT_SLOT] > 0


@pytest.mark.parametrize("grid", SGNN_GRIDS)
def test_sgnn_fused_against_two_call_with_clipping(dev, grid):
    c = hlg_case(dev, 3)
    e1, e2 = c.engine(grid_limit=grid, value_clip=C), c.engine(grid_limit=grid, value_clip=C)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    _, ov = old_values(e1, c, p1, OFFSETS * 0.5)
    for k in range(3):
        g1 = step(e1, c, p1, False, ov)
        before = e2.launches
        g2 = step(e2, c, p2, True, ov)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (k > 0)
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (k, worst, where)
        s1, s2 = (g.cpu().numpy()[e1.stat_offset:] for g in (g1, g2))
        assert np.isclose(s1[VCLIP_LOSS_SLOT], s2[VCLIP_LOSS_SLOT], rtol=1e-5)
        if k == 0:       # same parameters; later the paths' last-bit differences may flip graphs that sit on a tie
            assert s1[VCLIP_COUNT_SLOT] == s2[VCLIP_COUNT_SLOT]
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, k


@pytest.mark.parametrize("T,B", [(45, 16), (256, 64), (1000, 256), (7, 8)])
def test_adv_norm_kernel(dev, T, B):
    rng = np.random.default_rng(T)
    adv = rng.normal(1.0, 4.0, size=T).astype(np.float32)
    exps = (rng.random(T) > 0.2).astype(np.float32)
    order = rng.permutation(T).astype(np.int32)
    if T >= 2 * B:
        exps[order[:B]] = 0.0
        exps[order[0]] = 1.0                    # minibatch 0: one exps != 0 graph, kept as it is
    eng = Engine(dev, 16, 16)
    o = t(order, dev)
    out1 = eng.normalize_advantages(t(adv, dev), t(exps, dev), o, B)
    out2 = eng.normalize_advantages(t(adv, dev), t(exps, dev), o, B)
    got = out1.cpu().numpy()
    assert np.array_equal(got, out2.cpu().numpy())
    want = VO.normalize64(adv, exps, order, B)
    assert np.array_equal(got, want) or np.abs(got - want).max() <= 2 * np.spacing(np.abs(want).max()), \
        np.abs(got - want).max()
    assert np.array_equal(got[order[(T // B) * B:]], adv[order[(T // B) * B:]])


def rollout(seed, T):
    states, actions = synth.make_states(seed, "small", T, stages=[int(i % 3 == 1) for i in range(T)])
    rng = np.random.default_rng(seed)
    rewards = rng.normal(size=T).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[[9, 19, 29, T - 1]] = 0.0
    exps = np.ones(T, np.float32)
    exps[[2, 17]] = 0.0
    return states, actions, rewards, masks, exps


def port_replay(model, flat, states, actions, rewards, masks, exps, B, epochs, np_seed, gamma, tau):
    """The reference's update_params with the clipped value loss and SB3's advantage normalisation, in the torch ports."""
    mlp = model == "mlp"
    stack = MP.stack_states if mlp else TP.stack_states
    agent = (PPO.MLPPortAgent if mlp else PPO.PortAgent)(flat, value_clip=C)
    b_all = stack(states)
    act = torch.tensor(actions)
    with torch.no_grad():
        P = agent.P if mlp else agent.params()
        values = (MP.value if mlp else TP.value)(P, b_all).reshape(-1, 1).float()
        fixed, _ = (MP.log_prob_entropy if mlp else TP.log_prob_entropy)(P, b_all, act)
    adv, ret = TP.estimate_advantages(torch.tensor(rewards), torch.tensor(masks), values, gamma, tau)
    T = len(states)
    e_t = torch.tensor(exps)
    np.random.seed(np_seed)
    order, losses = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(T // B):
            idx = order[i * B:(i + 1) * B]
            ind = e_t[idx].nonzero(as_tuple=False).squeeze(1)
            a = adv[idx].clone()
            if ind.numel() > 1:
                a = (a - a[ind].mean()) / (a[ind].std() + 1e-8)
            agent.old_values = values[idx]
            losses.append(agent.step(stack([states[j] for j in idx]), act[idx], a, ret[idx],
                                     fixed[idx], ind))
    return np.array(losses), agent.flat()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_updater_with_both_options_against_the_port(dev, model):
    T, B, epochs, gamma, tau = 40, 16, 2, 0.99, 0.95
    states, actions, rewards, masks, exps = rollout(21, T)
    flat = PL.MLP.default_init(21) if model == "mlp" else PL.default_init(21)
    want_losses, want_flat = port_replay(model, flat, states, actions, rewards, masks, exps, B, epochs, 7, gamma, tau)
    runs = {}
    for name, kw in (("both", dict(value_clip=C, normalize_advantage=True)),
                     ("both_kl", dict(value_clip=C, normalize_advantage=True, target_kl=1e3)),
                     ("none", {}), ("off", dict(value_clip=None, normalize_advantage=False))):
        up = PPOUpdater(flat, 128, 512, dev, gamma=gamma, tau=tau, opt_num_epochs=epochs, mini_batch_size=B,
                        model=model, diagnostics=name == "both", **kw)
        logged = []
        np.random.seed(7)
        out = up.update_params(states, actions, rewards, masks, exps, log_fn=lambda tg, v, s: logged.append((tg, v, s)))
        runs[name] = (up.flat_params(), update_losses(logged), out, {tg for tg, _, _ in logged})
    got, losses, out, tags = runs["both"]
    assert losses.shape == want_losses.shape
    assert np.allclose(losses, want_losses, rtol=2e-4, atol=2e-5), np.abs(losses - want_losses).max()
    assert rel(got, want_flat) < 5e-5
    assert "diag/value_clip_fraction" in tags and "total_value_clip_fraction" in out
    # a target that never fires changes nothing (rl-mlp steps on general states are reproducible only to the last bits)
    assert rel(runs["both_kl"][0], got) < 1e-6
    assert rel(runs["none"][0], runs["off"][0]) < 1e-6 and runs["none"][3] == runs["off"][3]
    assert "diag/value_clip_fraction" not in runs["none"][3]
    assert rel(runs["none"][0], want_flat) > 1e-4


def test_use_b200_update_with_both_options(dev):
    from drl_urban_planning_b200.agent import use_b200_update
    T, B = 40, 16
    states, actions, rewards, masks, exps = rollout(21, T)
    flat = PL.default_init(21)
    want_losses, want_flat = port_replay("sgnn", flat, states, actions, rewards, masks, exps, B, 2, 7, 0.99, 0.95)
    logged = []
    ag = sgnn_agent(dev, 128, 512, flat, logged, num_optim_epoch=2, mini_batch_size=B)
    ctl = use_b200_update(ag, value_clip=C, normalize_advantage=True, target_kl=1e3)
    assert ctl.updater.engine.value_clip == C and ctl.updater.normalize_advantage
    batch = types.SimpleNamespace(states=states, actions=actions, rewards=rewards, masks=masks, exps=exps)
    np.random.seed(7)
    ag.update_params(batch, 0)
    assert np.allclose(update_losses(logged), want_losses, rtol=2e-4, atol=2e-5)
    assert rel(ag.actor_critic_net.flat_parameters(), want_flat) < 5e-5


# ---- the golden vectors recorded by the unmodified reference (tests/golden/make_golden_vf.py) ------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("name", ["small_mixed_vf", "mlp_small_vf"])
def test_golden_trajectory(dev, name, fused):
    """k_adv_norm on the raw advantages, then three steps with the recorded old values, the first one clipped (two-call
    on both paths): losses, every gradient tensor and the parameters after each step, at test_gpu_parity's bars."""
    z = load(GOLDEN, name)
    mlp = name.startswith("mlp")
    layout = PL.MLP if mlp else PL.SGNN
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE, model="mlp" if mlp else "sgnn",
                 value_clip=float(z["value_clip"]))
    params = t(z["params"], dev).clone()
    value, _, _ = eng.forward(blob, params, t(z["actions"], dev))
    assert rel(value.cpu().numpy(), z["values"].ravel()) < 1e-4
    exps = t(z["exps"], dev)
    adv = eng.normalize_advantages(t(z["advantages"], dev), exps, t(np.arange(B, dtype=np.int32), dev), B)
    assert np.allclose(adv.cpu().numpy(), z["advantages_normalized"].ravel(), rtol=0, atol=1e-6)
    args = (t(z["actions"], dev), adv, t(z["returns"], dev), t(z["fixed_log_probs"], dev), exps)
    n_ind = int((z["exps"] != 0).sum())
    ov = t(z["old_values"], dev)
    for k in range(3):
        before = eng.launches
        if fused:
            grad = eng.ppo_step(blob, params, *args, 1.0 / B, 1.0 / n_ind, old_values=ov)
        else:
            grad = eng.ppo_grad(blob, params, *args, 1.0 / B, 1.0 / n_ind, old_values=ov)
            eng.apply(params, grad)
        torch.cuda.synchronize()
        if fused:
            assert (eng.launches - before == 1) == (k > 0), k
        losses = eng.read_losses(grad)
        assert np.allclose(losses, z["losses"][k], rtol=1e-4, atol=1e-5), (k, losses, z["losses"][k])
        worst, where = per_tensor_rel(grad.cpu().numpy()[:layout.num_params], z["grads"][k], layout)
        assert worst < 1e-4, (k, worst, where)
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k
    st = grad.cpu().numpy()[eng.stat_offset:]
    assert st[VCLIP_COUNT_SLOT] > 0 and st[VCLIP_LOSS_SLOT] != st[0]
