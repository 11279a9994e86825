"""H100: the KL penalty on the exact categorical KL (upb_set_kl_penalty, upb_forward_cand, the *_refs entry points) on
both models.

  * off: a context that never set the penalty, one that set it and turned it off again, and candidate log-probs passed
    to a context without it give bit-identical steps (parameters, moments, counters, the whole gradient / statistics
    buffer, launch counts), fused and two-call; upb_forward equals upb_forward_cand(..., NULL);
  * upb_forward_cand against the float64 log-softmax on both sides of the fast-path limits, for an empty mask, above
    the caps (NaN) and for an ids subset;
  * per-graph KL_g (slot 18) and the policy-head gradients of one-graph steps against float64, including a graph whose
    new probabilities underflow; the whole gradient of a mixed minibatch against the float64 oracle (SGNN) and the torch
    port (rl-mlp);
  * fused against two-call with the penalty at the fused-tail grid sizes, the rl-mlp bit for bit;
  * PPOUpdater / use_b200_update with a fixed and an adaptive coefficient against a torch-port replay;
  * the penalty combined with every other option of the step, written once over a table."""
import os
import types

import numpy as np
import pytest
import torch

import klpen_oracle as KO
import ppo_oracle as PPO
from cross_path import MLP_GRIDS, SGNN_GRIDS, hlg_case
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine, adapt_kl_coef
from drl_urban_planning_b200.packing import pack_states
from drl_urban_planning_b200.ppo import GCLIP_NORM_SLOT, KLPEN_SLOT, PPOUpdater
from fixtures_io import expand_states
from harness import (Case, assert_same_state, dev, heads, load, lp_tol, nan_buffer, per_tensor_rel, rel,
                     reproducible_states, sgnn_agent, t, update_losses)
from oracle import mlp_port as MP
from oracle import torch_port as TP
from shape_cases import boundary_batch

pytestmark = pytest.mark.gpu
BETA = 3.0
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def mixed_case(dev, model, seed=5, count=12):
    states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    return Case(dev, model, states, actions, seed, zero_exps=(1,))


def cand_lp(eng, c, params):
    out = eng.forward(c.blob, params, c.dev_args[0], cand_log_probs=True)[-1]
    torch.cuda.synchronize()
    return out


def step(eng, c, params, fused, oc=None, sel=None):
    g = nan_buffer(eng)
    fn = eng.ppo_step if fused else eng.ppo_grad
    fn(c.blob, params, *c.step_args(sel), ids=c.ids(sel), out=g, old_cand_log_probs=oc)
    if not fused:
        eng.apply(params, g)
    return g


def moved(c, p0, n=3):
    """The parameters after n plain steps from p0 (fresh clip-free context, lr 2e-2): a policy well away from the
    pre-pass's.  Near it the penalty's logit seed p - p_old cancels in fp32 (relative error ~ 1e-7 p / |p - p_old|),
    which no fp32 implementation avoids and which would hide the comparison with float64 below that noise."""
    e = c.engine(clip_mode=_lib.CLIP_NEVER, lr=2e-2)
    p = p0.clone()
    for _ in range(n):
        step(e, c, p, True)
    torch.cuda.synchronize()
    return p


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_bit_identical(dev, model, fused):
    c = mixed_case(dev, model)
    never, off, ignored = c.engine(), c.engine(kl_coef=0.5), c.engine()
    off.set_kl_coef(0.0)
    ps = [t(c.flat, dev).clone() for _ in range(3)]
    oc = cand_lp(never, c, ps[0])
    for k in range(3):
        before = [e.launches for e in (never, off, ignored)]
        g0 = step(never, c, ps[0], fused)
        g1 = step(off, c, ps[1], fused, oc)
        g2 = step(ignored, c, ps[2], fused, oc)
        assert_same_state(never, ps[0], g0, off, ps[1], g1, (model, k))
        assert_same_state(never, ps[0], g0, ignored, ps[2], g2, (model, k))
        assert [e.launches - b for e, b in zip((never, off, ignored), before)].count(never.launches - before[0]) == 3
        assert g0.cpu().numpy()[never.stat_offset + KLPEN_SLOT] == 0.0
    # upb_forward is upb_forward_cand with NULL, on every output
    a = never.forward(c.blob, ps[0], c.dev_args[0], want_greedy=True)
    b = never.forward(c.blob, ps[0], c.dev_args[0], want_greedy=True, cand_log_probs=True)
    for x, y in zip(a, b[:4]):
        assert torch.equal(x, y)


def test_penalty_on_requires_the_candidate_log_probs(dev):
    for model in ("sgnn", "mlp"):
        c = mixed_case(dev, model)
        eng = c.engine(kl_coef=BETA)
        p = t(c.flat, dev).clone()
        for fn in (eng.ppo_grad, eng.ppo_step):
            with pytest.raises(_lib.UpbError, match="old_cand_log_probs"):
                fn(c.blob, p, *c.step_args(), out=eng.new_grad_buffer())
        with pytest.raises(ValueError):
            eng.set_kl_coef(-1.0)


def cand_logp64(model, flat, states):
    return (KO.mlp_cand_logp64 if model == "mlp" else KO.cand_logp64)(np.asarray(flat, np.float64), states)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_forward_cand_against_float64(dev, model):
    states, actions, labels = boundary_batch(3)
    flat = PL.MLP.default_init(3) if model == "mlp" else PL.default_init(3)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    p = t(flat, dev)
    got = eng.forward(blob, p, t(actions, dev), cand_log_probs=True)[-1].cpu().numpy()
    want = cand_logp64(model, flat, states)
    for i, (lp, idx) in enumerate(KO.per_graph(got, blob)):
        w = want[i]
        assert lp.shape == w.shape and lp.size > 0, labels[i]
        tol = lp_tol(w, np.abs(w).max() + 1.0)
        assert (np.abs(lp - w) <= tol).all(), (labels[i], np.abs(lp - w).max())
    # an ids subset leaves every other entry untouched
    ids = np.array([0, 5, 9, 17], np.int32)
    buf = torch.full((blob.cand_len,), 7.0, device=dev)
    fn = getattr(_lib.lib(), eng._p + "forward_cand")
    _lib.check(fn(eng._ctx, blob.dev_ptr(), t(ids, dev).data_ptr(), len(ids), p.data_ptr(), None, None, None, None,
                  None, buf.data_ptr(), eng._stream()))
    sub = buf.cpu().numpy()
    off, k, _ = KO.cand_layout(blob)
    listed = np.zeros(blob.cand_len, bool)
    for i in ids:
        listed[off[i]:off[i] + k[i]] = True
    assert np.array_equal(sub[listed], got[listed]) and (sub[~listed] == 7.0).all()
    # graphs above the context's caps get NaN (as their value does); the others are written
    small = Engine(dev, 500, 1500, model=model)
    buf = torch.zeros(blob.cand_len, device=dev)
    val = torch.zeros(blob.count, device=dev)
    _lib.check(getattr(_lib.lib(), small._p + "forward_cand")(small._ctx, blob.dev_ptr(), None, blob.count,
                                                               p.data_ptr(), None, val.data_ptr(), None, None, None,
                                                               buf.data_ptr(), small._stream()))
    b, v = buf.cpu().numpy(), val.cpu().numpy()
    over = (blob.info[:, 0] > 500) | (blob.info[:, 1] > 1500)
    assert over.any() and not over.all()
    for i in range(blob.count):
        seg = b[off[i]:off[i] + k[i]]
        assert np.isnan(seg).all() == bool(over[i]) and np.isnan(v[i]) == bool(over[i]), labels[i]
        if not over[i]:
            assert np.array_equal(seg, got[off[i]:off[i] + k[i]]), labels[i]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_forward_cand_empty_mask(dev, model):
    z = load(GOLDEN, "edge_empty")
    states = expand_states(z)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    flat = PL.MLP.default_init(1) if model == "mlp" else PL.default_init(1)
    _, k, _ = KO.cand_layout(blob)
    assert (k == 0).any()
    buf = torch.full((max(blob.cand_len, 1),), 7.0, device=dev)
    _lib.check(getattr(_lib.lib(), eng._p + "forward_cand")(eng._ctx, blob.dev_ptr(), None, blob.count,
                                                             t(flat, dev).data_ptr(), None, None, None, None, None,
                                                             buf.data_ptr(), eng._stream()))
    got = buf.cpu().numpy()[:blob.cand_len]
    want = cand_logp64(model, flat, states)
    for i, (lp, _) in enumerate(KO.per_graph(got, blob)):
        assert lp.size == want[i].size
        assert (np.abs(lp - want[i]) <= lp_tol(want[i], np.abs(want[i]).max(initial=0) + 1)).all()


def underflow_params(c, p):
    """p with both policy heads' output layers scaled so that most new candidate probabilities underflow in fp32."""
    q = p.clone()
    for name in ("lu_w1", "road_w1"):
        s = c.layout.slots[name]
        q[s.offset:s.offset + s.size] *= 400.0
    return q


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_per_graph_terms(dev, model, fused):
    """One-graph steps (B = 1, no clip) at a policy 3 plain steps away from the pre-pass: slot 18 against float64 KL_g
    of the kernel's own reference log-probs, and the policy head's gradient against the float64 oracle (SGNN) or the
    float64 rl-mlp port; also at a policy whose new probabilities underflow (a large finite KL)."""
    c = mixed_case(dev, model)
    p0 = t(c.flat, dev).clone()
    eng = c.engine(kl_coef=BETA, clip_mode=_lib.CLIP_NEVER)
    oc = cand_lp(eng, c, p0)
    lp_old = [x for x, _ in KO.per_graph(oc.cpu().numpy(), c.blob)]
    for p1 in (moved(c, p0), underflow_params(c, moved(c, p0))):
        flat1 = p1.cpu().numpy()
        lp_new = cand_logp64(model, flat1, c.states)
        for i in range(c.count):
            g = step(eng, c, p1.clone(), fused, oc, sel=[i])
            torch.cuda.synchronize()
            gn = g.cpu().numpy()
            st = gn[eng.stat_offset:]
            want = PPO.kl64(lp_old[i], lp_new[i])[0] if c.exps[i] != 0 else 0.0
            assert np.isfinite(st[KLPEN_SLOT]) and st[7] == 0, i
            assert np.isclose(st[KLPEN_SLOT], want, rtol=1e-4, atol=1e-6), (i, st[KLPEN_SLOT], want)
            if model == "sgnn":
                r = PPO.sgnn_minibatch(flat1.astype(np.float64), [c.states[i]], c.actions[[i]], c.adv[[i]],
                                       c.ret[[i]], c.fixed[[i]], c.exps[[i]], lp_old=[lp_old[i]], kl_coef=BETA)
                want_g = r["grad"]
            else:
                want_g = mlp_grad64(c, flat1, [i], lp_old)
            hd = heads(c.layout)[int(c.stage[i])]
            assert rel(gn[hd], want_g[hd], floor=1e-6) < 1e-4, (i, rel(gn[hd], want_g[hd], floor=1e-6))


def mlp_grad64(c, flat1, sel, lp_old):
    """float64 gradient of the rl-mlp loss plus BETA * kl (kl against the given old log-probs) on the graphs `sel`."""
    P = KO.mlp_params64(flat1, requires_grad=True)
    b = MP.stack_states([c.states[i] for i in sel])
    ex = torch.tensor(c.exps[sel])
    ind = ex.nonzero(as_tuple=False).squeeze(1)
    surr, vl, el = MP.ppo_losses(P, b, torch.tensor(c.actions[sel]), torch.tensor(c.adv[sel]).double(),
                                 torch.tensor(c.ret[sel]).double(), torch.tensor(c.fixed[sel]).double(), ind)
    zl, zr = MP.masked_logits(P, b)
    st0 = b["stage"][:, 0] > 0
    kls = []
    for j, i in enumerate(sel):
        z = (zl if st0[j] else zr)[j]
        mask = (b["land_use_mask"] if st0[j] else b["road_mask"])[j]
        lo = torch.tensor(np.asarray(lp_old[i], np.float64))
        kls.append(KO.kl_rows(lo, torch.log_softmax(z[mask], -1)) if mask.any() else z.sum() * 0)
    kl = torch.stack(kls)[ind].mean() if ind.numel() else torch.zeros((), dtype=torch.float64)
    (surr + 0.5 * vl + 0.01 * el + BETA * kl).backward()
    g = np.zeros(PL.MLP.num_params)
    for s in PL.MLP.slots.values():
        if P[s.name].grad is not None:
            g[s.offset:s.offset + s.size] = P[s.name].grad.numpy().reshape(-1)
    return g


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_mixed_minibatch_gradient(dev, model):
    c = mixed_case(dev, model)
    p0 = t(c.flat, dev).clone()
    eng = c.engine(kl_coef=BETA, clip_mode=_lib.CLIP_NEVER)
    oc = cand_lp(eng, c, p0)
    lp_old = [x for x, _ in KO.per_graph(oc.cpu().numpy(), c.blob)]
    p1 = moved(c, p0)
    flat1 = p1.cpu().numpy()
    g = eng.ppo_grad(c.blob, p1, *c.step_args(), old_cand_log_probs=oc)
    torch.cuda.synchronize()
    gn = g.cpu().numpy()
    if model == "sgnn":
        r = PPO.sgnn_minibatch(flat1.astype(np.float64), c.states, c.actions, c.adv, c.ret, c.fixed, c.exps,
                               lp_old=lp_old, kl_coef=BETA)
        want = r["grad"]
        assert np.isclose(gn[eng.stat_offset + KLPEN_SLOT], r["kl_sum"], rtol=1e-4)
        assert np.isclose(eng.read_losses(g)[0], r["loss"], rtol=1e-4, atol=1e-5)
    else:
        want = mlp_grad64(c, flat1, list(range(c.count)), lp_old)
    worst, where = per_tensor_rel(gn[:c.layout.num_params], want, c.layout)
    assert worst < 1e-4, (worst, where)
    plain = c.engine(clip_mode=_lib.CLIP_NEVER).ppo_grad(c.blob, p1, *c.step_args())
    assert per_tensor_rel(plain.cpu().numpy()[:c.layout.num_params], want, c.layout)[0] > 1e-3


@pytest.mark.parametrize("grid", MLP_GRIDS)
def test_mlp_fused_bit_identical_with_penalty(dev, grid):
    states, actions = reproducible_states(11, 40)
    c = Case(dev, "mlp", states, actions, 11)
    e1, e2 = c.engine(grid_limit=grid, kl_coef=BETA), c.engine(grid_limit=grid, kl_coef=BETA)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    oc = cand_lp(e1, c, p1)
    for k in range(3):
        g1 = step(e1, c, p1, False, oc)
        g2 = step(e2, c, p2, True, oc)
        assert_same_state(e1, p1, g1, e2, p2, g2, (grid, k))
    assert g2.cpu().numpy()[e2.stat_offset + KLPEN_SLOT] > 0


@pytest.mark.parametrize("grid", SGNN_GRIDS)
def test_sgnn_fused_against_two_call_with_penalty(dev, grid):
    c = hlg_case(dev, 3)
    e1, e2 = c.engine(grid_limit=grid, kl_coef=BETA), c.engine(grid_limit=grid, kl_coef=BETA)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    oc = cand_lp(e1, c, p1)
    for k in range(3):
        g1 = step(e1, c, p1, False, oc)
        before = e2.launches
        g2 = step(e2, c, p2, True, oc)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (k > 0)
        # after the first step the two paths' parameters differ in the last bits, and the penalty's seed p - p_old
        # (a small difference of close probabilities) and KL_g amplify that by |p| / |p - p_old|
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < (1e-5 if k == 0 else 1e-4), (k, worst, where)
        s1, s2 = (g.cpu().numpy()[e1.stat_offset + KLPEN_SLOT] for g in (g1, g2))
        assert np.isclose(s1, s2, rtol=1e-3, atol=1e-7) and (k == 0 or s2 > 0)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, k


# ---- the whole update against a torch-port replay ---------------------------------------------------------------------
def rollout(seed, T):
    states, actions = synth.make_states(seed, "small", T, stages=[int(i % 3 == 1) for i in range(T)])
    rng = np.random.default_rng(seed)
    rewards = rng.normal(size=T).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[[9, 19, 29, T - 1]] = 0.0
    exps = np.ones(T, np.float32)
    exps[[2, 17]] = 0.0
    return states, actions, rewards, masks, exps


def port_replay(model, flat, roll, B, epochs, np_seed, gamma, tau, beta, kl_target=None, iterations=1):
    """The reference's update_params plus beta * kl against each update's pre-pass policy, in the torch ports, over
    `iterations` updates of the same rollout; with kl_target, beta adapts after each update on the last epoch's mean
    KL.  (losses per step, the betas used, final parameters)."""
    states, actions, rewards, masks, exps = roll
    mlp = model == "mlp"
    stack = MP.stack_states if mlp else TP.stack_states
    agent = (PPO.MLPPortAgent if mlp else PPO.PortAgent)(flat, kl_coef=beta)
    b_all = stack(states)
    act = torch.tensor(actions)
    T = len(states)
    e_t = torch.tensor(exps)
    np.random.seed(np_seed)
    losses, betas = [], []
    for _ in range(iterations):
        agent.snapshot()
        with torch.no_grad():
            P = agent.P
            values = (MP.value if mlp else TP.value)(P, b_all).reshape(-1, 1).float()
            fixed, _ = (MP.log_prob_entropy if mlp else TP.log_prob_entropy)(P, b_all, act)
        adv, ret = TP.estimate_advantages(torch.tensor(rewards), torch.tensor(masks), values, gamma, tau)
        order = np.arange(T)
        betas.append(agent.kl_coef)
        for _ in range(epochs):
            perm = np.arange(T)
            np.random.shuffle(perm)
            order = order[perm]
            s18 = s4 = 0.0
            for i in range(T // B):
                idx = order[i * B:(i + 1) * B]
                ind = e_t[idx].nonzero(as_tuple=False).squeeze(1)
                losses.append(agent.step(stack([states[j] for j in idx]), act[idx], adv[idx], ret[idx], fixed[idx],
                                         ind))
                s18 += agent.last_kl * ind.numel()
                s4 += ind.numel()
        if kl_target is not None:
            agent.kl_coef = adapt_kl_coef(agent.kl_coef, s18, s4, kl_target)
    return np.array(losses), betas, agent.flat()


def run_updater(dev, model, flat, roll, B, epochs, iterations=1, **kw):
    up = PPOUpdater(flat, 128, 512, dev, gamma=0.99, tau=0.95, opt_num_epochs=epochs, mini_batch_size=B, model=model,
                    **kw)
    logged, outs, rows = [], [], []
    np.random.seed(7)
    for it in range(iterations):
        outs.append(up.update_params(*roll, log_fn=lambda tg, v, s: logged.append((tg, v, s)), iteration=it))
        so = up.engine.stat_offset
        ring = up._grad_ring.cpu().numpy()
        rows.append((float(ring[:, so + KLPEN_SLOT].astype(np.float64).sum()), float(ring[:, so + 4].sum())))
    return up, logged, outs, rows


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_updater_fixed_beta_against_the_port(dev, model):
    T, B, epochs = 40, 16, 2
    roll = rollout(21, T)
    flat = PL.MLP.default_init(21) if model == "mlp" else PL.default_init(21)
    want_losses, _, want_flat = port_replay(model, flat, roll, B, epochs, 7, 0.99, 0.95, BETA)
    up, logged, outs, _ = run_updater(dev, model, flat, roll, B, epochs, kl_coef=BETA)
    got = update_losses(logged)
    assert got.shape == want_losses.shape
    assert np.allclose(got, want_losses, rtol=2e-4, atol=2e-5), np.abs(got - want_losses).max()
    match = rel(up.flat_params(), want_flat)
    assert match < 5e-5
    kl = np.array([v for tg, v, _ in logged if tg == "loss/kl_loss"])
    assert kl.shape == (len(got),) and abs(kl[0]) < 1e-6 and (kl[1:] > 0).all()   # step 0: the pre-pass policy
    assert outs[0]["kl_coef"] == outs[0]["kl_coef_next"] == BETA
    assert np.isclose(outs[0]["total_kl_loss"], kl.sum() / epochs)
    _, _, plain_flat = port_replay(model, flat, roll, B, epochs, 7, 0.99, 0.95, 0.0)
    assert rel(up.flat_params(), plain_flat) > 10 * match         # the penalty moved the trajectory


@pytest.mark.parametrize("target_scale,factor", [(0.01, 2.0), (100.0, 0.5)])
def test_updater_adaptive_beta(dev, target_scale, factor):
    """Two updates with kl_target far below / above the measured KL: beta doubles / halves after each, the rule applied
    to the GPU's own slot-18 / slot-4 rows, and the trajectory follows the port's replay with its own decisions."""
    T, B, epochs = 40, 16, 2
    roll = rollout(21, T)
    flat = PL.default_init(21)
    _, _, _, rows = run_updater(dev, "sgnn", flat, roll, B, epochs, kl_coef=BETA)
    target = target_scale * rows[0][0] / rows[0][1]
    up, logged, outs, rows = run_updater(dev, "sgnn", flat, roll, B, epochs, iterations=2, kl_coef=BETA,
                                         kl_target=target)
    assert [o["kl_coef"] for o in outs] == [BETA, BETA * factor]
    for o, r in zip(outs, rows):
        assert o["kl_coef_next"] == adapt_kl_coef(o["kl_coef"], *r, target) == o["kl_coef"] * factor
    assert up.kl_coef == up.engine.kl_coef == BETA * factor ** 2
    assert [v for tg, v, _ in logged if tg == "diag/kl_coef"] == [BETA, BETA * factor]
    want_losses, betas, want_flat = port_replay("sgnn", flat, roll, B, epochs, 7, 0.99, 0.95, BETA, target, 2)
    assert betas == [BETA, BETA * factor]
    assert np.allclose(update_losses(logged), want_losses, rtol=5e-4, atol=5e-5)
    assert rel(up.flat_params(), want_flat) < 1e-4


def test_use_b200_update_with_the_penalty(dev):
    from drl_urban_planning_b200.agent import use_b200_update
    T, B = 40, 16
    roll = rollout(21, T)
    flat = PL.default_init(21)
    want_losses, _, want_flat = port_replay("sgnn", flat, roll, B, 2, 7, 0.99, 0.95, BETA)
    logged = []
    ag = sgnn_agent(dev, 128, 512, flat, logged, num_optim_epoch=2, mini_batch_size=B)
    ctl = use_b200_update(ag, kl_coef=BETA, kl_target=1e6)
    states, actions, rewards, masks, exps = roll
    batch = types.SimpleNamespace(states=states, actions=actions, rewards=rewards, masks=masks, exps=exps)
    np.random.seed(7)
    ag.update_params(batch, 0)
    assert np.allclose(update_losses(logged), want_losses, rtol=2e-4, atol=2e-5)
    assert rel(ag.actor_critic_net.flat_parameters(), want_flat) < 5e-5
    assert ctl.updater.kl_coef == BETA / 2 and ctl.optimizer_state()["kl_coef"] == BETA / 2
    assert "loss/kl_loss" in {tg for tg, _, _ in logged}


# ---- combinations ------------------------------------------------------------------------------------------------------
COMBOS = {
    "target_kl": dict(target_kl=0.02),
    "value_clip": dict(value_clip=0.2, normalize_advantage=True),
    "max_grad_norm": dict(max_grad_norm=0.3, clip_mode=_lib.CLIP_NEVER),
    "clip_always": dict(clip_mode=_lib.CLIP_ALWAYS),
    "weightdecay": dict(weight_decay=1e-2),
    "diagnostics": dict(diagnostics=True),
    "batch_stage": dict(batch_stage=True),
}


@pytest.mark.parametrize("combo", sorted(COMBOS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_combinations(dev, model, combo):
    """The penalty with each other option: the update runs, logs the KL, differs from the option alone, and (SGNN)
    reproduces itself bit for bit; with max_grad_norm, the norm the step clipped by includes the penalty's gradient."""
    T, B, epochs = 40, 16, 2
    roll = rollout(23, T)
    flat = PL.MLP.default_init(23) if model == "mlp" else PL.default_init(23)
    kw = COMBOS[combo]
    a, la, oa, _ = run_updater(dev, model, flat, roll, B, epochs, kl_coef=BETA, **kw)
    base, _, _, _ = run_updater(dev, model, flat, roll, B, epochs, **kw)
    assert np.isfinite(a.flat_params()).all()
    assert "loss/kl_loss" in {tg for tg, _, _ in la} and oa[0]["kl_coef"] == BETA
    assert rel(a.flat_params(), base.flat_params()) > 1e-5
    if model == "sgnn":
        b, lb, _, _ = run_updater(dev, model, flat, roll, B, epochs, kl_coef=BETA, **kw)
        assert np.array_equal(a.flat_params(), b.flat_params()) and la == lb
    if combo == "max_grad_norm":
        c = mixed_case(dev, model)
        eng = c.engine(kl_coef=BETA, **kw)
        p0 = t(c.flat, dev).clone()
        oc = cand_lp(eng, c, p0)
        p1 = moved(c, p0)
        g = step(eng, c, p1, True, oc).cpu().numpy()
        norm = np.sqrt((g[:c.layout.num_params].astype(np.float64) ** 2).sum())
        assert np.isclose(g[eng.stat_offset + GCLIP_NORM_SLOT], norm, rtol=1e-5)
        assert g[eng.stat_offset + KLPEN_SLOT] > 0
