"""GPU (H100): the SGNN and rl-mlp kernels at the shape limits where they change code path (tests/shape_cases.py),
graphs of different paths walked one after another by the same CTA, the fused tail at every grid size that changes
how the 114 gradient slices are owned, and the per-step liveness of the two policy heads in the fused tail.

Reference: the float64 oracle (oracle/sgnn_numpy.py; oracle/mlp_port.py for rl-mlp) at the 1e-4 per-tensor bar of
test_gpu_parity.py, and the kernel itself where results must not depend on placement (bit-identical)."""
import numpy as np
import pytest
import torch

import extreme_cases as EC
import shape_cases as SC
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from harness import dev, per_tensor_rel, rel, t
from oracle import sgnn_numpy as ON

pytestmark = pytest.mark.gpu

TOL = 1e-4
SEED = SC.BATCH_SEED


def scaled_edge_mlp(flat, scale):
    out = flat.copy()
    for name in ("gcn0_w", "gcn1_w"):
        sl = PL.SLOTS[name]
        out[sl.offset:sl.offset + sl.size] *= scale
    return out


@pytest.fixture(scope="module")
def batch(dev):
    return SC.Batch(dev)


def check_against_oracle(eng, b, params_flat, dev, ids=None):
    """forward (value, log-prob, entropy) and ppo_grad (32 tensors + losses) of the whole batch against the oracle;
    returns the forward outputs."""
    ref = b.oracle(params_flat)
    params = t(params_flat, dev)
    ids_dev = None if ids is None else t(np.asarray(ids, np.int32), dev)
    out = eng.forward(b.blob, params, b.dev_args[0], ids=ids_dev, want_greedy=True)
    value, logp, ent, _ = (x.cpu().numpy() for x in out)
    assert rel(value, ref["value"]) < TOL
    assert rel(logp, ref["log_prob"]) < TOL
    assert rel(ent, ref["entropy"]) < TOL
    grad = eng.ppo_grad(b.blob, params, *b.dev_args, 1.0 / b.count, 1.0 / b.n_ind, ids=ids_dev)
    worst, where = per_tensor_rel(grad.cpu().numpy()[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)
    assert np.allclose(eng.read_losses(grad), [ref["loss"], ref["value_loss"], ref["surr_loss"], ref["entropy_loss"]],
                       rtol=1e-4, atol=1e-5)
    return out


def test_boundary_sweep_matches_oracle(batch, dev):
    b = batch
    n, e, k, stage = b.info.T
    # every threshold is met from both sides, each by the dimension that alone decides it
    for lim in (SC.XEARLY_NODES, SC.HIN_NODES, SC.NS):
        assert (n == lim).any() and (n == lim + 1).any(), lim
    assert ((n == SC.NS + 1) & (stage == 0)).any() and ((n == SC.NS + 1) & (stage == 1)).any()
    for twice_e in (SC.AS - 2, SC.AS, SC.AS + 2):
        assert ((2 * e == twice_e) & (n <= SC.NS)).any(), twice_e
    assert (e % 2 == 1).any()
    small = (n <= SC.NS) & (2 * e <= SC.AS)
    for kk in (SC.CH, SC.CH + 1, SC.KS, SC.KS + 1, 2 * SC.CH, 2 * SC.CH + 1):
        assert ((k == kk) & (stage == 0) & small).any(), kk
    assert ((k == SC.KS) & (stage == 1)).any() and ((k == SC.KS + 1) & (stage == 1)).any()
    assert {15, 16, 17} <= set(n.tolist())
    degs = [SC.degrees(st) for st in b.states]
    assert any(d.max() == len(d) - 1 for d in degs) and any((d == 0).any() for d in degs)
    assert b.big.any() and not b.big.all()

    eng = Engine(dev, b.blob.n_cap, b.blob.e_cap)
    assert eng.grid >= b.count                                          # one graph per CTA
    _, _, _, greedy = check_against_oracle(eng, b, b.flat, dev)
    greedy = greedy.cpu().numpy()
    # greedy: the oracle's arg-max, bit for bit; where its top probabilities are within 1e-6 (a near tie, rare), one of
    # those candidates
    P = ON._p64(b.flat)
    ties = 0
    for i, st in enumerate(b.states):
        c = ON.forward(P, ON.unpad(st), keep=True)["cache"]
        near = c["idx"][c["p"] >= c["p"].max() - 1e-6]
        ties += near.size > 1
        assert greedy[i] in near, (b.labels[i], greedy[i], near)
    assert ties <= 2, ties
    params = t(b.flat, dev)
    assert np.array_equal(eng.select_action(b.blob, params).cpu().numpy(), greedy)


def cta_walks(ids, grid):
    """The graph ids each CTA walks, in order (item i -> CTA i % grid)."""
    return [list(ids[c::grid]) for c in range(grid)]


def transitions(b, walk):
    big, k, stage = b.big, b.info[:, 2], b.info[:, 3]
    seen = set()
    for x, y in zip(walk, walk[1:]):
        if big[x] and k[x] > SC.KS and not big[y]:
            seen.add("big k -> small k")
        if stage[x] == 0 and stage[y] == 1:
            seen.add("land-use -> road")
    for x, y, z in zip(walk, walk[1:], walk[2:]):
        if not big[x] and big[y] and not big[z]:
            seen.add("fast -> big -> fast")
    return seen


@pytest.mark.parametrize("grid", [1, 2, 3])
def test_graphs_walked_by_one_cta_match_one_graph_per_cta(grid, batch, dev):
    """Between the graphs of one CTA the kernel carries state (mbarrier phase parity, shared regions sized by the
    previous graph, the prefetch of the next one).  Per graph there are no atomics and a fixed order, so every
    per-sample forward output must be bit-identical to the launch with one graph per CTA; gradients match the oracle.
    The second parameter set scales the edge MLP x20 so the first GCN layer switches between its one- and
    two-reciprocal forms from one graph to the next."""
    b = batch
    full = Engine(dev, b.blob.n_cap, b.blob.e_cap)
    eng = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid)
    assert eng.grid == grid and full.grid >= b.count
    walk = SC.walk_order(b)
    ids = SC.placed(walk, grid)
    walks = cta_walks(ids, grid)
    assert set().union(*(transitions(b, w) for w in walks)) == {"big k -> small k", "land-use -> road",
                                                                 "fast -> big -> fast"}
    saturated = scaled_edge_mlp(b.flat, 20.0)
    P = ON._p64(saturated)
    tier = np.array([EC.graph_reciprocal_tiers(P, st)[0] for st in b.states])     # first GCN layer
    sat_walk = [i for pair in zip(np.flatnonzero(tier == 1), np.flatnonzero(tier == 0)) for i in pair]
    sat_walk += [i for i in range(b.count) if i not in sat_walk]
    sat_ids = SC.placed(sat_walk, grid)
    assert any(tier[x] == 1 and tier[y] == 0 for w in cta_walks(sat_ids, grid) for x, y in zip(w, w[1:]))
    for flat, order in ((b.flat, ids), (saturated, sat_ids)):
        params = t(flat, dev)
        want = full.forward(b.blob, params, b.dev_args[0], want_greedy=True)
        got = check_against_oracle(eng, b, flat, dev, ids=order)
        for name, x, y in zip(("value", "log_prob", "entropy", "greedy"), got, want):
            assert torch.equal(x, y), (name, grid, np.flatnonzero((x != y).cpu().numpy()))


def fill_batch(b, count):
    """The boundary batch topped up to `count` graphs with ordinary hlg graphs (enough for every CTA of a full grid)."""
    more, more_actions = synth.make_states(SEED + 1, "hlg", count - b.count)
    states = b.states + more
    actions = np.concatenate([b.actions, more_actions])
    adv, ret, exps = synth.make_ppo_targets(SEED + 1, count)
    exps[7] = 0.0
    fixed = np.random.default_rng(SEED + 1).normal(-3.0, 0.3, size=(count, 1)).astype(np.float32)
    return states, actions, adv, ret, fixed, exps


@pytest.mark.parametrize("grid", [1, 2, 3, 7, 8, 57, 113, 114, 115, 0])
def test_fused_tail_at_every_grid_size(grid, batch, dev):
    """upb_ppo_step against upb_ppo_grad + upb_apply (tolerances of test_fused_step_matches_two_call_path) over 4 steps
    on a batch holding big graphs, at grid sizes that change how the 114 slices of 128 gradient columns are owned
    (slice s -> CTA s % grid): one CTA owning them all, several slices per CTA, one each with idle CTAs (113, 114,
    115), and the full grid (0).  The last CTA also chains the attention gradients (slices 107..113)."""
    count = 140
    states, actions, adv, ret, fixed, exps = fill_batch(batch, count)
    blob = pack_states(states).to(dev)
    assert (blob.info[:, 0] > SC.NS).any() and (blob.info[:, 2] > SC.KS).any()
    a = tuple(t(x, dev) for x in (actions, adv, ret, fixed, exps))
    n_ind = int((exps != 0).sum())
    flat = PL.default_init(SEED + 1)
    e1 = Engine(dev, blob.n_cap, blob.e_cap, grid_limit=grid)
    e2 = Engine(dev, blob.n_cap, blob.e_cap, grid_limit=grid)
    assert e2.grid == (grid or e2.grid) and e2.grid <= count
    p1, p2 = t(flat, dev).clone(), t(flat, dev).clone()
    for step in range(4):
        before = e2.launches
        g1 = e1.ppo_grad(blob, p1, *a, 1.0 / count, 1.0 / n_ind)
        e1.apply(p1, g1)
        g2 = e2.ppo_step(blob, p2, *a, 1.0 / count, 1.0 / n_ind)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (step > 0)                 # step 0 clips: two-call path
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (step, worst, where)
        assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, step
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    assert s1.tolist() == s2.tolist() == [4, 4, 4, 4]
    assert rel(m2, m1) < 1e-5 and rel(v2, v1) < 1e-5


def test_policy_head_liveness_across_fused_steps(batch, dev):
    """The stage bits of the fused tail are double-buffered by step parity (the word of parity p is cleared by the
    launch of parity p ^ 1).  Minibatches mixed -> mixed -> land-use only -> road only -> land-use only -> road only ->
    mixed: every single-head step comes two fused steps after one where the other head was live, so a stale word
    would apply Adam to the absent head.  Against the oracle's clip / Adam / live mask: parameter trajectory, the
    absent head's parameters and moments untouched, and the per-segment step counters."""
    b = batch
    stage = b.info[:, 3]
    lu, rd = np.flatnonzero(stage == 0), np.flatnonzero(stage == 1)
    mixed = np.arange(b.count)
    assert b.big[lu].any() and b.big[rd].any()
    plan = [mixed, mixed, lu, rd, lu, rd, mixed]
    heads = {0: slice(PL.SLOTS["lu_w0"].offset, PL.SLOTS["road_w0"].offset),
             1: slice(PL.SLOTS["road_w0"].offset, PL.POLICY_END)}
    eng = Engine(dev, b.blob.n_cap, b.blob.e_cap, clip_mode=_lib.CLIP_REFERENCE)
    params = t(b.flat, dev).clone()
    f64, m, v, tt = b.flat.astype(np.float64), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS)
    for step, sel in enumerate(plan):
        sub = [b.states[i] for i in sel]
        ref = b.oracle(f64, sel)
        g = ON.clip_groups(ref["grad"]) if step == 0 else ref["grad"]
        f64, m, v, tt = ON.adam_step(f64, m, v, tt, g, ON.live_mask(sub))
        p_before = params.cpu().numpy()
        m_before, v_before, _ = eng.get_opt_state()
        before = eng.launches
        n_ind = int((b.exps[sel] != 0).sum())
        eng.ppo_step(b.blob, params, *b.dev_args, 1.0 / len(sel), 1.0 / n_ind, ids=t(sel.astype(np.int32), dev))
        torch.cuda.synchronize()
        assert (eng.launches - before == 1) == (step > 0), step             # fused from the second step on
        p_now = params.cpu().numpy()
        assert rel(p_now, f64) < 1e-5, step
        m_now, v_now, steps = eng.get_opt_state()
        for s, sl in heads.items():
            if not (stage[sel] == s).any():
                assert np.array_equal(p_now[sl], p_before[sl]), (step, s)
                assert np.array_equal(m_now[sl], m_before[sl]) and np.array_equal(v_now[sl], v_before[sl]), (step, s)
        want = [step + 1, tt[0], tt[heads[0].start], tt[heads[1].start]]
        assert steps.tolist() == want, (step, steps.tolist(), want)
    assert steps.tolist() == [7, 7, 5, 5]


@pytest.mark.parametrize("mode", ["zero", "one", "random"])
def test_sampling_on_big_graphs(mode, batch, dev):
    """upb_select_action with uniforms on the boundary batch, which holds graphs with 161 and 3000 candidates: the
    picked index brackets u in the oracle's CDF (as in test_select_action_greedy_and_sampled)."""
    b = batch
    k = b.info[:, 2]
    assert ((k == SC.KS + 1) & b.big).any() and (k == 3000).any()
    u = {"zero": np.zeros(b.count, np.float32),
         "one": np.full(b.count, 1.0 - 2.0 ** -24, np.float32),
         "random": np.random.default_rng(11).random(b.count).astype(np.float32)}[mode]
    eng = Engine(dev, b.blob.n_cap, b.blob.e_cap)
    picked = eng.select_action(b.blob, t(b.flat, dev), uniforms=t(u, dev)).cpu().numpy()
    P = ON._p64(b.flat)
    for i, st in enumerate(b.states):
        c = ON.forward(P, ON.unpad(st), keep=True)["cache"]
        idx, p = c["idx"], c["p"]
        assert picked[i] in idx, (b.labels[i], picked[i])
        j = int(np.flatnonzero(idx == picked[i])[0])
        cdf = np.cumsum(p)
        lo = cdf[j - 1] if j > 0 else 0.0
        assert lo - 1e-5 <= float(u[i]) <= cdf[j] + 1e-5, (b.labels[i], j, lo, float(u[i]), cdf[j])


def test_mlp_boundary_batch_in_one_cta_matches_oracle_port(batch, dev):
    """k_mlp has the same 464 / 5632 / 160 split: the boundary batch, fast and big graphs alternating in ONE CTA,
    against the oracle port (autograd on the padded states), as
    test_mlp_large_graphs_and_edge_cases_match_oracle_port does."""
    from oracle import mlp_port as MP
    b = batch
    L = PL.MLP
    flat = L.default_init(SEED)
    eng = Engine(dev, b.blob.n_cap, b.blob.e_cap, model="mlp", grid_limit=1)
    assert eng.grid == 1
    walk = SC.walk_order(b)          # k_mlp's M_NS / M_AS / M_KS are the SGNN kernel's NS / AS / KS (static_asserts)
    assert {"fast -> big -> fast", "big k -> small k", "land-use -> road"} <= transitions(b, walk)
    ids = t(np.array(walk, np.int32), dev)
    params = t(flat, dev)
    value, logp, ent, greedy = eng.forward(b.blob, params, b.dev_args[0], ids=ids, want_greedy=True)
    grad = eng.ppo_grad(b.blob, params, *b.dev_args, 1.0 / b.count, 1.0 / b.n_ind, ids=ids)
    torch.cuda.synchronize()
    agent = MP.MLPPortAgent(flat)
    pb = MP.stack_states(b.states)
    act = torch.tensor(b.actions)
    ind = torch.tensor(b.exps).nonzero(as_tuple=False).squeeze(1)
    with torch.no_grad():
        v_ref = MP.value(agent.P, pb).numpy().ravel()
        lp_ref, en_ref = MP.log_prob_entropy(agent.P, pb, act)
        gr_ref = MP.greedy_action(agent.P, pb).numpy()
    losses = agent.backward(pb, act, torch.tensor(b.adv), torch.tensor(b.ret), torch.tensor(b.fixed), ind)
    assert rel(value.cpu().numpy(), v_ref) < TOL
    assert rel(logp.cpu().numpy(), lp_ref.numpy().ravel()) < TOL
    assert rel(ent.cpu().numpy(), en_ref.numpy().ravel()) < TOL
    # greedy: the port's arg-max; where its top probabilities are within 1e-6, one of those candidates.  Ties are not
    # rare here: the rl-mlp scores a land-use edge from one endpoint's features, so edges sharing it tie exactly.
    with torch.no_grad():
        zl, zr = MP.masked_logits(agent.P, pb)
    greedy = greedy.cpu().numpy()
    for i, s in enumerate(b.info[:, 3]):
        p = torch.softmax((zl if s == 0 else zr)[i].double(), -1).numpy()
        near = np.flatnonzero(p >= p.max() - 1e-6)
        assert int(gr_ref[i, s]) in near
        assert greedy[i] in near, (b.labels[i], greedy[i], near)
    assert np.allclose(eng.read_losses(grad), losses, rtol=1e-4, atol=1e-5)
    worst, where = per_tensor_rel(grad.cpu().numpy()[:L.num_params], agent.flat_grad(), L)
    assert worst < TOL, (worst, where)
