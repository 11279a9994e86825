"""GPU (H100): the CUDA path, called through the C ABI, against
  (a) the golden vectors produced by the unmodified reference (tests/golden/*.npz), and
  (b) the float64 numpy oracle on seeded synthetic minibatches.
Tolerance: per-tensor max|delta| / max|ref| <= 1e-4 (the task's fp32 bar; observed ~1e-6), integer action
indices and GAE bit-exact."""
import numpy as np
import pytest
import torch

import cross_path as XP
import extreme_cases as EC
import shape_cases as SC
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from harness import Case, dev, load, per_tensor_rel, rel, t
from oracle import sgnn_numpy as ON

pytestmark = pytest.mark.gpu

TOL = 1e-4
FIXTURES = ["tiny_mixed", "small_mixed", "hlg", "concept", "caps_concept"]


def make_engine(dev, n_cap, e_cap, **kw):
    from drl_urban_planning_b200.engine import Engine
    return Engine(dev, n_cap, e_cap, **kw)


@pytest.mark.parametrize("name", FIXTURES)
def test_forward_matches_reference_golden(name, golden_dir, dev):
    z = load(golden_dir, name)
    states = expand_states(z)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(z["params"], dev)
    value, logp, ent, greedy = eng.forward(blob, params, t(z["actions"], dev), want_greedy=True)
    torch.cuda.synchronize()
    assert rel(value.cpu().numpy(), z["values"].ravel()) < TOL
    assert rel(logp.cpu().numpy(), z["log_probs"].ravel()) < TOL
    assert rel(ent.cpu().numpy(), z["entropies"].ravel()) < TOL
    stage = z["stage"][:, :2].argmax(1)
    want = z["greedy"][np.arange(len(states)), stage].astype(np.int64)
    assert np.array_equal(greedy.cpu().numpy().astype(np.int64), want)      # bit-exact action indices


@pytest.mark.parametrize("name", FIXTURES)
def test_gradient_and_steps_match_reference_golden(name, golden_dir, dev):
    z = load(golden_dir, name)
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE)
    params = t(z["params"], dev).clone()
    n_ind = int((z["exps"] != 0).sum())
    args = (t(z["actions"], dev), t(z["advantages"], dev), t(z["returns"], dev), t(z["fixed_log_probs"], dev),
            t(z["exps"], dev))
    for k in range(3):
        grad = eng.ppo_grad(blob, params, *args, 1.0 / B, 1.0 / n_ind)
        losses = eng.read_losses(grad)
        g = grad.cpu().numpy()
        assert np.allclose(losses, z["losses"][k], rtol=1e-4, atol=1e-5), (k, losses, z["losses"][k])
        worst, where = per_tensor_rel(g[:PL.NUM_PARAMS], z["grads"][k])
        assert worst < TOL, (k, worst, where)
        st = g[_lib.UPB_STAT_OFFSET:_lib.UPB_STAT_OFFSET + 8]
        assert st[3] == B and st[4] == n_ind and st[7] == 0
        eng.apply(params, grad)
        torch.cuda.synchronize()
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k


@pytest.mark.parametrize("name", ["hlg256", "dhm256", "grid64", "concept_mixed256"])
def test_baseline_size_minibatch_matches_reference_golden(name, golden_dir, dev):
    """BASELINE.json sizes (HLG / DHM, 256 graphs per minibatch; the two-stage grid community; hlg_concept + dhm_concept
    mixed in one minibatch, where graphs beyond the shared-memory fast path share the launch with fast ones) against
    vectors produced by the unmodified reference: forward values, then three optimiser steps through upb_ppo_step
    exactly as the product runs them (ids in the LPT order of Engine.balance_ids, full grid of CTAs, fused tail from
    step 2 on; step 1 clips and takes the two-call path like the reference's first step): losses, all 32 gradients and
    the parameter trajectory."""
    from drl_urban_planning_b200.engine import Engine
    from fixtures_io import states_digest, synth_states
    z = load(golden_dir, name)
    states, actions = synth_states(int(z["seed"]), str(z["community"]), int(z["count"]))
    assert states_digest(states) == str(z["digest"]), "synth.py no longer reproduces the fixture's states"
    assert np.array_equal(actions, z["actions"])
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE)
    params = t(z["params"], dev).clone()
    value, logp, ent, greedy = eng.forward(blob, params, t(z["actions"], dev), want_greedy=True)
    assert rel(value.cpu().numpy(), z["values"].ravel()) < TOL
    assert rel(logp.cpu().numpy(), z["log_probs"].ravel()) < TOL
    assert rel(ent.cpu().numpy(), z["entropies"].ravel()) < TOL
    stage = np.array([int(s[8][:2].argmax()) for s in states])
    assert np.array_equal(greedy.cpu().numpy().astype(np.int64), z["greedy"][np.arange(B), stage].astype(np.int64))
    n_ind = int((z["exps"] != 0).sum())
    args = (t(z["actions"], dev), t(z["advantages"], dev), t(z["returns"], dev), t(z["fixed_log_probs"], dev),
            t(z["exps"], dev))
    ids = eng.balance_ids(np.arange(B), Engine.graph_cost(blob.info.astype(np.int64)))
    ids_dev = t(ids.astype(np.int32), dev)
    launches = []
    for k in range(3):
        before = eng.launches
        grad = eng.ppo_step(blob, params, *args, 1.0 / B, 1.0 / n_ind, ids=ids_dev)
        launches.append(eng.launches - before)
        losses = eng.read_losses(grad)
        g = grad.cpu().numpy()
        assert np.allclose(losses, z["losses"][k], rtol=1e-4, atol=1e-5), (k, losses, z["losses"][k])
        worst, where = per_tensor_rel(g[:PL.NUM_PARAMS], z["grads"][k])
        assert worst < TOL, (k, worst, where)
        st = g[_lib.UPB_STAT_OFFSET:_lib.UPB_STAT_OFFSET + 8]
        assert st[3] == B and st[4] == n_ind and st[7] == 0
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k
    assert launches == [3, 1, 1]       # clipping step: kernel + reduce + apply; then one cooperative launch per step


@pytest.mark.parametrize("community,count,seed", [("tiny", 64, 1), ("small", 48, 2), ("grid", 12, 3), ("dhm", 6, 4)])
def test_matches_numpy_oracle(community, count, seed, dev):
    states, actions = synth.make_states(seed, community, count)
    adv, ret, exps = synth.make_ppo_targets(seed, count)
    exps[::5] = 0.0
    flat = PL.default_init(seed)
    rng = np.random.default_rng(seed)
    fixed = rng.normal(-3.0, 0.3, size=(count, 1)).astype(np.float32)
    ref = ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    value, logp, ent = eng.forward(blob, params, t(actions, dev))
    assert rel(value.cpu().numpy(), ref["value"]) < TOL
    assert rel(logp.cpu().numpy(), ref["log_prob"]) < TOL
    assert rel(ent.cpu().numpy(), ref["entropy"]) < TOL
    n_ind = int((exps != 0).sum())
    grad = eng.ppo_grad(blob, params, t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev),
                        1.0 / count, 1.0 / n_ind)
    g = grad.cpu().numpy()
    worst, where = per_tensor_rel(g[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)
    losses = eng.read_losses(grad)
    assert np.allclose(losses, [ref["loss"], ref["value_loss"], ref["surr_loss"], ref["entropy_loss"]],
                       rtol=1e-4, atol=1e-5)


def _reciprocal_tiers(flat, states):
    """Per GCN layer, the set of forms (graph_reciprocal_tiers) the kernel will pick over the batch."""
    P = ON._p64(flat)
    tiers = [set(), set()]
    for st in states:
        for l, tier in enumerate(EC.graph_reciprocal_tiers(P, st)):
            tiers[l].add(tier)
    return tiers


@pytest.mark.parametrize("scale,want", [(10.0, {0}), (20.0, {0, 1}), (30.0, {1})])
def test_saturated_edge_activations_match_numpy_oracle(scale, want, dev):
    """The pulls compute both tanh terms of an entry from ONE reciprocal while the product of their denominators
    cannot overflow, and from two otherwise; the form is picked per graph and layer from the measured
    |pre-activation|.  Edge-MLP weights scaled up walk a batch through both forms (checked from the oracle's own
    activations), up to near the exp-form's clamp, and values / log-probs / entropies / gradients stay within the
    fp32 bar of the float64 oracle."""
    count, seed = 24, 5
    states, actions = synth.make_states(seed, "small", count)
    adv, ret, exps = synth.make_ppo_targets(seed, count)
    flat = PL.default_init(seed).copy()
    for name in ("gcn0_w", "gcn1_w"):
        sl = PL.SLOTS[name]
        flat[sl.offset:sl.offset + sl.size] *= scale
    tiers = _reciprocal_tiers(flat, states)
    assert want <= (tiers[0] | tiers[1]), tiers
    fixed = np.random.default_rng(seed).normal(-3.0, 0.3, size=(count, 1)).astype(np.float32)
    ref = ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    value, logp, ent = eng.forward(blob, params, t(actions, dev))
    assert rel(value.cpu().numpy(), ref["value"]) < TOL
    assert rel(logp.cpu().numpy(), ref["log_prob"]) < TOL
    assert rel(ent.cpu().numpy(), ref["entropy"]) < TOL
    grad = eng.ppo_grad(blob, params, t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev),
                        1.0 / count, 1.0 / int((exps != 0).sum()))
    worst, where = per_tensor_rel(grad.cpu().numpy()[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)


def test_large_graph_path_matches_numpy_oracle(dev):
    count = 5
    states, actions = SC.big_states(9, count)
    adv, ret, exps = synth.make_ppo_targets(9, count)
    flat = PL.default_init(9)
    fixed = np.full((count, 1), -4.0, np.float32)
    ref = ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)
    blob = pack_states(states).to(dev)
    info = blob.info
    assert (info[:, 0] > 464).any() and (info[:, 2] > 160).any()
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    value, logp, ent = eng.forward(blob, params, t(actions, dev))
    assert rel(value.cpu().numpy(), ref["value"]) < TOL
    assert rel(logp.cpu().numpy(), ref["log_prob"]) < TOL
    assert rel(ent.cpu().numpy(), ref["entropy"]) < TOL
    grad = eng.ppo_grad(blob, params, t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev),
                        1.0 / count, 1.0 / count)
    worst, where = per_tensor_rel(grad.cpu().numpy()[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)


def test_edge_cases_match_numpy_oracle(dev):
    """single-node graph, empty candidate mask, all-edges mask, action outside the mask."""
    spec = synth.COMMUNITIES["tiny"]
    rng = np.random.default_rng(0)
    s0, a0 = synth.make_state(rng, spec, n=2, stage=1, e=1)
    s1, a1 = synth.make_state(rng, spec, n=spec.max_num_nodes, stage=0)
    s2, _ = synth.make_state(rng, spec, n=10, stage=0); s2[6][:] = False
    s3, _ = synth.make_state(rng, spec, n=12, stage=0); s3[6][:int(s3[5].sum())] = True
    s4, a4 = synth.make_state(rng, spec, n=15, stage=1)
    states = [s0, s1, s2, s3, s4]
    actions = np.zeros((5, 2), np.float32)
    actions[0, 1], actions[1, 0], actions[2, 0], actions[3, 0], actions[4, 1] = a0, a1, 0, 3, a4
    adv, ret, exps = synth.make_ppo_targets(3, 5)
    flat = PL.default_init(4)
    fixed = np.full((5, 1), -2.0, np.float32)
    ref = ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    value, logp, ent = eng.forward(blob, params, t(actions, dev))
    assert rel(value.cpu().numpy(), ref["value"]) < TOL
    assert rel(logp.cpu().numpy(), ref["log_prob"]) < TOL
    assert rel(ent.cpu().numpy(), ref["entropy"]) < TOL
    grad = eng.ppo_grad(blob, params, t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev),
                        1.0 / 5, 1.0 / 5)
    worst, where = per_tensor_rel(grad.cpu().numpy()[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)


def test_minibatch_as_index_list_and_determinism(dev):
    """A minibatch is an index list into a resident blob; grads do not depend on the CTA count beyond fp32
    summation order, and two identical launches are bit-identical."""
    count = 96
    states, actions = synth.make_states(21, "small", count)
    adv, ret, exps = synth.make_ppo_targets(21, count)
    flat = PL.default_init(21)
    fixed = np.full((count, 1), -3.5, np.float32)
    blob = pack_states(states).to(dev)
    params = t(flat, dev)
    ids = torch.tensor(np.random.default_rng(0).permutation(count)[:40].astype(np.int32), device=dev)
    sub = [states[i] for i in ids.cpu().numpy()]
    sel = ids.cpu().numpy()
    ref = ON.ppo_minibatch(flat, sub, actions[sel], adv[sel], ret[sel], fixed[sel], exps[sel])
    a = (t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev))
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    g1 = eng.ppo_grad(blob, params, *a, 1.0 / 40, 1.0 / 40, ids=ids).clone()
    g2 = eng.ppo_grad(blob, params, *a, 1.0 / 40, 1.0 / 40, ids=ids).clone()
    assert torch.equal(g1, g2)
    worst, where = per_tensor_rel(g1.cpu().numpy()[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)
    eng1 = make_engine(dev, blob.n_cap, blob.e_cap, grid_limit=3)      # 3 CTAs walk 40 graphs
    g3 = eng1.ppo_grad(blob, params, *a, 1.0 / 40, 1.0 / 40, ids=ids)
    worst, where = per_tensor_rel(g3.cpu().numpy()[:PL.NUM_PARAMS], ref["grad"])
    assert worst < TOL, (worst, where)
    v, lp, en = eng.forward(blob, params, a[0], ids=ids)
    untouched = np.setdiff1d(np.arange(count), sel)
    assert not v.cpu().numpy()[untouched].any()
    assert rel(v.cpu().numpy()[sel], ref["value"]) < TOL


def test_clip_modes_and_head_skipping(dev):
    """CLIP_ALWAYS clips every step; a policy head whose stage is absent is not touched by Adam."""
    count = 16
    states, actions = synth.make_states(31, "small", count, stages=[0] * count)    # land-use only
    adv, ret, exps = synth.make_ppo_targets(31, count)
    flat = PL.default_init(31)
    fixed = np.full((count, 1), -3.0, np.float32)
    blob = pack_states(states).to(dev)
    a = (t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev))
    eng = make_engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_ALWAYS)
    params = t(flat, dev).clone()
    f64, m, v, tt = flat.astype(np.float64), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS), np.zeros(PL.NUM_PARAMS)
    live = ON.live_mask(states)
    assert not live[PL.SLOTS["road_w0"].offset]
    for _ in range(2):
        ref = ON.ppo_minibatch(f64, states, actions, adv, ret, fixed, exps)
        f64, m, v, tt = ON.adam_step(f64, m, v, tt, ON.clip_groups(ref["grad"]), live)
        grad = eng.ppo_grad(blob, params, *a, 1.0 / count, 1.0 / count)
        eng.apply(params, grad)
        assert rel(params.cpu().numpy(), f64) < 1e-5
    road = slice(PL.SLOTS["road_w0"].offset, PL.POLICY_END)
    assert np.array_equal(params.cpu().numpy()[road], flat[road])
    mm, vv, steps = eng.get_opt_state()
    assert steps.tolist() == [2, 2, 2, 0] and not mm[road].any()
    eng.set_opt_state(mm, vv, steps)
    assert eng.get_opt_state()[2].tolist() == [2, 2, 2, 0]


def test_gae_bit_exact(golden_dir, dev):
    z = load(golden_dir, "gae")
    eng = make_engine(dev, 64, 64)
    for tag, (gamma, tau) in {"g1t0": (1.0, 0.0), "g99t95": (0.99, 0.95)}.items():
        adv, ret = eng.gae(t(z["rewards"], dev), t(z["masks"], dev), t(z["values"], dev), gamma, tau)
        assert np.array_equal(adv.cpu().numpy(), z[f"adv_{tag}"].ravel()), tag
        assert np.array_equal(ret.cpu().numpy(), z[f"ret_{tag}"].ravel()), tag
    # one unbroken trajectory (no episode ends): still the reference's sequential scan
    rng = np.random.default_rng(5)
    r, v = rng.standard_normal(3000).astype(np.float32), rng.standard_normal(3000).astype(np.float32)
    mk = np.ones(3000, np.float32)
    a_ref, r_ref = ON.estimate_advantages(r, mk, v, 0.99, 0.95)
    adv, ret = eng.gae(t(r, dev), t(mk, dev), t(v, dev), 0.99, 0.95)
    assert np.array_equal(adv.cpu().numpy(), a_ref.ravel()) and np.array_equal(ret.cpu().numpy(), r_ref.ravel())


def test_full_size_minibatch_properties(dev):
    """BASELINE config 2 at full size (HLG, B=256): size-independent properties instead of the slow oracle --
    (1) shards sum to the batch gradient (the multi-GPU decomposition), (2) permutation invariance,
    (3) probabilities normalise: entropy <= log(k), log-prob <= 0, (4) a 32-graph sample agrees with the oracle."""
    count = 256
    states, actions = synth.make_states(111, "hlg", count)
    adv, ret, exps = synth.make_ppo_targets(111, count)
    flat = PL.default_init(111)
    fixed = np.full((count, 1), -4.0, np.float32)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    a = (t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev))
    full = eng.ppo_grad(blob, params, *a, 1.0 / count, 1.0 / count).clone()
    parts = torch.zeros_like(full)
    for lo in range(0, count, 64):
        ids = torch.arange(lo, lo + 64, dtype=torch.int32, device=dev)
        parts += eng.ppo_grad(blob, params, *a, 1.0 / count, 1.0 / count, ids=ids)
    worst, where = per_tensor_rel(parts.cpu().numpy()[:PL.NUM_PARAMS], full.cpu().numpy()[:PL.NUM_PARAMS])
    assert worst < 1e-5, (worst, where)
    perm = torch.tensor(np.random.default_rng(1).permutation(count).astype(np.int32), device=dev)
    shuffled = eng.ppo_grad(blob, params, *a, 1.0 / count, 1.0 / count, ids=perm)
    worst, where = per_tensor_rel(shuffled.cpu().numpy()[:PL.NUM_PARAMS], full.cpu().numpy()[:PL.NUM_PARAMS])
    assert worst < 1e-5, (worst, where)
    v, lp, en = eng.forward(blob, params, a[0])
    k = blob.info[:, 2]
    assert (lp.cpu().numpy() <= 1e-6).all() and (en.cpu().numpy() <= np.log(k) + 1e-4).all()
    sel = np.arange(0, count, 8)
    ref = ON.ppo_minibatch(flat, [states[i] for i in sel], actions[sel], adv[sel], ret[sel], fixed[sel], exps[sel],
                           want_grad=False)
    assert rel(v.cpu().numpy()[sel], ref["value"]) < TOL
    assert rel(lp.cpu().numpy()[sel], ref["log_prob"]) < TOL
    assert rel(en.cpu().numpy()[sel], ref["entropy"]) < TOL


def test_fused_step_matches_two_call_path(dev):
    """upb_ppo_step against upb_ppo_grad + upb_apply (cross_path.check_sgnn_fused_against_two_call) at the shipped
    settings and the full grid, on mixed stages and on a land-use-only batch (a head that never fires)."""
    for stages in (None, [0] * 64):
        states, actions = synth.make_states(51, "small", 64, stages=stages)
        c = Case(dev, "sgnn", states, actions, 51, zero_exps=(3,), fixed=np.full((64, 1), -3.2, np.float32))
        XP.check_sgnn_fused_against_two_call(c, "shipped", 0)


def test_select_action_greedy_and_sampled(dev):
    """upb_select_action (policy.py:67-85): greedy = the forward kernel's arg-max (bit-exact); sampled = inverse CDF of
    the float64 oracle's candidate probabilities at the supplied uniform (the index must bracket u up to fp32 rounding
    of the cumulative sums), including u = 0, u -> 1 and an empty action mask."""
    states, actions = synth.make_states(21, "small", 40)
    states[3][6][:] = False; states[3][7][:] = False                      # empty mask: uniform over the padded width
    flat = PL.default_init(21)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    _, _, _, greedy = eng.forward(blob, params, t(actions, dev), want_greedy=True)
    assert torch.equal(eng.select_action(blob, params), greedy.to(torch.int32))
    rng = np.random.default_rng(5)
    u = rng.random(len(states)).astype(np.float32)
    u[0], u[1] = 0.0, np.float32(1.0 - 2.0 ** -24)
    picked = eng.select_action(blob, params, uniforms=t(u, dev)).cpu().numpy()
    P = ON._p64(flat)
    for i, st in enumerate(states):
        g = ON.unpad(st)
        c = ON.forward(P, g, keep=True)["cache"]
        idx, p = c["idx"], c["p"]
        if idx.size == 0:
            cap = blob.e_cap if st[8][0] > 0 else blob.n_cap
            assert picked[i] == min(cap - 1, int(u[i] * cap))
            continue
        assert picked[i] in idx, i
        j = int(np.flatnonzero(idx == picked[i])[0])
        cdf = np.cumsum(p)
        lo = cdf[j - 1] if j > 0 else 0.0
        assert lo - 1e-5 <= float(u[i]) <= cdf[j] + 1e-5, (i, j, lo, float(u[i]), cdf[j])
    # a subset through an index list leaves the other slots untouched (zero-initialised output)
    ids = torch.as_tensor(np.array([5, 7, 11], np.int32), device=dev)
    part = eng.select_action(blob, params, uniforms=t(u, dev), ids=ids).cpu().numpy()
    assert np.array_equal(part[[5, 7, 11]], picked[[5, 7, 11]]) and part[[0, 1, 2]].tolist() == [0, 0, 0]


def test_empty_action_masks_match_reference(golden_dir, dev):
    """The reference's fp32 behaviour on an all-masked state (log_prob = 0, entropy = 0, arg-max = 0), both stages, for
    the SGNN kernel; the rl-mlp kernel shares the code path (tests/test_mlp.py)."""
    z = load(golden_dir, "edge_empty")
    states = expand_states(z)
    blob = pack_states(states).to(dev)
    eng = make_engine(dev, blob.n_cap, blob.e_cap)
    value, logp, ent, greedy = eng.forward(blob, t(z["params"], dev), t(z["actions"], dev), want_greedy=True)
    assert rel(value.cpu().numpy(), z["values"].ravel()) < TOL
    assert np.allclose(logp.cpu().numpy(), z["log_probs"].ravel(), rtol=1e-4, atol=1e-7)
    assert np.allclose(ent.cpu().numpy(), z["entropies"].ravel(), rtol=1e-4, atol=1e-7)
    stage = z["stage"][:, :2].argmax(1)
    assert np.array_equal(greedy.cpu().numpy(), z["greedy"][np.arange(3), stage].astype(np.int64))
