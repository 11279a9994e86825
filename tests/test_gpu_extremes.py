"""GPU (H100): the training kernels at the magnitudes a trained policy reaches, against the float64 oracles
(oracle/sgnn_numpy.py for the SGNN; oracle/mlp_port.py run in float64, gradients by autograd, for the rl-mlp), and
against vectors recorded by the unmodified reference in the same regimes (tests/golden/make_golden_extremes.py).

Regimes (parameter transforms and batches in tests/extreme_cases.py), each checked from the oracle's own float64
activations:
  * GCN edge factors beyond exp2a's clamp (|P|, |Q| > 40) with moderate edge pre-activations P_u + Q_v -- the edge MLP
    reading the difference of its endpoints' embeddings, which share a common offset -- on either layer and on both,
    land-use and road graphs, the shared-memory and the large-graph path, straddling the clamp in one launch.  The
    kernel keeps the raw pre-activations for such graphs (tier 2 of the EPQ phase, sgnn_kernel.cuh);
  * factors and edge pre-activations both beyond the clamp: tanh saturates at +-1 and its gradient is 0;
  * peaked attention (logits spanning more than 104, where fp32 exp underflows), with two nodes tied at the maximum;
  * peaked policy heads in training: arg-max, zero-probability and masked actions, the ratio inside, below, above the
    clip range and underflowing to 0, each with A > 0, A < 0 and A = 0 (both models);
  * saturated tanh units (numeric encoder, value head, policy-head hidden layer past |9|, where fp32 tanh is +-1);
  * the fused step on a beyond-clamp batch, and the non-finite guard.

Bars: gradients per tensor max|delta| / max|float64| < 1e-4 (the suite's), except on a golden batch where the
reference's own recorded gradient of that tensor is further than 5e-5 from float64: there twice the reference's
deviation; values and entropies |delta| <= 1e-4 max|ref| over the batch; log-probs lp_tol (tail log-probs of -150
need a relative bar); greedy picks equal the float64 arg-max away from near-ties; one Adam step within 1e-5."""
import os

import numpy as np
import pytest
import torch

import extreme_cases as EC
from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from test_gpu_parity import per_tensor_rel, t
from test_gpu_select import LOG_TINY, lp_tol

pytestmark = pytest.mark.gpu

TOL = 1e-4
GOLDEN = {name: (mlp, case) for name, _, mlp, case in EC.FIXTURES}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need an H100"
    return torch.device("cuda", 0)


def tensor_errors(model, g, want):
    """Per tensor max|delta| / max|want|; tensors whose error is below 1e-7 x the largest entry of `want` (fp32
    cancellation noise on near-zero tensors, as in test_gpu_parity.per_tensor_rel) count as 0."""
    floor = 1e-7 * max(np.abs(want).max(), 1e-9)
    out = {}
    for s in (PL.SLOTS if model == "sgnn" else PL.MLP.slots).values():
        a, b = np.asarray(g[s.offset:s.offset + s.size], np.float64), want[s.offset:s.offset + s.size]
        d = np.abs(a - b).max()
        out[s.name] = 0.0 if d <= floor else float(d / max(np.abs(b).max(), 1e-30))
    return out


def check(dev, model, flat, states, actions, adv, ret, fixed, exps, bars=None):
    """Forward, ppo_grad (all tensors, loss statistics, non-finite count) and one apply against the float64 oracle.
    `bars`: per-tensor gradient bars replacing TOL.  Returns the kernel's gradient."""
    ref = (EC.sgnn_reference if model == "sgnn" else EC.mlp_reference)(flat, states, actions, adv, ret, fixed, exps)
    bars = bars or {}
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    params = t(flat, dev).clone()
    value, logp, ent, greedy = eng.forward(blob, params, t(actions, dev), want_greedy=True)
    value, logp, ent = (x.cpu().numpy().astype(np.float64) for x in (value, logp, ent))
    dv, de = np.abs(value - ref["value"]), np.abs(ent - ref["entropy"])
    assert dv.max() <= TOL * np.abs(ref["value"]).max(), ("value", int(dv.argmax()), dv.max())
    assert de.max() <= TOL * max(np.abs(ref["entropy"]).max(), 1e-6), ("entropy", int(de.argmax()), de.max())
    finite = np.abs(ref["log_prob"]) < 2.0 ** 31          # a masked action's log-prob is the fill value, ulp 512
    dl = np.abs(logp - ref["log_prob"]) - lp_tol(ref["log_prob"], np.asarray(ref["zabs"]))
    assert (dl[finite] <= 0).all(), ("log_prob", np.flatnonzero(finite & (dl > 0))[:8])
    assert np.allclose(logp[~finite], ref["log_prob"][~finite], rtol=1e-6)
    keep = ~np.asarray(ref["tie"])
    assert np.array_equal(greedy.cpu().numpy()[keep], np.asarray(ref["greedy"])[keep]), "greedy"
    n_ind = max(int((exps != 0).sum()), 1)
    grad = eng.ppo_grad(blob, params, t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev),
                        1.0 / B, 1.0 / n_ind)
    g = grad.cpu().numpy()
    nparam = PL.NUM_PARAMS if model == "sgnn" else PL.MLP.num_params
    bad = {k: e for k, e in tensor_errors(model, g[:nparam], ref["grad"]).items() if e >= bars.get(k, TOL)}
    assert not bad, (bad, {k: bars.get(k, TOL) for k in bad})
    assert np.allclose(eng.read_losses(grad), [ref["loss"], ref["value_loss"], ref["surr_loss"], ref["entropy_loss"]],
                       rtol=1e-4, atol=1e-5)
    st = g[eng.stat_offset:eng.stat_offset + 8]
    assert st[3] == B and st[4] == int((exps != 0).sum()) and st[7] == 0, st
    eng.apply(params, grad)
    d = np.abs(params.cpu().numpy() - ref["after"])
    assert d.max() <= 1e-5 * np.abs(ref["after"]).max(), ("apply", int(d.argmax()), d.max())
    return g[:nparam], ref


def seeded_batch(seed, states):
    adv, ret, exps = EC.targets(seed, len(states))
    fixed = np.random.default_rng(seed).normal(-3.0, 0.3, size=(len(states), 1)).astype(np.float32)
    return adv, ret, fixed, exps


# ---------------------------------------------------------------------------------------------------- regimes
def tier(amax):
    """The form of the pull's tanh terms the kernel picks for a layer (sgnn_kernel.cuh epq_phase): 0 = one shared
    reciprocal (<= 10.9, as test_gpu_parity.graph_reciprocal_tiers), 1 = two, 2 = raw pre-activations (beyond the
    clamp)."""
    return 0 if amax <= 10.9 else 1 if amax <= EC.CLAMP else 2


def assert_beyond_clamp(flat, states, layers):
    """From the float64 activations: every form occurs, some graph lies in [38, 40) and some beyond the clamp on each
    layer in `layers` (both stages), while edge pre-activations stay below it."""
    P = ON._p64(flat)
    am = [EC.edge_amax(P, st) for st in states]
    amax, emax = np.array([[a for a, _ in x] for x in am]), np.array([[e for _, e in x] for x in am])
    stage = np.array([int(np.argmax(st[8][:2])) for st in states])
    top = amax[:, layers].max(1)
    assert {tier(a) for a in amax.ravel()} == {0, 1, 2}, amax
    assert ((top >= 38.0) & (top < EC.CLAMP)).any(), top
    for l in layers:
        for s in (0, 1):
            assert (amax[stage == s, l] > EC.CLAMP).any(), (l, s, amax[:, l])
    assert emax.max() < 20.0, emax


def pre_activations(model, flat, states):
    """Float64 pre-activations of the numeric encoder, value head and policy-head hidden layers over the batch."""
    if model == "sgnn":
        P = ON._p64(flat)
        pre = {k: [] for k in ("num", "val", "head")}
        for st in states:
            fw = ON.forward(P, ON.unpad(st), keep=True)
            c = fw["cache"]
            pre["num"] += [P["num_w0"] @ ON.unpad(st).numerical + P["num_b0"], P["num_w1"] @ c["a0"] + P["num_b1"]]
            pre["val"] += [P["val_w0"] @ c["sv"] + P["val_b0"], P["val_w1"] @ c["y0"] + P["val_b1"]]
            if c["idx"].size:
                w0, b0 = ("lu_w0", "lu_b0") if fw["stage_id"] == 0 else ("road_w0", "road_b0")
                pre["head"].append((c["xin"] @ P[w0].T + P[b0]).ravel())
        return {k: np.concatenate(v) for k, v in pre.items()}
    P = MP.params_from_flat(flat, torch.float64)
    b = MP.stack_states(states)
    with torch.no_grad():
        lu, hn, sv = MP.encode(P, b)
        a0 = b["numerical"].double() @ P["num_w0"].T + P["num_b0"]
        a1 = torch.tanh(a0) @ P["num_w1"].T + P["num_b1"]
        y0 = sv @ P["val_w0"].T + P["val_b0"]
        y1 = torch.tanh(y0) @ P["val_w1"].T + P["val_b1"]
        hl = (lu @ P["lu_w0"].T + P["lu_b0"])[b["land_use_mask"]]
        hr = (hn @ P["road_w0"].T + P["road_b0"])[b["road_mask"]]
    cat = lambda *x: np.concatenate([np.asarray(v).ravel() for v in x])
    return {"num": cat(a0, a1), "val": cat(y0, y1), "head": cat(hl, hr)}


def assert_regime(name, model, flat, states, actions, fixed, adv):
    """The golden batch `name` is in its regime, from the oracle's float64 activations."""
    if name == "extreme_clamp":
        info = pack_states(states).info
        assert (info[:, 0] > 464).any() and (info[:, 0] <= 464).any()
        assert_beyond_clamp(flat, states, [0, 1])
    elif name == "extreme_attention":
        P = ON._p64(flat)
        spans = [np.ptp(EC.attention_logits(P, st)) for st in states]
        assert min(spans) > 104.0, spans
        s = EC.attention_logits(P, states[-1])
        top = np.sort(s)
        assert np.isclose(top[-1], top[-2], rtol=1e-12, atol=0) and top[-3] < top[-1] - 1.0
    elif name.endswith("heads"):
        heads = EC.head_logits(model, flat, states)
        assert np.median([np.ptp(z) for idx, z in heads if idx.size > 1]) > 104.0
        seen = set()
        for i, st in enumerate(states):
            stage = int(np.argmax(st[8][:2]))
            idx, lp = heads[i][0], EC.log_softmax(heads[i][1])
            j = int(actions[i, stage])
            if j not in idx:
                seen.add(("masked", None, float(adv[i])))
                continue
            lpa = lp[int(np.flatnonzero(idx == j)[0])]
            kind = "argmax" if lpa == lp.max() else "zero" if lpa < LOG_TINY else "other"
            r = np.exp(lpa - float(fixed[i]))
            seen.add((kind, 0 if r < 1e-30 else -1 if r < 0.8 else 1 if r > 1.2 else 0.5, float(adv[i])))
        assert {k for k, _, _ in seen} >= {"argmax", "zero", "masked"}, seen
        assert {(r, a) for k, r, a in seen if k == "argmax"} == {(r, a) for r in (0.5, -1, 1, 0) for a in EC.ADVS}
    else:
        for k, v in pre_activations(model, flat, states).items():
            assert (np.abs(v) > 9.0).mean() > 0.3, (k, (np.abs(v) > 9.0).mean())


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("layers", [[0], [1], [0, 1]], ids=["layer0", "layer1", "both"])
def test_factors_beyond_clamp_match_oracle(layers, dev):
    """Moderate edge pre-activations from node factors beyond exp2a's clamp: the product of two clamped factors
    would turn tanh(P_u + Q_v) into tanh(40 - 40) = 0, in the pulls, the head's candidate embeddings and the backward."""
    flat, states, actions = EC.small_clamp_batch(PL.default_init(5), layers)
    assert_beyond_clamp(flat, states, layers)
    check(dev, "sgnn", flat, states, actions, *seeded_batch(5, states))


@pytest.mark.parametrize("name", list(GOLDEN))
def test_golden_regime_matches_oracle_and_reference(name, golden_dir, dev):
    """Each golden batch of the unmodified reference (make_golden_extremes.py): the kernel against the float64 oracle
    at the suite's bars, a tensor's gradient bar raised to twice the reference's own deviation from float64 where that
    exceeds half the bar, and against the reference's recorded gradient within the sum of both bars."""
    mlp, case = GOLDEN[name]
    model = "mlp" if mlp else "sgnn"
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    states = expand_states(z)
    flat, actions, adv, ret, fixed, exps = (z[k] for k in ("params", "actions", "advantages", "returns",
                                                         "fixed_log_probs", "exps"))
    assert_regime(name, model, flat, states, actions, fixed, adv)
    ref = (EC.sgnn_reference if model == "sgnn" else EC.mlp_reference)(flat, states, actions, adv, ret, fixed, exps)
    dev_ref = EC.reference_deviation(model, z, ref)
    bars = {k: max(TOL, 2.0 * d) for k, d in dev_ref.items()}
    g, _ = check(dev, model, flat, states, actions, adv, ret, fixed, exps, bars=bars)
    err = tensor_errors(model, g, z["grads"][0].astype(np.float64))
    bad = {k: e for k, e in err.items() if e >= bars[k] + dev_ref[k]}
    assert not bad, bad


def test_saturated_edges_beyond_clamp_match_oracle(dev):
    """Factors AND edge pre-activations beyond the clamp (both layers sum their endpoints' embeddings, which share a
    large offset): tanh is +-1 and its gradient 0 in fp32."""
    seed = 6
    states, actions = synth.make_states(seed, "small", 16)
    flat = EC.difference_detector(PL.default_init(seed), [0, 1], 4.0, sign=1.0)
    states = EC.place_offsets(flat, states, [0, 1], [100.0 + 10.0 * i for i in range(len(states))])
    P = ON._p64(flat)
    for st in states:
        g = ON.unpad(st)
        hs = ON.forward(P, g, keep=True)["cache"]["hs"]
        for l in range(2):
            W, b = P[f"gcn{l}_w"], P[f"gcn{l}_b"]
            Pn, Qn = hs[l] @ W[:, :16].T + b, hs[l] @ W[:, 16:].T
            x = np.abs(Pn[g.edges[:, 0]] + Qn[g.edges[:, 1]])
            beyond = (x > EC.CLAMP).mean()
            assert max(np.abs(Pn).max(), np.abs(Qn).max()) > EC.CLAMP and beyond > 0.5, (l, beyond)
    check(dev, "sgnn", flat, states, actions, *seeded_batch(seed, states))


def test_fused_step_on_beyond_clamp_batch(dev):
    """upb_ppo_step against upb_ppo_grad + upb_apply over three steps on a batch with tier-2 graphs."""
    flat, states, actions = EC.small_clamp_batch(PL.default_init(5), [0, 1])
    seed = 5
    adv, ret, fixed, exps = seeded_batch(seed, states)
    count, n_ind = len(states), int((exps != 0).sum())
    blob = pack_states(states).to(dev)
    a = (t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev))
    e1, e2 = Engine(dev, blob.n_cap, blob.e_cap), Engine(dev, blob.n_cap, blob.e_cap)
    p1, p2 = t(flat, dev).clone(), t(flat, dev).clone()
    for k in range(3):
        g1 = e1.ppo_grad(blob, p1, *a, 1.0 / count, 1.0 / n_ind)
        e1.apply(p1, g1)
        g2 = e2.ppo_step(blob, p2, *a, 1.0 / count, 1.0 / n_ind)
        torch.cuda.synchronize()
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (k, worst, where)
        assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
        q1, q2 = p1.cpu().numpy(), p2.cpu().numpy()
        assert np.abs(q2 - q1).max() <= 1e-6 * np.abs(q1).max(), k


# ---------------------------------------------------------------------------------------------------- non-finite guard
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_nonfinite_guard_counts_graphs_and_stops_the_update(model, dev):
    """A NaN in the value head makes every graph's value non-finite: statistics slot 7 counts them all and
    PPOUpdater.update_params raises FloatingPointError instead of stepping."""
    from drl_urban_planning_b200.ppo import PPOUpdater
    seed, count = 15, 16
    layout = PL.SGNN if model == "sgnn" else PL.MLP
    states, actions = synth.make_states(seed, "small", count)
    flat = layout.default_init(seed).copy()
    EC.slot(flat, "val_w2", layout)[0, 3] = np.nan
    adv, ret, exps = synth.make_ppo_targets(seed, count)
    fixed = np.full((count, 1), -3.0, np.float32)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    grad = eng.ppo_grad(blob, t(flat, dev), t(actions, dev), t(adv, dev), t(ret, dev), t(fixed, dev), t(exps, dev),
                        1.0 / count, 1.0 / count)
    st = grad.cpu().numpy()[eng.stat_offset:eng.stat_offset + 8]
    assert st[3] == count and st[7] == count, st
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, gamma=0.99, tau=0.95, opt_num_epochs=1,
                    mini_batch_size=count, model=model)
    rewards = np.random.default_rng(seed).standard_normal(count).astype(np.float32)
    with pytest.raises(FloatingPointError):
        up.update_params(states, actions, rewards, np.ones(count, np.float32))
