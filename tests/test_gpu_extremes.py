"""GPU (H100): the training kernels at the magnitudes a trained policy reaches, against the float64 oracles
(oracle/sgnn_numpy.py for the SGNN; oracle/mlp_port.py run in float64, gradients by autograd, for the rl-mlp), and
against vectors recorded by the unmodified reference in the same regimes (tests/golden/make_golden_extremes.py).

Regimes (parameter transforms, batches and the regime checks in tests/extreme_cases.py), each checked from the oracle's own float64
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
import numpy as np
import pytest
import torch

import extreme_cases as EC
from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from oracle import sgnn_numpy as ON
from harness import dev, load, lp_tol, per_tensor_rel, t, tensor_errors

pytestmark = pytest.mark.gpu

TOL = 1e-4
GOLDEN = {name: (mlp, case) for name, _, mlp, case in EC.FIXTURES}


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
    layout = PL.MLP if model == "mlp" else PL.SGNN
    bad = {k: e for k, e in tensor_errors(g[:layout.num_params], ref["grad"], layout).items() if e >= bars.get(k, TOL)}
    assert not bad, (bad, {k: bars.get(k, TOL) for k in bad})
    assert np.allclose(eng.read_losses(grad), [ref["loss"], ref["value_loss"], ref["surr_loss"], ref["entropy_loss"]],
                       rtol=1e-4, atol=1e-5)
    st = g[eng.stat_offset:eng.stat_offset + 8]
    assert st[3] == B and st[4] == int((exps != 0).sum()) and st[7] == 0, st
    eng.apply(params, grad)
    d = np.abs(params.cpu().numpy() - ref["after"])
    assert d.max() <= 1e-5 * np.abs(ref["after"]).max(), ("apply", int(d.argmax()), d.max())
    return g[:layout.num_params], ref


def seeded_batch(seed, states):
    adv, ret, exps = EC.targets(seed, len(states))
    fixed = np.random.default_rng(seed).normal(-3.0, 0.3, size=(len(states), 1)).astype(np.float32)
    return adv, ret, fixed, exps


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("layers", [[0], [1], [0, 1]], ids=["layer0", "layer1", "both"])
def test_factors_beyond_clamp_match_oracle(layers, dev):
    """Moderate edge pre-activations from node factors beyond exp2a's clamp: the product of two clamped factors
    would turn tanh(P_u + Q_v) into tanh(40 - 40) = 0, in the pulls, the head's candidate embeddings and the backward."""
    flat, states, actions = EC.small_clamp_batch(PL.default_init(5), layers)
    EC.assert_beyond_clamp(flat, states, layers)
    check(dev, "sgnn", flat, states, actions, *seeded_batch(5, states))


@pytest.mark.parametrize("name", list(GOLDEN))
def test_golden_regime_matches_oracle_and_reference(name, golden_dir, dev):
    """Each golden batch of the unmodified reference (make_golden_extremes.py): the kernel against the float64 oracle
    at the suite's bars, a tensor's gradient bar raised to twice the reference's own deviation from float64 where that
    exceeds half the bar, and against the reference's recorded gradient within the sum of both bars."""
    mlp, case = GOLDEN[name]
    model = "mlp" if mlp else "sgnn"
    z = load(golden_dir, name)
    states = expand_states(z)
    flat, actions, adv, ret, fixed, exps = (z[k] for k in ("params", "actions", "advantages", "returns",
                                                         "fixed_log_probs", "exps"))
    EC.assert_regime(name, model, flat, states, actions, fixed, adv)
    ref = (EC.sgnn_reference if model == "sgnn" else EC.mlp_reference)(flat, states, actions, adv, ret, fixed, exps)
    dev_ref = EC.reference_deviation(model, z, ref)
    bars = {k: max(TOL, 2.0 * d) for k, d in dev_ref.items()}
    g, _ = check(dev, model, flat, states, actions, adv, ret, fixed, exps, bars=bars)
    err = tensor_errors(g, z["grads"][0], PL.MLP if mlp else PL.SGNN)
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
