"""GPU (H100): action selection (upb_select_action / upb_mlp_select_action, policy.py:67-85) on both models against
the float64 candidate probabilities: oracle/sgnn_numpy.py for the SGNN, oracle/mlp_port.py run in float64 for the
rl-mlp.

Each case is one graph (synth.make_exact_state) with k candidates at the limits of the sampler's scan (chunks of 32
candidates carried into the next chunk, the 160-candidate shared-memory limit, a graph at the 1000 / 3000 caps) or
with an empty mask.  The graph is packed as many copies, so one launch evaluates one candidate or one uniform per copy:
  * forward with actions[m] = the m-th candidate returns the kernel's fp32 log-prob of every candidate;
  * select_action with one uniform per copy sweeps the inverse CDF: a stratified grid, the fp32 neighbours of every
    CDF boundary, u = 0 and u = 1 - 2^-24.
Peaked parameter sets scale the policy head's output layer until logit gaps exceed 104, where fp32 exp underflows:
such a candidate has probability 0 and must never be sampled (Categorical.sample never returns one)."""
import math

import numpy as np
import pytest
import torch

import shape_cases as SC
from drl_urban_planning_b200 import synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from extreme_cases import LOG_TINY, scaled_head
from harness import dev, load, lp_tol, t
from oracle import mlp_port as MP
from policy_cases import SEED, SPEC, caps_case, cases, flat_params, ref_logits

pytestmark = pytest.mark.gpu

LOG_ZERO = math.log(2.0 ** -150)          # below this an fp32 probability rounds to 0
GRID = 256                                # stratified uniforms per sweep
BELOW_ONE = np.float32(1.0 - 2.0 ** -24)
# the cases (policy_cases.cases): every k of policy_cases.KS for both stages, then an empty mask for each


def band(k):
    """How far an interval boundary of the kernel's sampler may lie from the cumulative sum of the kernel's own
    (normalised) probabilities.  Candidate j's boundary is c_j / S: c_j is a Hillis-Steele scan over the chunk of 32
    (5 roundings) plus one carry per earlier chunk, S a per-lane sum of k / 32 terms plus a 5-step butterfly, every term
    an expf within 2 ulp, u * S one more rounding, and each log-prob z_j - lse one rounding relative to its size (summed
    against p_j: entropy * 2^-24 <= log(k) * 2^-24).  Together well under (k + 64) ulp of 1."""
    return (k + 64) * 2.0 ** -24


def log_softmax(z):
    zs = z - z.max()
    return zs - math.log(np.exp(zs).sum())


def peak_scale(z):
    """A scale for the logits z that gives some candidates probability 0 in fp32 (float64 log-prob below log(2^-150),
    where p = exp(z - zmax) / sum rounds to 0) and keeps every candidate out of [log(2^-150) - 1, log(2^-149) + 0.5),
    where rounding could go either way, so that "float64 log-prob below log(2^-149)" and "fp32 probability 0" pick out
    the same candidates.  Scales that zero the first candidate (the u = 0 pick) are preferred."""
    fallback = None
    for s in 30.0 * 1.1 ** np.arange(80):
        lp = log_softmax(s * z)
        if (lp < LOG_TINY).any() and not ((lp >= LOG_ZERO - 1.0) & (lp < LOG_TINY + 0.5)).any():
            if lp[0] < LOG_TINY:
                return float(s)
            fallback = fallback or float(s)
    assert fallback is not None, "no scale separates the logits"
    return fallback


# ---------------------------------------------------------------------------------------------------- kernel calls
def copies(st, m, dev):
    return pack_states([st] * m).to(dev)


def kernel_logp(eng, params, st, cand, stage, dev):
    """The kernel's fp32 log-prob of each candidate index in `cand`, one copy of the graph per candidate."""
    blob = copies(st, len(cand), dev)
    actions = np.zeros((len(cand), 2), np.float32)
    actions[:, stage] = cand
    _, lp, _ = eng.forward(blob, params, t(actions, dev))
    return lp.cpu().numpy().astype(np.float64)


def kernel_picks(eng, params, st, u, dev):
    blob = copies(st, len(u), dev)
    return eng.select_action(blob, params, uniforms=t(np.asarray(u, np.float32), dev)).cpu().numpy()


def boundary_uniforms(bounds):
    """Each boundary rounded to fp32 and its two fp32 neighbours, inside [0, 1)."""
    b = np.asarray(bounds, np.float64).astype(np.float32)
    u = np.concatenate([np.nextafter(b, np.float32(0)), b, np.nextafter(b, np.float32(1))])
    return u[(u >= 0) & (u < 1)]


def grid_uniforms(m):
    return ((np.arange(m) + 0.5) / m).astype(np.float32)


def check_sweep(label, u, picks, idx, lp64, cdfs, m_grid):
    """The inverse-CDF properties of one sweep.  `cdfs`: [(name, cdf, tolerance)] the picks must bracket u in."""
    u = np.asarray(u, np.float64)
    assert np.isin(picks, idx).all(), (label, "pick outside the mask", picks[~np.isin(picks, idx)][:5])
    pos = np.searchsorted(idx, picks)
    order = np.argsort(u, kind="stable")
    assert (np.diff(pos[order]) >= 0).all(), (label, "picks not monotone in u")
    for name, cdf, tol in cdfs:
        lo = np.where(pos > 0, cdf[np.maximum(pos - 1, 0)], 0.0)
        bad = (u < lo - tol) | (u > cdf[pos] + tol)
        assert not bad.any(), (label, name, "u outside its pick's interval", u[bad][:3], pos[bad][:3], tol)
    zero = lp64[pos] < LOG_TINY
    assert not zero.any(), (label, "zero-probability candidate sampled", u[zero][:3], idx[pos[zero]][:3],
                            lp64[pos[zero]][:3])
    p64 = np.exp(lp64)
    counts = np.bincount(pos[:m_grid], minlength=idx.size) / m_grid
    tol = cdfs[-1][2]
    worst = np.abs(counts - p64).max()
    assert worst <= 1.0 / m_grid + 2 * tol, (label, "grid share", worst)


# ---------------------------------------------------------------------------------------------------- sweeps
class Sweep:
    """One case run through both kernel calls: per-candidate log-probs, then the inverse-CDF sweep."""

    def __init__(self, eng, model, flat, st, stage, dev, label):
        self.label = label
        self.idx, z = ref_logits(model, flat, st)
        k = self.idx.size
        self.k = k
        self.lp64 = log_softmax(z)
        params = t(flat, dev)
        self.lpk = kernel_logp(eng, params, st, self.idx, stage, dev)
        self.zabs = float(np.abs(z).max())
        self.lp_err = np.abs(self.lpk - self.lp64)
        self.lp_ratio = float((self.lp_err / lp_tol(self.lp64, self.zabs)).max())
        pk = np.exp(self.lpk - self.lpk.max())
        self.cdfk = np.cumsum(pk) / pk.sum()
        self.cdf64 = np.cumsum(np.exp(self.lp64))
        # the sampler against the float64 CDF: its own band plus how far the kernel's probabilities are from float64
        self.err64 = float(2 * (np.exp(self.lp64) * self.lp_err).sum())
        self.u = np.concatenate([grid_uniforms(GRID), boundary_uniforms(self.cdfk[:-1]), [0.0, BELOW_ONE]])
        self.picks = kernel_picks(eng, params, st, self.u, dev)

    def check(self):
        assert self.lp_ratio <= 1.0, (self.label, "log-prob", self.lp_ratio,
                                      int(np.argmax(self.lp_err / lp_tol(self.lp64, self.zabs))))
        b = band(self.k)
        check_sweep(self.label, self.u, self.picks, self.idx, self.lp64,
                    [("kernel", self.cdfk, b), ("float64", self.cdf64, b + self.err64)], GRID)


@pytest.fixture(scope="module")
def all_cases():
    return cases()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_log_probs_and_inverse_cdf_at_scan_limits(model, all_cases, dev):
    """Every candidate's log-prob element by element, and the inverse-CDF sweep, for k = 1 ... 161 on both stages."""
    flat = flat_params(model)
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model=model)
    for label, st, stage in all_cases:
        if not st[6 + stage].any():
            continue
        Sweep(eng, model, flat, st, stage, dev, f"{model}_{label}").check()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_peaked_logits_never_sample_a_zero_probability_candidate(model, all_cases, dev):
    """The output layer of the policy head scaled per graph until logit gaps pass 104: candidates whose float64
    log-prob is below log(2^-149) have fp32 probability 0 and must not be picked, at u = 0 and u = 1 - 2^-24
    included.  The scales are chosen so that the first candidate is such a one wherever possible (what u = 0 picked
    when the sampler took the first cumulative sum >= u * sum)."""
    flat = flat_params(model)
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model=model)
    first_zero = later_chunk_zero = 0
    for label, st, stage in all_cases:
        idx, z = ref_logits(model, flat, st)
        if idx.size < 2:
            continue
        peaked = scaled_head(model, flat, stage, peak_scale(z))
        sw = Sweep(eng, model, peaked, st, stage, dev, f"{model}_{label}_peaked")
        assert not ((sw.lp64 >= LOG_ZERO - 0.5) & (sw.lp64 < LOG_TINY)).any(), (sw.label, "a candidate at the line")
        sw.check()
        first_zero += sw.lp64[0] < LOG_TINY
        later_chunk_zero += (sw.lp64[32:] < LOG_TINY).any()
    assert first_zero >= 4 and later_chunk_zero >= 2, (first_zero, later_chunk_zero)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_graph_at_the_caps_with_3000_candidates(model, dev):
    """k = 3000 on the 1000 / 3000 caps in a few hundred copies: the log-probs of the 150 most probable candidates and
    of 150 others spread over the index range, and a sweep over a grid and both boundaries of the 30 most probable
    candidates, against the float64 CDF (the tolerance adds the measured log-prob error, lp_tol for the others)."""
    st = caps_case()
    flat = flat_params(model)
    eng = Engine(dev, 1000, 3000, model=model)
    idx, z = ref_logits(model, flat, st)
    assert idx.size == 3000
    lp64 = log_softmax(z)
    zabs = float(np.abs(z).max())
    params = t(flat, dev)
    top = np.argsort(-lp64, kind="stable")
    sel = np.unique(np.concatenate([top[:150], np.linspace(0, 2999, 150).astype(np.int64)]))
    lpk = kernel_logp(eng, params, st, idx[sel], 0, dev)
    err = np.abs(lpk - lp64[sel])
    assert (err <= lp_tol(lp64[sel], zabs)).all(), float((err / lp_tol(lp64[sel], zabs)).max())
    cdf64 = np.cumsum(np.exp(lp64))
    ends = np.concatenate([top[:30], np.maximum(top[:30] - 1, 0)])
    u = np.concatenate([grid_uniforms(200), boundary_uniforms(cdf64[ends]), [0.0, BELOW_ONE]])
    picks = kernel_picks(eng, params, st, u, dev)
    errs = lp_tol(lp64, zabs)
    errs[sel] = err
    p_err = float(2 * (np.exp(lp64) * errs).sum())
    check_sweep(f"{model}_k3000", u, picks, idx, lp64, [("float64", cdf64, band(3000) + p_err)], 200)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_empty_mask_picks_uniformly_over_the_padded_width(model, all_cases, dev):
    """With no candidate the reference's distribution is uniform over the padded width (every logit is the fill value):
    the pick is min(cap - 1, floor(u * cap)) in fp32, cap = the blob's edge cap for land use, node cap for road."""
    flat = flat_params(model)
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model=model)
    u = np.concatenate([grid_uniforms(GRID), [0.0, BELOW_ONE, np.float32(0.5)]]).astype(np.float32)
    for label, st, stage in all_cases:
        if st[6 + stage].any():
            continue
        cap = np.float32(SPEC.max_num_edges if stage == 0 else SPEC.max_num_nodes)
        picks = kernel_picks(eng, t(flat, dev), st, u, dev)
        want = np.minimum(cap - 1, np.floor(u * cap)).astype(np.int64)
        assert np.array_equal(picks, want), (label, np.flatnonzero(picks != want)[:5])


# ---------------------------------------------------------------------------------------------------- greedy
def near_ties(lp64, idx):
    """The candidates within 1e-6 of the largest float64 probability (test_boundary_sweep_matches_oracle's rule)."""
    p = np.exp(lp64)
    return idx[p >= p.max() - 1e-6]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_greedy_is_the_forward_arg_max_and_the_float64_arg_max(model, all_cases, dev):
    """select_action without uniforms equals forward(want_greedy=True) bit for bit, and the float64 arg-max wherever
    the top two are not within 1e-6 (then one of the near-tied candidates; the smallest index where they tie exactly,
    as rl-mlp land-use candidates selecting the same node do)."""
    flat = flat_params(model)
    labelled = [(label, st) for label, st, stage in all_cases if st[6 + stage].any()]
    blob = pack_states([st for _, st in labelled]).to(dev)
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model=model)
    params = t(flat, dev)
    greedy = eng.select_action(blob, params)
    _, _, _, fwd = eng.forward(blob, params, want_greedy=True)
    assert torch.equal(greedy, fwd.to(torch.int32))
    greedy = greedy.cpu().numpy()
    unique = tied = 0
    for i, (label, st) in enumerate(labelled):
        idx, z = ref_logits(model, flat, st)
        near = near_ties(log_softmax(z), idx)
        assert greedy[i] in near, (label, greedy[i], near)
        if near.size == 1 or (z[np.isin(idx, near)] >= z.max() - 1e-12).all():
            assert greedy[i] == near.min(), (label, greedy[i], near)
            unique += near.size == 1
            tied += near.size > 1
    assert unique >= 8, unique
    assert model == "sgnn" or tied >= 1, tied


def tied_mlp_case():
    """A land-use graph whose best candidates share their selected endpoint, so their rl-mlp logits tie exactly.  A hub
    node is the selected endpoint of most of its edges (of every edge (hub, j) whose j is not of type FEASIBLE).  The
    candidates: every edge selecting the best-scored node among those selected by 3 edges or more, and up to 40 edges
    scored below it.  Returns (state, the tied edge indices)."""
    rng = np.random.default_rng(SEED + 2)
    st, _ = synth.make_exact_state(rng, SPEC, 120, 300, 1, 0, hub=True)
    e = int(st[5].sum())
    st[6][:e] = True                                  # score every edge once
    flat = flat_params("mlp")
    idx, z = ref_logits("mlp", flat, st)
    x = st[1]
    u, v = st[2][:e, 0], st[2][:e, 1]
    feas = np.argmax(x[:, :14], axis=1) == 1
    sel = np.where(feas[v], v, u)
    counts = np.bincount(sel, minlength=x.shape[0])
    best = max((n for n in range(x.shape[0]) if counts[n] >= 3), key=lambda n: z[np.flatnonzero(sel == n)[0]])
    zb = z[np.flatnonzero(sel == best)[0]]
    below = np.flatnonzero(z < zb - 1e-3)
    keep = np.concatenate([np.flatnonzero(sel == best), rng.choice(below, size=min(40, below.size), replace=False)])
    st[6][:] = False
    st[6][keep] = True
    return st, np.flatnonzero(sel == best)


def test_mlp_exact_ties_pick_the_smallest_edge_index(dev):
    """rl-mlp land-use candidates that select the same node have bit-identical logits: greedy must take the smallest
    edge index, as the fp32 port's softmax(...).argmax (the reference's probs.argmax) does."""
    st, tied = tied_mlp_case()
    assert tied.size >= 3
    flat = flat_params("mlp")
    with torch.no_grad():
        want = MP.greedy_action(MP.params_from_flat(flat), MP.stack_states([st])).numpy()[0, 0]
    assert int(want) == tied.min()
    blob = pack_states([st] * 3).to(dev)
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model="mlp")
    params = t(flat, dev)
    got = eng.select_action(blob, params).cpu().numpy()
    _, _, _, fwd = eng.forward(blob, params, want_greedy=True)
    assert got.tolist() == [tied.min()] * 3 and fwd.cpu().numpy().tolist() == got.tolist()


@pytest.mark.parametrize("name", ["mlp_small", "mlp_hlg"])
def test_mlp_golden_greedy_through_select_action(name, golden_dir, dev):
    """upb_mlp_select_action against the greedy actions the unmodified reference recorded."""
    from fixtures_io import expand_states
    z = load(golden_dir, name)
    states = expand_states(z)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model="mlp")
    got = eng.select_action(blob, t(z["params"], dev)).cpu().numpy()
    stage = z["stage"][:, :2].argmax(1)
    assert np.array_equal(got.astype(np.int64), z["greedy"][np.arange(len(states)), stage].astype(np.int64))


# ---------------------------------------------------------------------------------------------------- placement
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_picks_do_not_depend_on_placement(model, dev):
    """The boundary batch (fast and big graphs, k up to 3000): greedy and sampled picks are identical with one graph
    per CTA, with one CTA walking every graph fast -> big -> fast, and for an LPT-ordered subset of ids, whose
    other output slots stay 0."""
    b = SC.Batch(dev)
    flat = flat_params(model)
    params = t(flat, dev)
    rng = np.random.default_rng(SEED)
    u = rng.random(b.count).astype(np.float32)
    u[:2] = [0.0, BELOW_ONE]
    ud = t(u, dev)
    full = Engine(dev, b.blob.n_cap, b.blob.e_cap, model=model)
    one = Engine(dev, b.blob.n_cap, b.blob.e_cap, model=model, grid_limit=1)
    assert full.grid >= b.count and one.grid == 1
    want_s = full.select_action(b.blob, params, uniforms=ud).cpu().numpy()
    want_g = full.select_action(b.blob, params).cpu().numpy()
    walk = t(SC.placed(SC.walk_order(b), 1), dev)
    assert np.array_equal(one.select_action(b.blob, params, uniforms=ud, ids=walk).cpu().numpy(), want_s)
    assert np.array_equal(one.select_action(b.blob, params, ids=walk).cpu().numpy(), want_g)
    subset = np.arange(0, b.count, 2)
    ids = full.balance_ids(subset, Engine.graph_cost(b.info))
    ids_d = t(ids.astype(np.int32), dev)
    rest = np.setdiff1d(np.arange(b.count), subset)
    for uu, want in ((ud, want_s), (None, want_g)):
        got = full.select_action(b.blob, params, uniforms=uu, ids=ids_d).cpu().numpy()
        assert np.array_equal(got[subset], want[subset]) and not got[rest].any()
