"""GPU (H100): the masked logit rows of both policy heads (upb_policy_logits / upb_mlp_policy_logits, Engine.policy_logits,
policy_net(states) on CUDA; reference policy.py:45-65) on both models.

  * reference pin: policy_net(states) on CUDA against the distributions the unmodified reference recorded
    (tests/golden/make_golden_logits.py), masked entries bit for bit, candidates at the per-tensor bar of 1e-4;
  * float64 oracle: every candidate's logit against policy_cases.ref_logits, and the fill value everywhere else,
    for k = 1 ... 161 on both stages, empty masks and k = 3000 at the caps in one mixed launch, the boundary graphs of
    tests/shape_cases.py and a batch with tier-2 GCN graphs (tests/extreme_cases.py);
  * consistency: Categorical.log_prob / entropy over the rows against Engine.forward's, the first-index arg-max against
    forward(want_greedy=True), and a forward after policy_logits unchanged;
  * placement: rows bit-identical at every grid size and for LPT-ordered and reversed ids;
  * edges: an ids subset, a NULL road matrix, a graph over the context's caps, bad arguments;
  * the drop-in modules on CUDA: shapes, None for a stage without a graph, agreement with the CPU modules."""
import os

import numpy as np
import pytest
import torch

import extreme_cases as EC
import shape_cases as SC
from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.model import MASK_FILL
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from harness import dev, lp_tol, t, tensorfy
from policy_cases import (LOGIT_FIXTURES as FIXTURES, caps_case, cases, check_distribution, flat_params, load_policy,
                          ref_logits)

pytestmark = pytest.mark.gpu

FILL = np.float32(MASK_FILL)
EPS = 2.0 ** -23
SEED = 23


# ---------------------------------------------------------------------------------------------------- helpers
def repad(st, N, E):
    """The same graph padded to the caps (N, E)."""
    numerical, nf, ei, cur, nm, em, lm, rm, stage = st
    n0, e0 = nf.shape[0], ei.shape[0]
    nf2 = np.zeros((N, nf.shape[1]), nf.dtype); nf2[:n0] = nf
    ei2 = np.full((E, 2), N - 1, ei.dtype); ei2[:e0] = ei
    pad = lambda m, L: np.concatenate([m, np.zeros(L - m.size, m.dtype)])
    return [numerical, nf2, ei2, cur, pad(nm, N), pad(em, E), pad(lm, E), pad(rm, N), stage]


def mixed_cases():
    """Every case of test_gpu_select (k = 1 ... 161 and empty masks, both stages) and the k = 3000 graph, on the
    1000 / 3000 caps, stages interleaved."""
    states = [repad(st, SC.SPEC.max_num_nodes, SC.SPEC.max_num_edges) for _, st, _ in cases()] + [caps_case()]
    order = np.random.default_rng(SEED).permutation(len(states))
    return [states[i] for i in order]


def rows_by_graph(lu, rd, stage, order):
    """{blob position: its row} from Engine.policy_logits' matrices, rows numbered per stage in `order`."""
    out, nxt = {}, [0, 0]
    mats = [None if lu is None else lu.cpu().numpy(), None if rd is None else rd.cpu().numpy()]
    for g in order:
        s = int(stage[g])
        out[int(g)] = mats[s][nxt[s]]
        nxt[s] += 1
    assert all(m is None or m.shape[0] == n for m, n in zip(mats, nxt))
    return out


def check_against_oracle(model, flat, states, rows, n_cap, e_cap, label):
    worst = 0.0
    for g, st in enumerate(states):
        stage = int(np.argmax(st[8][:2]))
        row = rows[g]
        assert row.shape == ((e_cap,) if stage == 0 else (n_cap,)), (label, g, row.shape)
        idx, z64 = ref_logits(model, flat, st)
        masked = np.ones(row.size, bool)
        masked[idx] = False
        assert (row[masked] == FILL).all(), (label, g, "fill")
        if idx.size:
            zabs = float(np.abs(z64).max())
            ratio = np.abs(row[idx].astype(np.float64) - z64) / lp_tol(z64, zabs)
            worst = max(worst, float(ratio.max()))
            assert ratio.max() <= 1.0, (label, g, float(ratio.max()), int(idx[np.argmax(ratio)]))
    return worst


def raw_call(eng, blob, params, ids, count, rows, lu, rd):
    """The C entry point itself, for what Engine.policy_logits does not expose (caller-owned rows and matrices)."""
    fn = getattr(_lib.lib(), eng._p + "policy_logits")
    ptr = lambda x: None if x is None else x.data_ptr()
    rc = fn(eng._ctx, None if blob is None else blob.dev_ptr(), ptr(ids), count, ptr(params), ptr(rows), ptr(lu),
            ptr(rd), eng._stream())
    torch.cuda.synchronize()
    return rc


MODELS = ["sgnn", "mlp"]


# ---------------------------------------------------------------------------------------------------- reference pin
@pytest.mark.parametrize("name", list(FIXTURES))
def test_cuda_forward_matches_reference_distributions(name, golden_dir, dev):
    """policy_net(states) with the modules on CUDA: the reference's logits / probs (masked entries bit for bit, an
    all-masked row all 0 as the reference's fp32 normalisation gives) and stage."""
    z, ref, states, policy_net = load_policy(name, golden_dir)
    policy_net.to(dev)
    d0, d1, stage = policy_net(tensorfy(states))
    assert stage.is_cuda and stage.dtype == torch.float32
    assert np.array_equal(stage.cpu().numpy(), ref["stage"])
    check_distribution("lu", d0, ref)
    check_distribution("rd", d1, ref)
    if name == "edge_empty":
        for d in (d0, d1):
            assert (d.logits == 0).all(dim=1).any()


# ---------------------------------------------------------------------------------------------------- float64 oracle
@pytest.mark.parametrize("model", MODELS)
def test_scan_limits_empty_masks_and_caps_in_one_launch(model, dev):
    states = mixed_cases()
    flat = flat_params(model)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    lu, rd, stage = eng.policy_logits(blob, t(flat, dev))
    assert lu is not None and rd is not None and int(blob.info[:, 2].max()) == 3000
    rows = rows_by_graph(lu, rd, stage, range(blob.count))
    check_against_oracle(model, flat, states, rows, blob.n_cap, blob.e_cap, f"{model}_cases")


@pytest.mark.parametrize("model", MODELS)
def test_boundary_graphs(model, dev):
    """Both sides of every shared-memory / global-scratch limit (n = 464, 2e = 5632, k = 160 / 161) and the caps."""
    states, _, _ = SC.boundary_batch(SEED)
    flat = flat_params(model)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    lu, rd, stage = eng.policy_logits(blob, t(flat, dev))
    rows = rows_by_graph(lu, rd, stage, range(blob.count))
    check_against_oracle(model, flat, states, rows, blob.n_cap, blob.e_cap, f"{model}_boundary")


def test_tier2_gcn_batch(dev):
    """Graphs whose GCN factors pass exp2a's clamp (tier 2 of the EPQ phase) next to ordinary ones."""
    flat, states, _ = EC.small_clamp_batch(PL.default_init(5), [0, 1])
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap)
    lu, rd, stage = eng.policy_logits(blob, t(flat, dev))
    rows = rows_by_graph(lu, rd, stage, range(blob.count))
    check_against_oracle("sgnn", flat, states, rows, blob.n_cap, blob.e_cap, "tier2")


# ---------------------------------------------------------------------------------------------------- consistency
@pytest.mark.parametrize("model", MODELS)
def test_distributions_agree_with_forward_outputs(model, dev):
    """On one batch: Categorical.log_prob(a) / entropy() over the rows equal Engine.forward's log-prob / entropy within
    a few ulps of their magnitude, the first-index arg-max of every row is forward's greedy action bit for bit, and
    policy_logits leaves a following forward bit-identical."""
    states = mixed_cases()
    flat = flat_params(model)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    params = t(flat, dev)
    rng = np.random.default_rng(SEED)
    actions = np.zeros((blob.count, 2), np.float32)
    for g, st in enumerate(states):
        s = int(np.argmax(st[8][:2]))
        cand = np.flatnonzero(st[6 + s])
        actions[g, s] = rng.choice(cand) if cand.size else 0
    a_d = t(actions, dev)
    before = eng.forward(blob, params, a_d, want_greedy=True)
    lu, rd, stage = eng.policy_logits(blob, params)
    after = eng.forward(blob, params, a_d, want_greedy=True)
    for x, y in zip(before, after):
        assert torch.equal(x, y)
    _, lp, ent, greedy = (x.cpu().numpy() for x in after)
    for s, mat in ((0, lu), (1, rd)):
        sel = np.flatnonzero(stage == s)
        d = torch.distributions.Categorical(logits=mat)
        lp_d = d.log_prob(t(actions[sel, s].astype(np.int64), dev)).cpu().numpy().astype(np.float64)
        ent_d = d.entropy().cpu().numpy().astype(np.float64)
        zmax = np.abs(np.where(mat.cpu().numpy() == FILL, 0.0, mat.cpu().numpy())).max(axis=1)
        assert (np.abs(lp_d - lp[sel]) <= 16 * EPS * (1.0 + np.abs(lp_d) + zmax)).all(), (s, np.abs(lp_d - lp[sel]).max())
        assert (np.abs(ent_d - ent[sel]) <= 16 * EPS * (1.0 + ent_d + zmax)).all(), (s, np.abs(ent_d - ent[sel]).max())
        assert np.array_equal(torch.argmax(mat, dim=1).cpu().numpy(), greedy[sel]), s


# ---------------------------------------------------------------------------------------------------- placement
@pytest.mark.parametrize("model", MODELS)
def test_rows_do_not_depend_on_placement(model, dev):
    """The boundary batch with one, two, three CTAs and a full grid, and with LPT-ordered and reversed ids."""
    states, _, _ = SC.boundary_batch(SEED)
    blob = pack_states(states).to(dev)
    params = t(flat_params(model), dev)
    full = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    lu, rd, stage = full.policy_logits(blob, params)
    want = rows_by_graph(lu, rd, stage, range(blob.count))
    for grid in (1, 2, 3):
        eng = Engine(dev, blob.n_cap, blob.e_cap, model=model, grid_limit=grid)
        got = rows_by_graph(*eng.policy_logits(blob, params), range(blob.count))
        assert all(np.array_equal(got[g], want[g]) for g in want), grid
    lpt = full.balance_ids(np.arange(blob.count), Engine.graph_cost(blob.info))
    for order in (lpt, lpt[::-1].copy()):
        ids = t(order.astype(np.int32), dev)
        got = rows_by_graph(*full.policy_logits(blob, params, ids=ids), order)
        assert all(np.array_equal(got[g], want[g]) for g in want)


# ---------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("model", MODELS)
def test_ids_subset_writes_only_listed_rows(model, dev):
    """Every graph has a row, only every third graph is listed: the others' rows keep their sentinel."""
    states, _, _ = SC.boundary_batch(SEED)
    blob = pack_states(states).to(dev)
    params = t(flat_params(model), dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    want = rows_by_graph(*eng.policy_logits(blob, params), range(blob.count))
    stage = blob.info[:, 3]
    rows = torch.arange(blob.count, dtype=torch.int32, device=dev)
    lu = torch.full((blob.count, blob.e_cap), 7.0, device=dev)
    rd = torch.full((blob.count, blob.n_cap), 7.0, device=dev)
    listed = np.arange(0, blob.count, 3)
    assert raw_call(eng, blob, params, t(listed.astype(np.int32), dev), listed.size, rows, lu, rd) == 0
    mats = (lu.cpu().numpy(), rd.cpu().numpy())
    for g in range(blob.count):
        for s in (0, 1):
            if g in listed and stage[g] == s:
                assert np.array_equal(mats[s][g], want[g]), g
            else:
                assert (mats[s][g] == 7.0).all(), (g, s)


@pytest.mark.parametrize("model", MODELS)
def test_null_road_matrix_writes_land_use_rows_only(model, golden_dir, dev):
    """A land-use-only batch (hlg) and a mixed one (small_mixed) with road_logits = NULL."""
    params = t(flat_params(model), dev)
    for name in ("hlg", "small_mixed"):
        states = expand_states(np.load(os.path.join(golden_dir, name + ".npz")))
        blob = pack_states(states).to(dev)
        eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
        want = rows_by_graph(*eng.policy_logits(blob, params), range(blob.count))
        stage = blob.info[:, 3]
        rows = torch.as_tensor(np.where(stage == 0, np.cumsum(stage == 0) - 1, np.cumsum(stage == 1) - 1)
                               .astype(np.int32), device=dev)
        lu = torch.full((int((stage == 0).sum()), blob.e_cap), 7.0, device=dev)
        assert raw_call(eng, blob, params, None, blob.count, rows, lu, None) == 0
        got = lu.cpu().numpy()
        for r, g in enumerate(np.flatnonzero(stage == 0)):
            assert np.array_equal(got[r], want[g]), (name, g)


@pytest.mark.parametrize("model", MODELS)
def test_graph_over_the_caps_gets_a_nan_row(model, dev):
    """A context with caps 464 / 1500 on the boundary batch (packed at 1000 / 3000): graphs beyond them get a NaN row,
    the others the same row as on a context at the full caps, up to the smaller width."""
    states, _, _ = SC.boundary_batch(SEED)
    blob = pack_states(states).to(dev)
    params = t(flat_params(model), dev)
    full = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    want = rows_by_graph(*full.policy_logits(blob, params), range(blob.count))
    n_cap, e_cap = 464, 1500
    small = Engine(dev, n_cap, e_cap, model=model)
    info = blob.info
    over = (info[:, 0] > n_cap) | (info[:, 1] > e_cap)
    assert over.any() and (~over).any()
    stage = info[:, 3]
    rows = torch.as_tensor(np.where(stage == 0, np.cumsum(stage == 0) - 1, np.cumsum(stage == 1) - 1)
                           .astype(np.int32), device=dev)
    lu = torch.zeros(int((stage == 0).sum()), e_cap, device=dev)
    rd = torch.zeros(int((stage == 1).sum()), n_cap, device=dev)
    assert raw_call(small, blob, params, None, blob.count, rows, lu, rd) == 0
    mats = (lu.cpu().numpy(), rd.cpu().numpy())
    for g in range(blob.count):
        row = mats[stage[g]][int(rows[g])]
        if over[g]:
            assert np.isnan(row).all(), g
        else:
            assert np.array_equal(row, want[g][:row.size]) and (want[g][row.size:] == FILL).all(), g


def test_bad_arguments_return_an_error(dev):
    states, _, _ = SC.boundary_batch(SEED)
    blob = pack_states(states[:4]).to(dev)
    for model in MODELS:
        eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
        params = t(flat_params(model), dev)
        rows = torch.zeros(4, dtype=torch.int32, device=dev)
        lu = torch.full((1, blob.e_cap), 7.0, device=dev)
        for args in ((None, params, 4, rows), (blob, None, 4, rows), (blob, params, 4, None), (blob, params, -1, rows)):
            rc = raw_call(eng, args[0], args[1], None, args[2], args[3], lu, None)
            assert rc != 0 and b"policy_logits" in _lib.lib().upb_last_error(), (model, rc)
        assert raw_call(eng, blob, params, None, 0, rows, lu, None) == 0          # count 0: nothing launched
        assert (lu == 7.0).all()
        fn = getattr(_lib.lib(), eng._p + "policy_logits")
        assert fn(None, blob.dev_ptr(), None, 4, params.data_ptr(), rows.data_ptr(), None, None, None) != 0


# ---------------------------------------------------------------------------------------------------- drop-in
@pytest.mark.parametrize("name", ["small_mixed", "hlg", "mlp_small"])
def test_dropin_on_cuda_agrees_with_cpu_modules(name, golden_dir, dev):
    z, _, states, policy_net = load_policy(name, golden_dir)
    with torch.no_grad():
        cpu = policy_net(tensorfy(states))
    policy_net.to(dev)
    gpu = policy_net(tensorfy(states))
    n_cap, e_cap = int(z["n_cap"]), int(z["e_cap"])
    stage = z["stage"][:, :2].argmax(1)
    for s, width in ((0, e_cap), (1, n_cap)):
        b = int((stage == s).sum())
        if b == 0:
            assert gpu[s] is None and cpu[s] is None
            continue
        assert gpu[s].logits.shape == (b, width) and gpu[s].logits.is_cuda
        ref = {"x_logits": cpu[s].logits.numpy(), "x_probs": cpu[s].probs.numpy()}
        check_distribution("x", gpu[s], ref)
    assert torch.equal(gpu[2].cpu(), cpu[2])
