"""GPU (H100): the PPO diagnostics the step kernels report -- statistics slots 8-12 (approx. KL, clip count, sums of R,
R^2 and V - R), the per-row gradient norms of upb_grad_norms / upb_mlp_grad_norms, and PPOUpdater(diagnostics=True).

References: float64 values from the oracles (oracle/sgnn_numpy.py, oracle/mlp_port.py) at the parameters the step
starts from; the two-call path for the fused tails; the reference's own gradients (tests/golden) for the norms."""
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.diagnostics import NAMES, ppo_diagnostics
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states, synth_states
from harness import dev, reproducible_states, spawn, t

pytestmark = pytest.mark.gpu

EPS = 0.2          # clip_epsilon of every shipped cfg and of Engine's default


def load_fixture(golden_dir, name):
    """states, actions, flat parameters, advantages, returns, fixed log-probs and exps of a golden fixture; edge_empty
    stores forward values only, so its PPO targets are seeded."""
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    if "digest" in z.files:
        states, actions = synth_states(int(z["seed"]), str(z["community"]), int(z["count"]))
    else:
        states, actions = expand_states(z), z["actions"]
    B = len(states)
    if "advantages" in z.files:
        adv, ret, flp, exps = (np.array(z[k]) for k in ("advantages", "returns", "fixed_log_probs", "exps"))
    else:
        adv, ret, exps = synth.make_ppo_targets(13, B)
        flp = np.full((B, 1), -3.0, np.float32)
    # old log-probs away from the new ones, so that the KL and the clip count are not trivially zero
    flp = (flp.reshape(B, 1) + np.random.default_rng(B).normal(0.0, 0.2, (B, 1))).astype(np.float32)
    return states, np.asarray(actions, np.float32), z, adv, ret, flp, exps


def oracle_value_logp(model, flat, states, actions, adv, ret, flp, exps):
    """float64 per-graph value and log-prob at `flat`."""
    if model == "sgnn":
        from oracle import sgnn_numpy as ON
        r = ON.ppo_minibatch(flat, states, actions, adv, ret, flp, exps, want_grad=False)
        return np.asarray(r["value"]), np.asarray(r["log_prob"])
    from oracle import mlp_port as MP
    P = MP.params_from_flat(flat, dtype=torch.float64)
    b = MP.stack_states(states)
    with torch.no_grad():
        V = MP.value(P, b).numpy().ravel()
        lp, _ = MP.log_prob_entropy(P, b, torch.tensor(actions))
    return V, lp.numpy().ravel()


CASES = [("sgnn", "small_mixed"), ("sgnn", "hlg256"), ("sgnn", "concept_mixed256"), ("sgnn", "edge_empty"),
         ("mlp", "mlp_small"), ("mlp", "mlp_hlg")]


@pytest.mark.parametrize("zero_fifth", [False, True])
@pytest.mark.parametrize("model,name", CASES)
def test_statistics_slots_match_float64_oracle(model, name, zero_fifth, golden_dir, dev):
    states, actions, z, adv, ret, flp, exps = load_fixture(golden_dir, name)
    exps = np.array(exps, np.float32).reshape(-1)
    if zero_fifth:
        exps[::5] = 0.0
    B = len(states)
    blob = pack_states(states).to(dev)
    if name == "concept_mixed256":
        import shape_cases as SC
        assert any(SC.is_big(*row[:3]) for row in blob.info.astype(np.int64)), "graphs on the large-graph path"
    flat = np.asarray(z["params"], np.float32)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model, diagnostics=True)
    plain = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    n_ind = int((exps != 0).sum())
    step_args = (t(flat, dev), t(actions, dev), t(adv, dev), t(ret, dev), t(flp, dev), t(exps, dev), 1.0 / B,
                 1.0 / max(n_ind, 1))
    grad = eng.ppo_grad(blob, *step_args)
    base = plain.ppo_grad(blob, *step_args).cpu().numpy()
    so = eng.stat_offset
    st = grad[so:so + _lib.UPB_STAT_COUNT].cpu().numpy().astype(np.float64)
    assert st[3] == B and st[4] == n_ind and st[7] == 0
    assert not st[13:].any()
    # without diagnostics the buffer is the one a build without them writes: slots 8-27 zero, the rest unchanged
    assert not base[so + 8:].any()
    if model == "sgnn":              # (k_mlp's shared-memory atomics reorder the last bits of land-use gradients)
        assert np.array_equal(base[:so + 8], grad.cpu().numpy()[:so + 8])

    V, lp = oracle_value_logp(model, flat, states, actions, adv, ret, flp, exps)
    R = np.asarray(ret, np.float64).reshape(-1)
    ind = exps != 0
    d = lp - np.asarray(flp, np.float64).reshape(-1)
    r = np.exp(d)
    outside = ind & ~((r >= 1 - EPS) & (r <= 1 + EPS))
    near = ind & (np.abs(np.abs(r - 1) - EPS) <= 1e-5)
    if B >= 8:
        assert outside.any() and (ind & ~outside).any(), "both sides of the clip range are exercised"
    assert (outside & ~near).sum() <= st[9] <= (outside & ~near).sum() + near.sum(), (st[9], outside.sum(), near.sum())
    scale_r, scale_e = np.abs(R).sum(), np.abs(V - R).sum()
    assert abs(st[10] - R.sum()) <= 1e-4 * scale_r
    assert abs(st[11] - (R * R).sum()) <= 1e-4 * (R * R).sum()
    assert abs(st[12] - (V - R).sum()) <= 1e-4 * scale_e
    assert abs(st[0] - ((V - R) ** 2).sum()) <= 1e-4 * ((V - R) ** 2).sum()
    kl_ref = (np.expm1(d) - d)[ind].sum() / max(n_ind, 1)
    got = ppo_diagnostics(st[None], np.zeros((1, 3)))
    assert abs(got["approx_kl"][0] - kl_ref) <= max(1e-3 * kl_ref, 1e-7), (got["approx_kl"][0], kl_ref)
    ev_ref = 1 - np.var(V - R) / np.var(R)
    assert abs(got["explained_variance"][0] - ev_ref) <= 1e-4 * max(abs(ev_ref), 1.0), (got["explained_variance"], ev_ref)


def lpt_ids(eng, blob, sel):
    return t(eng.balance_ids(np.asarray(sel), Engine.graph_cost(blob.info.astype(np.int64))).astype(np.int32),
             eng.device)


def fused_against_two_call(model, blob, flat, args, B, n_ind, grid, dev, exact):
    """Three steps through ppo_step (LPT ids; the first step clips and takes the two-call path) against ppo_grad +
    apply; the statistics rows of every step."""
    e1 = Engine(dev, blob.n_cap, blob.e_cap, model=model, grid_limit=grid, diagnostics=True)
    e2 = Engine(dev, blob.n_cap, blob.e_cap, model=model, grid_limit=grid, diagnostics=True)
    assert e2.grid == min(grid, torch.cuda.get_device_properties(dev).multi_processor_count)
    ids = lpt_ids(e2, blob, np.arange(B))
    p1, p2 = t(flat, dev).clone(), t(flat, dev).clone()
    so = e1.stat_offset
    for step in range(3):
        g1 = torch.full((e1.grad_stride,), float("nan"), device=dev)
        g2 = torch.full((e2.grad_stride,), float("nan"), device=dev)
        e1.ppo_grad(blob, p1, *args, 1.0 / B, 1.0 / n_ind, ids=ids, out=g1)
        e1.apply(p1, g1)
        before = e2.launches
        e2.ppo_step(blob, p2, *args, 1.0 / B, 1.0 / n_ind, ids=ids, out=g2)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (step > 0), step
        s1 = g1[so:so + _lib.UPB_STAT_COUNT].cpu().numpy()
        s2 = g2[so:so + _lib.UPB_STAT_COUNT].cpu().numpy()
        assert not s1[13:].any() and not s2[13:].any(), step
        assert s2[9] == s1[9] and s2[3] == s1[3] and s2[4] == s1[4], step
        if exact:
            assert np.array_equal(s1[:13], s2[:13]), (step, s1[:13], s2[:13])
        else:
            assert np.allclose(s2[:13], s1[:13], rtol=1e-5, atol=1e-6), (step, s1[:13], s2[:13])


@pytest.mark.parametrize("grid", [1, 2, 7, 113, 114, 115, 132])
def test_sgnn_fused_tail_carries_the_new_slots(grid, golden_dir, dev):
    states, actions, z, adv, ret, flp, exps = load_fixture(golden_dir, "hlg256")
    B = len(states)
    blob = pack_states(states).to(dev)
    args = tuple(t(x, dev) for x in (actions, adv, ret, flp, exps))
    fused_against_two_call("sgnn", blob, z["params"], args, B, int((exps != 0).sum()), grid, dev, exact=False)


@pytest.mark.parametrize("grid", [1, 2, 80, 81, 82, 132])
def test_mlp_fused_tail_carries_the_new_slots_bit_for_bit(grid, dev):
    states, actions = reproducible_states(21, 150)      # graphs whose k_mlp gradient rows are reproducible
    B = len(states)
    adv, ret, exps = synth.make_ppo_targets(21, B)
    exps[::5] = 0.0
    flp = np.random.default_rng(21).normal(-3.0, 0.3, size=(B, 1)).astype(np.float32)
    blob = pack_states(states).to(dev)
    args = tuple(t(x, dev) for x in (actions, adv, ret, flp, exps))
    fused_against_two_call("mlp", blob, PL.MLP.default_init(21), args, B, int((exps != 0).sum()), grid, dev, exact=True)


@pytest.mark.parametrize("model,name", [("sgnn", "small_mixed"), ("sgnn", "hlg256"), ("mlp", "mlp_small")])
def test_grad_norms_match_float64_and_the_reference_gradients(model, name, golden_dir, dev):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    states = (synth_states(int(z["seed"]), str(z["community"]), int(z["count"]))[0] if "digest" in z.files
              else expand_states(z))
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model, diagnostics=True)
    args = tuple(t(z[k], dev) for k in ("actions", "advantages", "returns", "fixed_log_probs", "exps"))
    n_ind = int((z["exps"] != 0).sum())
    rows = torch.zeros(3, eng.grad_stride, device=dev)
    for k in range(3):       # the reference's steps start from params, params_after[0], params_after[1]
        start = z["params"] if k == 0 else z["params_after"][k - 1]
        eng.ppo_grad(blob, t(start, dev), *args, 1.0 / B, 1.0 / n_ind, out=rows[k])
    before = eng.launches
    sq = eng.grad_norms(rows)
    torch.cuda.synchronize()
    assert eng.launches - before == 1
    again = eng.grad_norms(rows)
    assert torch.equal(sq, again)                           # fixed summation order
    layout = PL.MLP if model == "mlp" else PL.SGNN
    bounds = (0, layout.encoder_end, layout.policy_end, layout.num_params)

    def groups(g):
        g = np.asarray(g, np.float64)
        return np.array([(g[bounds[j]:bounds[j + 1]] ** 2).sum() for j in range(3)])

    got = sq.cpu().numpy().astype(np.float64)
    g = rows.cpu().numpy()
    for k in range(3):
        want = groups(g[k])
        assert np.allclose(np.sqrt(got[k]), np.sqrt(want), rtol=1e-6, atol=0), (k, got[k], want)
        ref = groups(z["grads"][k])
        assert np.allclose(np.sqrt(got[k]), np.sqrt(ref), rtol=1e-4, atol=0), (k, got[k], ref)
        d = ppo_diagnostics(np.zeros((1, 16)), got[k:k + 1])
        assert np.isclose(d["grad_norm_policy"][0], np.sqrt(ref[0] + ref[1]), rtol=1e-4)
        assert np.isclose(d["grad_norm_value"][0], np.sqrt(ref[0] + ref[2]), rtol=1e-4)


LOSS_TAGS = {"loss/loss", "loss/value_loss", "loss/surr_loss", "loss/entropy_loss", "loss/epoch_loss",
             "loss/epoch_value_loss", "loss/epoch_surr_loss", "loss/epoch_entropy_loss", "loss/total_loss",
             "loss/total_value_loss", "loss/total_surr_loss", "loss/total_entropy_loss"}
TOTAL_KEYS = {"total_loss", "total_value_loss", "total_surr_loss", "total_entropy_loss"}


def run_updater(make, inputs, np_seed, diagnostics):
    from drl_urban_planning_b200.ppo import PPOUpdater
    up = make(PPOUpdater, diagnostics)
    logged = []
    np.random.seed(np_seed)
    out = up.update_params(*inputs, log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    torch.cuda.synchronize()
    return up, logged, out


def check_diagnostics_on_and_off(make, inputs, np_seed, epochs, nb):
    off, log_off, out_off = run_updater(make, inputs, np_seed, False)
    on, log_on, out_on = run_updater(make, inputs, np_seed, True)
    assert np.array_equal(on.flat_params(), off.flat_params())
    assert [x for x in log_on if x[0].startswith("loss/")] == log_off
    assert {tag for tag, _, _ in log_off} == LOSS_TAGS and set(out_off) == TOTAL_KEYS
    assert on.engine.launches - off.engine.launches == epochs          # one norm launch per epoch, none per step
    steps = [s for tag, _, s in log_on if tag == "loss/loss"]
    for name in NAMES:
        assert [s for tag, _, s in log_on if tag == "diag/" + name] == steps
    # the last epoch's values from its ring rows, through the numpy function
    ring = on._grad_ring[:nb]
    so = on.engine.stat_offset
    assert not off._grad_ring[:nb, so + 8:].any()        # off: the fused steps leave the diagnostic slots zero
    assert ring[:, so + 8:so + 13].any() and not ring[:, so + 13:].any()
    want = ppo_diagnostics(ring[:, so:so + 16].cpu().numpy(), on.engine.grad_norms(ring).cpu().numpy())
    for name in NAMES:
        got = np.array([v for tag, v, _ in log_on if tag == "diag/" + name])
        assert got.shape == (epochs * nb,)
        assert np.array_equal(got[-nb:], want[name], equal_nan=True), name
        assert np.isfinite(got).all(), name
        assert out_on["total_" + name] == pytest.approx(got.mean(), rel=1e-12)
        assert [v for tag, v, s in log_on if tag == "diag/total_" + name] == [out_on["total_" + name]]
    assert set(out_on) == TOTAL_KEYS | {"total_" + n for n in NAMES}
    assert (np.array([v for tag, v, _ in log_on if tag == "diag/approx_kl"]) > 0).any()      # the policy moved


def test_updater_diagnostics_on_update_small(golden_dir):
    z = np.load(os.path.join(golden_dir, "update_small.npz"))
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    states = expand_states(z)
    dev = torch.device("cuda", 0)

    def make(cls, diagnostics):
        return cls(z["params"], int(z["n_cap"]), int(z["e_cap"]), dev, gamma=float(z["gamma_tau"][0]),
                   tau=float(z["gamma_tau"][1]), opt_num_epochs=epochs, mini_batch_size=B,
                   clip_mode=_lib.CLIP_REFERENCE, diagnostics=diagnostics)
    check_diagnostics_on_and_off(make, (states, z["actions"], z["rewards"], z["masks"], z["exps"]), np_seed, epochs,
                                 T // B)


def test_updater_diagnostics_on_rl_mlp(dev):
    T, B, epochs = 96, 32, 3
    states, actions = reproducible_states(31, T)
    rng = np.random.default_rng(31)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    exps = np.ones(T, np.float32); exps[::5] = 0.0
    spec = synth.COMMUNITIES["small"]

    def make(cls, diagnostics):
        return cls(PL.MLP.default_init(31), spec.max_num_nodes, spec.max_num_edges, dev, gamma=0.99, tau=0.95,
                   opt_num_epochs=epochs, mini_batch_size=B, model="mlp", diagnostics=diagnostics)
    check_diagnostics_on_and_off(make, (states, actions, rewards, masks, exps), 5, epochs, T // B)


# ---- two GPUs -------------------------------------------------------------------------------------------------------
def _dist_case():
    T = 96
    states, actions = synth.make_states(77, "small", T)
    rng = np.random.default_rng(77)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    exps = np.ones(T, np.float32); exps[::5] = 0.0
    return PL.default_init(77), states, actions, rewards, masks, exps


def _diag_run(dev, case, **kw):
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat, states, actions, rewards, masks, exps = case
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, gamma=0.99, tau=0.95, opt_num_epochs=2,
                    mini_batch_size=32, diagnostics=True, **kw)
    logged = []
    np.random.seed(5)
    up.update_params(states, actions, rewards, masks, exps, log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    return up, np.array([[v for tag, v, _ in logged if tag == "diag/" + n] for n in NAMES])


def _dist_worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    out = {}
    for mode, use_peers in (("nccl", False), ("peers", True)):
        up, diag = _diag_run(torch.device("cuda", rank), _dist_case(), use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        out[mode] = diag
    dist.destroy_process_group()
    return out


def test_two_gpu_ranks_report_the_global_diagnostics():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _dist_worker)
    _, want = _diag_run(torch.device("cuda", 0), _dist_case(), process_group=None)
    for mode in ("nccl", "peers"):
        assert np.array_equal(got[0][mode], got[1][mode]), mode
        assert np.allclose(got[0][mode], want, rtol=1e-4, atol=1e-6), (mode, np.abs(got[0][mode] - want).max())
