"""GPU (H100): the rl-mlp optimiser step in one cooperative launch (upb_mlp_ppo_step, mlp_fused_tail in
csrc/mlp_kernel.cuh) against the two-call path it replaces (upb_mlp_ppo_grad + upb_mlp_apply).

On one GPU the fused step reduces every gradient column in k_mlp_reduce's order and applies k_apply's Adam, so from
the same per-CTA gradient rows it is bit-identical: parameters, the whole gradient / statistics buffer, both Adam
moments and the four step counters are compared with np.array_equal, never a tolerance.  The per-CTA rows are
themselves reproducible only where k_mlp's node-gradient scatter is (harness.reproducible_states); ordinary land-use
graphs are compared within rounding.  The bit-identity check at the grid sizes around the 81 gradient slices, at each
optimiser setting, is written once in tests/cross_path.py.

Here: that check at the shipped settings, graphs beyond the shared-memory budget, the per-step liveness of the two policy heads, the golden trajectories
of the unmodified reference, the clip modes and the first-step clip latch after a resume, and the refusal to run with
peers connected."""
import types

import numpy as np
import pytest
import torch

import cross_path as XP
import shape_cases as SC
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from harness import (Agent, Case, Cfg, assert_same_state, dev, fused_step, heads, load, per_tensor_rel,
                     rel, reproducible_states, spawn, t, two_call_step)

pytestmark = pytest.mark.gpu

L = PL.MLP
HEADS = heads(L)


@pytest.fixture(scope="module")
def mixed(dev):
    """150 graphs of both stages (more than the 132 CTAs of a full grid), one exps == 0 entry, reproducible rows."""
    states, actions = reproducible_states(21, 150)
    stage = np.array([int(s[8].argmax()) for s in states])
    return Case(dev, "mlp", states, actions, 21, zero_exps=(int(np.flatnonzero(stage == 0)[1]),))


@pytest.mark.parametrize("grid", XP.MLP_GRIDS)
def test_fused_step_is_bit_identical_to_two_call_path(grid, mixed, dev):
    """cross_path.check_mlp_fused_bit_identical at the shipped settings: 4 steps (mixed, clipping; mixed; land-use
    only; mixed) at grids where one CTA owns every slice, several, one each with idle CTAs, and the full H100 grid."""
    XP.check_mlp_fused_bit_identical(mixed, "shipped", grid)


@pytest.mark.parametrize("grid", [3, 0])
def test_policy_head_liveness_across_fused_steps(grid, mixed, dev):
    """Minibatches mixed -> mixed -> land-use only -> road only -> land-use only -> road only -> mixed: the stage
    words are double-buffered by step parity, so a stale word would update the absent head two steps later.  The
    absent head's parameters and moments stay bit-untouched and every step equals the two-call path."""
    c = mixed
    lu, rd, allg = np.flatnonzero(c.stage == 0), np.flatnonzero(c.stage == 1), np.arange(c.count)
    e1 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid)
    e2 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for step, sel in enumerate([allg, allg, lu, rd, lu, rd, allg]):
        p_before = p2.cpu().numpy()
        m_before, v_before, _ = e2.get_opt_state()
        g1 = two_call_step(e1, c, p1, sel)
        g2 = fused_step(e2, c, p2, sel)
        steps = assert_same_state(e1, p1, g1, e2, p2, g2, step)
        p_now = p2.cpu().numpy()
        m_now, v_now, _ = e2.get_opt_state()
        for s, sl in HEADS.items():
            if not (c.stage[sel] == s).any():
                assert np.array_equal(p_now[sl], p_before[sl]), (step, s)
                assert np.array_equal(m_now[sl], m_before[sl]) and np.array_equal(v_now[sl], v_before[sl]), (step, s)
    assert steps.tolist() == [7, 7, 5, 5]


def reproducible_boundary_batch(seed):
    """The rows of tests/shape_cases.py BOUNDARY with every land-use graph cut to two candidates (module docstring):
    n = 464 / 465 of both stages, 2e = 5630 / 5632 / 5634, road k = 160 / 161, the hub graph, the 1000 / 3000 caps."""
    rng = np.random.default_rng(seed)
    states, actions = [], np.zeros((len(SC.BOUNDARY), 2), np.float32)
    for i, (_, n, e, k, stage, hub, isolated) in enumerate(SC.BOUNDARY):
        st, a = synth.make_exact_state(rng, SC.SPEC, n, e, k if stage == 1 else min(k, 2), stage, hub=hub,
                                       isolated=isolated)
        states.append(st)
        actions[i, stage] = a
    return states, actions


def run_against_two_call(c, dev, grid, steps, exact):
    e1 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid)
    e2 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    allg = np.arange(c.count)
    for step in range(steps):
        before = e2.launches
        g1 = two_call_step(e1, c, p1, allg)
        g2 = fused_step(e2, c, p2, allg)
        assert (e2.launches - before == 1) == (step > 0)
        if exact:
            assert_same_state(e1, p1, g1, e2, p2, g2, (grid, step))
            continue
        torch.cuda.synchronize()       # within rounding (the tolerances of test_fused_tail_at_every_grid_size)
        worst, where = per_tensor_rel(g2.cpu().numpy()[:L.num_params], g1.cpu().numpy()[:L.num_params], L)
        assert worst < 1e-5, (step, worst, where)
        assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, step
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    assert s1.tolist() == s2.tolist() == [steps] * 4
    assert rel(m2, m1) < 1e-5 and rel(v2, v1) < 1e-5


@pytest.mark.parametrize("grid", [2, 0])
def test_graphs_beyond_the_shared_memory_budget(grid, dev):
    """Graphs on both sides of k_mlp's shared-memory limits in fused steps: bit-identical to the two-call path on the
    reproducible boundary batch, within rounding on tests/shape_cases.py's own (land-use k = 160 / 161 / 3000)."""
    states, actions = reproducible_boundary_batch(3)
    c = Case(dev, "mlp", states, actions, 3, zero_exps=(5,))
    n, e, k, stage = c.info.T
    assert ((n == SC.NS) & (stage == 0)).any() and ((n == SC.NS + 1) & (stage == 0)).any()
    assert ((n == SC.NS) & (stage == 1)).any() and ((n == SC.NS + 1) & (stage == 1)).any()
    assert (2 * e == SC.AS).any() and (2 * e == SC.AS + 2).any()
    assert ((k == SC.KS) & (stage == 1)).any() and ((k == SC.KS + 1) & (stage == 1)).any()
    assert (n == 1000).any() and any(SC.degrees(s).max() == len(SC.degrees(s)) - 1 for s in states)
    run_against_two_call(c, dev, grid, 3, exact=True)
    states, actions, _ = SC.boundary_batch(3)
    c = Case(dev, "mlp", states, actions, 3, zero_exps=(5,))
    assert ((c.info[:, 2] == SC.KS + 1) & (c.info[:, 3] == 0)).any() and (c.info[:, 2] == 3000).any()
    run_against_two_call(c, dev, grid, 3, exact=False)


def test_ordinary_graphs_match_two_call_within_rounding(dev):
    """Generator-sized graphs of both stages (land-use nodes selected by many candidates) at the full grid."""
    stages = np.random.default_rng(22).integers(0, 2, 150)
    states, actions = synth.make_states(22, "small", 150, stages=stages)
    run_against_two_call(Case(dev, "mlp", states, actions, 22), dev, 0, 4, exact=False)


@pytest.mark.parametrize("name", ["mlp_small", "mlp_hlg"])
def test_golden_trajectory_through_the_fused_step(name, golden_dir, dev):
    """test_mlp_cuda_path_matches_reference with upb_mlp_ppo_step: the reference's losses, gradients and parameters
    after each of 3 steps (the first clips and falls back, the others run fused), same tolerances."""
    z = load(golden_dir, name)
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE, model="mlp")
    params = t(z["params"], dev).clone()
    n_ind = int((z["exps"] != 0).sum())
    args = tuple(t(z[k], dev) for k in ("actions", "advantages", "returns", "fixed_log_probs", "exps"))
    for k in range(3):
        before = eng.launches
        grad = eng.ppo_step(blob, params, *args, 1.0 / B, 1.0 / n_ind)
        assert (eng.launches - before == 1) == (k > 0)
        losses = eng.read_losses(grad)
        assert np.allclose(losses, z["losses"][k], rtol=1e-4, atol=1e-5), (k, losses, z["losses"][k])
        worst, where = per_tensor_rel(grad.cpu().numpy()[:L.num_params], z["grads"][k], L)
        assert worst < 1e-4, (k, worst, where)
        torch.cuda.synchronize()
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k


def test_clip_always_never_fuses(mixed, dev):
    c = mixed
    allg = np.arange(c.count)
    e1 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", clip_mode=_lib.CLIP_ALWAYS)
    e2 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", clip_mode=_lib.CLIP_ALWAYS)
    p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
    for step in range(3):
        assert not e2.next_step_fused()
        before = e2.launches
        g1 = two_call_step(e1, c, p1, allg)
        g2 = fused_step(e2, c, p2, allg)
        assert e2.launches - before == 3
        assert_same_state(e1, p1, g1, e2, p2, g2, step)


def trained_state(c, dev):
    """Adam state after two steps (global step 2), and the parameters they produced."""
    eng = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp")
    params = t(c.flat, dev).clone()
    for _ in range(2):
        fused_step(eng, c, params, np.arange(c.count))
    m, v, steps = eng.get_opt_state()
    assert steps[0] == 2
    return m, v, steps, params


def clipped_reference_step(c, dev, state, params):
    """The two-call path with clipping on, from a restored state."""
    m, v, steps = state
    ref = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", clip_mode=_lib.CLIP_ALWAYS)
    ref.set_opt_state(m, v, steps)
    p = params.clone()
    g = two_call_step(ref, c, p, np.arange(c.count))
    return ref, p, g


def test_resume_rearms_the_first_step_clip(mixed, dev):
    """set_opt_state(..., rearm_first_step_clip=True) on a state with a non-zero global step: the next step clips (it
    equals a clipping two-call step), next_step_fused() is False before it and True after it.  Without re-arming the
    restored step is fused."""
    c = mixed
    m, v, steps, params = trained_state(c, dev)
    ref, p_ref, g_ref = clipped_reference_step(c, dev, (m, v, steps), params)
    eng = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp")
    eng.set_opt_state(m, v, steps, rearm_first_step_clip=True)
    assert not eng.next_step_fused()
    p = params.clone()
    before = eng.launches
    g = fused_step(eng, c, p, np.arange(c.count))
    assert eng.launches - before == 3
    assert eng.next_step_fused()
    assert_same_state(ref, p_ref, g_ref, eng, p, g, "rearmed")
    # rearm_first_step_clip=False: continue as if never interrupted -- fused, equal to a non-clipping two-call step
    cont = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp")
    cont.set_opt_state(m, v, steps, rearm_first_step_clip=False)
    assert cont.next_step_fused()
    p_cont = params.clone()
    before = cont.launches
    g_cont = fused_step(cont, c, p_cont, np.arange(c.count))
    assert cont.launches - before == 1
    plain = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", clip_mode=_lib.CLIP_NEVER)
    plain.set_opt_state(m, v, steps)
    p_plain = params.clone()
    g_plain = two_call_step(plain, c, p_plain, np.arange(c.count))
    assert_same_state(plain, p_plain, g_plain, cont, p_cont, g_cont, "continued")


def mlp_agent(dev, n_cap, e_cap):
    """An rl-mlp agent as B200Update sees it (train.py --agent rl-mlp): cfg, device and the actor-critic modules."""
    from drl_urban_planning_b200.mlp import ActorCritic, create_mlp_model
    cfg = Cfg(n_cap, e_cap)
    cfg.agent = "rl-mlp"
    cfg.lr, cfg.eps, cfg.clip_epsilon, cfg.value_pred_coef, cfg.entropy_coef = 4e-4, 1e-5, 0.2, 0.5, 0.01
    cfg.gamma, cfg.tau, cfg.num_optim_epoch, cfg.mini_batch_size = 0.99, 0.95, 1, 16
    cfg.agent_specs, cfg.weightdecay = {}, 0.0
    torch.manual_seed(5)
    p, v = create_mlp_model(cfg, Agent())
    return types.SimpleNamespace(cfg=cfg, device=dev, actor_critic_net=ActorCritic(p, v))


@pytest.mark.parametrize("clip_like_new_process", [True, False])
def test_load_optimizer_state_on_an_rl_mlp_agent(clip_like_new_process, mixed, dev):
    """B200Update.load_optimizer_state on an rl-mlp agent: with the default clip_like_new_process=True the resumed
    run's first step clips, like the SGNN's and like the reference (a new process clips its first step)."""
    from drl_urban_planning_b200.agent import B200Update
    c = mixed
    m, v, steps, params = trained_state(c, dev)
    ctl = B200Update(mlp_agent(dev, c.blob.n_cap, c.blob.e_cap))
    eng = ctl.updater.engine
    assert eng.model == "mlp"
    ctl.load_optimizer_state({"exp_avg": m, "exp_avg_sq": v, "steps": steps}, clip_like_new_process=clip_like_new_process)
    assert eng.next_step_fused() == (not clip_like_new_process)
    got = ctl.optimizer_state()
    assert np.array_equal(got["exp_avg"], m) and got["steps"].tolist() == steps.tolist()
    p = params.clone()
    before = eng.launches
    g = fused_step(eng, c, p, np.arange(c.count))
    assert eng.launches - before == (3 if clip_like_new_process else 1)
    assert eng.next_step_fused()
    if clip_like_new_process:
        ref, p_ref, g_ref = clipped_reference_step(c, dev, (m, v, steps), params)
        assert_same_state(ref, p_ref, g_ref, eng, p, g, "load_optimizer_state")


def test_step_arguments_are_checked_before_launching(mixed, dev):
    """A fused step with a missing per-sample array is refused with UPB_ERR_ARG and launches nothing."""
    import ctypes as C
    c = mixed
    eng = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", clip_mode=_lib.CLIP_NEVER)
    assert eng.next_step_fused()
    params = t(c.flat, dev).clone()
    g = eng.new_grad_buffer()
    a = c.dev_args
    before = eng.launches
    rc = _lib.lib().upb_mlp_ppo_step(eng._ctx, c.blob.dev_ptr(), None, c.count, params.data_ptr(), a[0].data_ptr(),
                                     a[1].data_ptr(), a[2].data_ptr(), None, a[4].data_ptr(), C.c_float(1.0),
                                     C.c_float(1.0), g.data_ptr(), None)
    assert rc == -1 and b"mlp_ppo_step" in _lib.lib().upb_last_error()
    assert eng.launches == before
    torch.cuda.synchronize()
    assert np.array_equal(params.cpu().numpy(), c.flat)


def _peer_worker(rank, world):
    """Maps the peers' exchange buffers on an rl-mlp engine (connect_peers declines the model, so directly); the fused
    step must then refuse instead of launching a kernel whose local sums would skip the other ranks."""
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    states, actions = synth.make_states(40 + rank, "small", 16)
    c = Case(dev, "mlp", states, actions, 40 + rank)
    eng = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", clip_mode=_lib.CLIP_NEVER)
    assert not eng.connect_peers()
    mine = torch.frombuffer(bytearray(eng.peer_export()), dtype=torch.uint8).to(dev)
    everyone = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(everyone, mine)
    eng.peer_connect(world, rank, b"".join(bytes(x.cpu().numpy().tobytes()) for x in everyone))
    dist.barrier()
    out = {"fused": eng.next_step_fused()}
    before = eng.launches
    try:
        fused_step(eng, c, t(c.flat, dev).clone(), np.arange(c.count))
        out["error"] = None
    except _lib.UpbError as err:
        out["error"] = str(err)
    out["launched"] = eng.launches - before
    dist.barrier()
    dist.destroy_process_group()
    return out


def test_fused_step_refuses_with_peers_connected():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (on one GPU the argument checks are covered by "
                    "test_step_arguments_are_checked_before_launching)")
    got = spawn(2, _peer_worker)[0]
    assert got["fused"] is False and got["launched"] == 0
    assert got["error"] and "upb_mlp_ppo_grad" in got["error"], got
