"""GPU (H100): the KL stop decided inside the step kernels (upb_set_target_kl).

References: a run of the same engine configuration with the stop off and diagnostics on, one minibatch step at a time,
with the parameters and optimiser state snapshotted before every step; the stop step is the first of its statistics
rows where the criterion, replayed in numpy float32, holds.  Both models; the fused step, the two-call path and the
first-step clip of CLIP_REFERENCE."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from harness import dev, reproducible_states, sgnn_agent, spawn, t

pytestmark = pytest.mark.gpu

STOP, SKIP = 13, 14
SPEC = synth.COMMUNITIES["small"]
LR = 3e-3                      # the policy moves far enough in a few steps for the KL to grow from step to step


class Case:
    """One minibatch of B graphs; old log-probs a little off the log-probs at the start, so the KL starts small and
    grows as the steps move the policy."""

    def __init__(self, model, dev, B=96, seed=5):
        if model == "sgnn":
            states, actions = synth.make_states(seed, "small", B)
            self.flat = PL.default_init(seed)
        else:
            states, actions = reproducible_states(seed, B)
            self.flat = PL.MLP.default_init(seed)
        self.model, self.dev, self.B = model, dev, B
        self.blob = pack_states(states).to(dev)
        adv, ret, exps = synth.make_ppo_targets(seed, B)
        exps[::5] = 0.0
        probe = Engine(dev, self.blob.n_cap, self.blob.e_cap, model=model)
        _, lp, _ = probe.forward(self.blob, t(self.flat, dev), t(actions, dev))
        probe.close()
        lp = lp.cpu().numpy().reshape(B, 1)
        flp = (lp + np.random.default_rng(seed).normal(0.0, 0.02, (B, 1))).astype(np.float32)
        self.args = tuple(t(x, dev) for x in (actions, adv, ret, flp, exps))
        self.n_ind = int((exps != 0).sum())

    def engine(self, clip_mode=_lib.CLIP_NEVER, grid=0, **kw):
        return Engine(self.dev, self.blob.n_cap, self.blob.e_cap, model=self.model, clip_mode=clip_mode,
                      grid_limit=grid, lr=LR, **kw)

    def step(self, eng, p, grad, two_call=False):
        a = (self.blob, p) + self.args + (1.0 / self.B, 1.0 / self.n_ind)
        if two_call:
            eng.ppo_grad(*a, out=grad)
            eng.apply(p, grad)
        else:
            eng.ppo_step(*a, out=grad)


def opt_state(eng):
    m, v, steps = eng.get_opt_state()
    return m.copy(), v.copy(), steps.copy()


def reference(case, n, clip_mode=_lib.CLIP_NEVER, grid=0, two_call=False):
    """Stop off, diagnostics on: rows, and (params, m, v, steps) before every step and after the last."""
    eng = case.engine(clip_mode, grid, diagnostics=True)
    p = t(case.flat, case.dev).clone()
    rows, snaps = [], []
    for _ in range(n):
        snaps.append((p.cpu().numpy().copy(),) + opt_state(eng))
        g = eng.new_grad_buffer()
        case.step(eng, p, g, two_call)
        torch.cuda.synchronize()
        rows.append(g.cpu().numpy().copy())
    snaps.append((p.cpu().numpy().copy(),) + opt_state(eng))
    eng.close()
    return np.stack(rows), snaps


def q_values(rows, so):
    """S8 / max(S4, 1) per row (float64), the quantity the target is compared with."""
    return rows[:, so + 8].astype(np.float64) / np.maximum(rows[:, so + 4].astype(np.float64), 1.0)


def replay_stop(rows, so, target):
    """First row where the device criterion holds in numpy float32 (None: never)."""
    limit = np.float32(1.5 * float(np.float32(target)))
    s8 = rows[:, so + 8].astype(np.float32)
    s4 = rows[:, so + 4].astype(np.float32)
    hit = np.flatnonzero(s8 > limit * np.maximum(s4, np.float32(1.0)))
    return int(hit[0]) if hit.size else None


def target_for(rows, so, s):
    """A float32 target whose stop step, replayed, is s (s must raise the running maximum of q)."""
    q = q_values(rows, so)
    prev = q[:s].max() if s else 0.0
    assert q[s] > prev, (s, q)
    tgt = float(np.float32((prev + q[s]) / 2 / 1.5))
    assert replay_stop(rows, so, tgt) == s, (s, q, tgt)
    return tgt


def records(rows, so):
    q = q_values(rows, so)
    return [i for i in range(len(q)) if q[i] > (q[:i].max() if i else 0.0)]


def run_with_target(case, target, n, clip_mode=_lib.CLIP_NEVER, grid=0, two_call=False):
    eng = case.engine(clip_mode, grid, target_kl=target)
    p = t(case.flat, case.dev).clone()
    rows = []
    for _ in range(n):
        g = torch.full((eng.grad_stride,), float("nan"), device=case.dev)
        case.step(eng, p, g, two_call)
        rows.append(g)
    torch.cuda.synchronize()
    return eng, p, np.stack([r.cpu().numpy() for r in rows])


def check_stopped_at(case, eng, p, rows, ref_rows, snaps, s):
    so, npar = eng.stat_offset, eng.num_params
    pp, m, v, steps = snaps[s]
    m2, v2, steps2 = opt_state(eng)
    got = p.cpu().numpy()
    assert np.array_equal(got, pp), (s, np.flatnonzero(got != pp)[:8])       # not one element half-updated
    assert np.array_equal(m2, m) and np.array_equal(v2, v) and np.array_equal(steps2, steps), s
    for i in range(s + 1):
        assert np.array_equal(rows[i, :npar], ref_rows[i, :npar]), i
        assert np.array_equal(rows[i, so:so + 9], ref_rows[i, so:so + 9]), (i, rows[i, so:so + 9], ref_rows[i, so:so + 9])
        assert not rows[i, so + 9:so + 13].any() and not rows[i, so + 15:].any(), i
        assert rows[i, so + STOP] == (1.0 if i == s else 0.0) and rows[i, so + SKIP] == 0.0, i
    for i in range(s + 1, rows.shape[0]):
        want = np.zeros(eng.grad_stride, np.float32)
        want[so + SKIP] = 1.0
        assert np.array_equal(rows[i], want), i


def set_target(eng, value):
    return _lib.lib().upb_set_target_kl(eng._ctx, C.c_float(value))


# ---- 1. off is today ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("two_call", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_is_bit_identical_to_a_context_that_never_set_it(model, two_call, dev):
    case = Case(model, dev, B=64)
    out = []
    for mode in ("never", "zero", "set_then_zero", "never_fires"):
        eng = case.engine()
        if mode == "zero":
            assert set_target(eng, 0.0) == 0
        elif mode == "set_then_zero":
            assert set_target(eng, 0.01) == 0 and set_target(eng, 0.0) == 0
        elif mode == "never_fires":
            assert set_target(eng, 1e30) == 0
        for bad in (-1.0, float("nan"), float("inf")):
            assert set_target(eng, bad) == -1 and b"target_kl" in _lib.lib().upb_last_error()    # UPB_ERR_ARG
        p = t(case.flat, dev).clone()
        before = eng.launches
        rows = []
        for _ in range(3):
            g = torch.full((eng.grad_stride,), float("nan"), device=dev)
            case.step(eng, p, g, two_call)
            rows.append(g)
        torch.cuda.synchronize()
        out.append((p.cpu().numpy(), opt_state(eng), np.stack([r.cpu().numpy() for r in rows]), eng.launches - before))
        eng.close()
    base = out[0]
    so = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    for k, (p, (m, v, st), rows, launches) in enumerate(out[1:], 1):
        assert np.array_equal(p, base[0]) and launches == base[3], k
        assert all(np.array_equal(a, b) for a, b in zip((m, v, st), base[1])), k
        if k < 3:
            assert np.array_equal(rows, base[2]), k
        else:             # on but never firing: the rows differ at most in slot 8
            keep = np.ones(rows.shape[1], bool)
            keep[so + 8] = False
            assert np.array_equal(rows[:, keep], base[2][:, keep])
            assert not base[2][:, so + 8].any() and rows[:, so + 8].any()


# ---- 2. device decision = host replay; 3. every grid size ------------------------------------------------------------
@pytest.mark.parametrize("path", ["fused", "two_call"])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_stop_step_matches_the_float32_replay(model, path, dev):
    case = Case(model, dev)
    two_call = path == "two_call"
    clip = _lib.CLIP_ALWAYS if two_call else _lib.CLIP_NEVER
    n = 6
    ref_rows, snaps = reference(case, n, clip)
    so = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    rec = records(ref_rows, so)
    wanted = [0, 1, next(i for i in rec if i >= 2)]
    assert set(wanted) <= set(rec), (rec, q_values(ref_rows, so))
    for s in wanted:
        eng, p, rows = run_with_target(case, target_for(ref_rows, so, s), n, clip, two_call=two_call)
        check_stopped_at(case, eng, p, rows, ref_rows, snaps, s)
        eng.close()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_first_step_clip_of_clip_reference_can_stop(model, dev):
    case = Case(model, dev)
    ref_rows, snaps = reference(case, 3, _lib.CLIP_REFERENCE)
    so = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    eng, p, rows = run_with_target(case, target_for(ref_rows, so, 0), 3, _lib.CLIP_REFERENCE)
    check_stopped_at(case, eng, p, rows, ref_rows, snaps, 0)
    eng.close()


@pytest.mark.parametrize("model,grid", [("sgnn", g) for g in (1, 2, 7, 113, 114, 115, 132)] +
                         [("mlp", g) for g in (1, 2, 80, 81, 82, 132)])
def test_every_grid_size(model, grid, dev):
    case = Case(model, dev, B=150)
    ref_rows, snaps = reference(case, 4, grid=grid)
    so = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    rec = [i for i in records(ref_rows, so) if i >= 1]
    s = rec[0]
    eng, p, rows = run_with_target(case, target_for(ref_rows, so, s), 4, grid=grid)
    assert eng.grid == min(grid, torch.cuda.get_device_properties(dev).multi_processor_count)
    check_stopped_at(case, eng, p, rows, ref_rows, snaps, s)
    eng.close()


# ---- 4. boundary ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_boundary_targets_stop_exactly_where_the_replay_does(model, dev):
    case = Case(model, dev, B=64)
    n = 3
    ref_rows, snaps = reference(case, n)
    so = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    q0 = np.float32(q_values(ref_rows, so)[0] / 1.5)
    below, above = [q0], [q0]
    for _ in range(3):
        below.append(np.nextafter(below[-1], np.float32(0)))
        above.append(np.nextafter(above[-1], np.float32(np.inf)))
    targets = sorted(set(below + above))
    expect = [replay_stop(ref_rows, so, float(x)) for x in targets]
    assert 0 in expect and any(e != 0 for e in expect), (targets, expect)      # fp32(1.5 t) straddles row 0
    for tgt, s in zip(targets, expect):
        eng, p, rows = run_with_target(case, float(tgt), n)
        marked = np.flatnonzero(rows[:, so + STOP])
        assert (int(marked[0]) if marked.size else None) == s, (tgt, s, rows[:, so + STOP])
        if s is not None:
            check_stopped_at(case, eng, p, rows, ref_rows, snaps, s)
        eng.close()


# ---- 5. skip and reset ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_skipped_steps_change_nothing_and_reset_trains_again(model, dev):
    case = Case(model, dev)
    ref_rows, snaps = reference(case, 4)
    so = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    s = [i for i in records(ref_rows, so) if i >= 1][0]
    eng, p, rows = run_with_target(case, target_for(ref_rows, so, s), s + 1)
    check_stopped_at(case, eng, p, rows, ref_rows, snaps, s)
    want_skip = np.zeros(eng.grad_stride, np.float32)
    want_skip[so + SKIP] = 1.0
    for two_call in (False, True, False):
        before = eng.launches
        g = torch.full((eng.grad_stride,), float("nan"), device=dev)
        case.step(eng, p, g, two_call)
        torch.cuda.synchronize()
        assert eng.launches - before == (3 if two_call else 1)
        assert np.array_equal(g.cpu().numpy(), want_skip), two_call
        check_stopped_at(case, eng, p, rows, ref_rows, snaps, s)
    # after the reset (and a target that no longer fires) the next step is the reference's step s, bit for bit
    eng.reset_kl_stop()
    assert set_target(eng, 1e30) == 0
    g = eng.new_grad_buffer()
    case.step(eng, p, g)
    torch.cuda.synchronize()
    pp, m, v, steps = snaps[s + 1]
    m2, v2, steps2 = opt_state(eng)
    assert np.array_equal(p.cpu().numpy(), pp)
    assert np.array_equal(m2, m) and np.array_equal(v2, v) and np.array_equal(steps2, steps)
    gg = g.cpu().numpy()
    assert np.array_equal(gg[:eng.num_params], ref_rows[s, :eng.num_params])
    assert np.array_equal(gg[so:so + 9], ref_rows[s, so:so + 9]) and gg[so + STOP] == 0 and gg[so + SKIP] == 0
    eng.close()


# ---- 6. PPOUpdater / use_b200_update ---------------------------------------------------------------------------------
def updater_inputs(model, T=1000, seed=11):
    if model == "sgnn":
        states, actions = synth.make_states(seed, "small", T)
        flat = PL.default_init(seed)
    else:
        states, actions = reproducible_states(seed, T)
        flat = PL.MLP.default_init(seed)
    rng = np.random.default_rng(seed)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    exps = np.ones(T, np.float32); exps[::5] = 0.0
    return flat, (states, actions, rewards, masks, exps)


def run_updater(model, flat, inputs, dev, record=False, **kw):
    from drl_urban_planning_b200.ppo import PPOUpdater
    up = PPOUpdater(flat, SPEC.max_num_nodes, SPEC.max_num_edges, dev, lr=LR, gamma=0.99, tau=0.95, opt_num_epochs=4,
                    mini_batch_size=256, model=model, **kw)
    rows = []
    if record:
        step = up.minibatch_step

        def recording(*a):
            step(*a)
            rows.append(up.grad.clone())
        up.minibatch_step = recording
    logged = []
    np.random.seed(3)
    before = up.engine.launches
    out = up.update_params(*inputs, log_fn=lambda tag, v, s: logged.append((tag, v, s)), iteration=1)
    torch.cuda.synchronize()
    return up, logged, out, up.engine.launches - before, (np.stack([r.cpu().numpy() for r in rows]) if rows else None)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_updater_stops_where_the_replay_predicts(model, dev):
    flat, inputs = updater_inputs(model)
    nb, epochs = 1000 // 256, 4
    plain, log_plain, out_plain, l_plain, _ = run_updater(model, flat, inputs, dev)
    none, log_none, out_none, l_none, _ = run_updater(model, flat, inputs, dev, target_kl=None)
    assert log_none == log_plain and out_none.keys() == out_plain.keys() and l_none == l_plain
    assert all(out_none[k] == out_plain[k] for k in out_plain)
    assert np.array_equal(none.flat_params(), plain.flat_params())
    # the replay: the stop on but never firing trains exactly as off and fills slot 8 of every row
    far, log_far, out_far, l_far, rows = run_updater(model, flat, inputs, dev, record=True, target_kl=1e30)
    assert np.array_equal(far.flat_params(), plain.flat_params()) and l_far == l_plain
    assert out_far["kl_stop"] is None and out_far["steps_applied"] == nb * epochs
    so = far.engine.stat_offset
    k = next(i for i in records(rows, so) if i >= nb)          # a stop in a later epoch
    up, logged, out, launches, _ = run_updater(model, flat, inputs, dev, target_kl=target_for(rows, so, k))
    e, mb = divmod(k, nb)
    assert out["kl_stop"] == (e, mb) and out["steps_applied"] == k
    assert launches == l_plain - (epochs - 1 - e) * nb          # no later epoch was launched
    tags = [tag for tag, _, _ in logged]
    assert tags.count("loss/loss") == k + 1 and tags.count("loss/epoch_loss") == e + 1
    assert [s for tag, _, s in logged if tag == "loss/loss"] == list(range(k + 1))
    assert ("diag/steps_applied", float(k), 1) in logged
    assert [v for tag, v, _ in logged if tag == "loss/loss"] == [v for tag, v, _ in log_far if tag == "loss/loss"][:k + 1]
    assert up.loss_iter == k + 1
    # the next update resets the word and trains
    before = up.flat_params()
    np.random.seed(4)
    out2 = up.update_params(*inputs, iteration=2)
    assert out2["steps_applied"] >= 1 and not np.array_equal(up.flat_params(), before)


def test_use_b200_update_passes_target_kl(dev):
    """The agent path stops where PPOUpdater(target_kl=...) does on the same update."""
    from drl_urban_planning_b200.agent import use_b200_update
    flat, inputs = updater_inputs("sgnn")
    nb = 1000 // 256
    far, _, _, _, rows = run_updater("sgnn", flat, inputs, dev, record=True, target_kl=1e30)
    so = far.engine.stat_offset
    k = next(i for i in records(rows, so) if i >= 1)
    tgt = target_for(rows, so, k)
    _, _, want, _, _ = run_updater("sgnn", flat, inputs, dev, target_kl=tgt)
    logged = []
    ag = sgnn_agent(dev, SPEC.max_num_nodes, SPEC.max_num_edges, flat, logged, lr=LR, num_optim_epoch=4,
                    mini_batch_size=256)
    with pytest.raises(ValueError):
        use_b200_update(ag, target_kl=-1.0)
    ctl = use_b200_update(ag, target_kl=tgt)
    assert ctl.updater.target_kl == tgt and ctl.updater.engine.target_kl == tgt
    states, actions, rewards, masks, exps = inputs
    np.random.seed(3)
    ag.update_params(types.SimpleNamespace(states=states, actions=actions, rewards=rewards, masks=masks, exps=exps), 1)
    assert want["kl_stop"] == divmod(k, nb)
    assert ("diag/steps_applied", float(k), 1) in logged
    assert [tag for tag, _, _ in logged].count("loss/loss") == k + 1 and ag.loss_iter == k + 1


# ---- 7. two GPUs ----------------------------------------------------------------------------------------------------
def _dist_worker(rank, world, target):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    flat, inputs = updater_inputs("sgnn", T=512)
    out = {}
    for use_peers in (False, True):
        from drl_urban_planning_b200.ppo import PPOUpdater
        up = PPOUpdater(flat, SPEC.max_num_nodes, SPEC.max_num_edges, torch.device("cuda", rank), lr=LR, gamma=0.99,
                        tau=0.95, opt_num_epochs=4, mini_batch_size=128, use_peers=use_peers, target_kl=target)
        np.random.seed(3)
        o = up.update_params(*inputs)
        out[use_peers] = (o["kl_stop"], up.flat_params(), up.engine.peer_timeouts() if up.fused_exchange else 0)
    dist.destroy_process_group()
    return out


def test_two_gpu_ranks_stop_at_the_same_step():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _dist_worker, 2e-4)
    for use_peers in (False, True):
        (s0, p0, t0), (s1, p1, t1) = got[0][use_peers], got[1][use_peers]
        assert s0 == s1 and np.array_equal(p0, p1) and t0 == 0 and t1 == 0, use_peers
