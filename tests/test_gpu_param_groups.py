"""GPU (H100): parameter groups and frozen tensors, both models.

1. Identity: a table with every tensor trained in one group at the engine's lr and weight decay is bit-identical to no
   table (parameters, moments, per-segment counters, gradient / statistics rows), on the fused step with and without
   max_grad_norm, the two-call path with CLIP_REFERENCE's first-step clip and CLIP_ALWAYS, skip_nonfinite, target_kl and
   the fused tail at grid sizes where one CTA owns several slices; each tensor's count follows its segment's.
2. use_b200_update(param_groups=True) against the oracle ports with torch.optim.Adam rebuilt over the same groups and
   requires_grad_(False) on the frozen tensors: a frozen encoder (unchanged bit for bit, zero gradient columns), two
   groups with their own lr and weight decay, and freeze-then-unfreeze with each tensor's count equal to the port's
   opt.state[p]["step"], with land-use-only updates that leave the road head absent, and the diagnostics' gradient norms
   equal to clip_grad_norm_'s over the trained tensors.  A non-finite step the guard skips keeps every count.
3. A checkpoint taken with frozen tensors resumes bit-identically; value_norm refuses a frozen val_w2."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.agent import use_b200_update
import cross_path as XP
from harness import (Case, assert_same_state, dev, fused_step, nan_buffer, rel, reproducible_states, t, two_call_step,
                     update_losses)
from oracle import mlp_port as MP, torch_port as TP
from test_gpu_live_hyperparams import SPEC, T, batch, flat_init, make_agent, port_iteration

pytestmark = pytest.mark.gpu

LR = 2.0 ** -11            # an fp32 number: the context's lr from upb_create is (double)(float)lr


def layout(model):
    return PL.MLP if model == "mlp" else PL.SGNN


def seg_of(lay):
    """Each tensor's segment: 0 encoder / value, 1 land-use head, 2 road head."""
    return [0 if sl.owner != "pol" else (1 if sl.name.startswith("lu_") else 2) for sl in lay.slots.values()]


@pytest.fixture(scope="module")
def cases(dev):
    states, actions = reproducible_states(41, 150)
    return {m: Case(dev, m, states, actions, 41) for m in ("sgnn", "mlp")}


# ---- 1. identity -------------------------------------------------------------------------------------------------------
PATHS = {
    "fused": dict(clip_mode=_lib.CLIP_NEVER),
    "fused_max_grad_norm": dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=0.05),
    "two_call_reference_clip": dict(clip_mode=_lib.CLIP_REFERENCE),
    "two_call_clip_always": dict(clip_mode=_lib.CLIP_ALWAYS),
    "skip_nonfinite": dict(clip_mode=_lib.CLIP_NEVER, skip_nonfinite=True),
    "two_call_skip_nonfinite": dict(clip_mode=_lib.CLIP_ALWAYS, skip_nonfinite=True),
    "target_kl": dict(clip_mode=_lib.CLIP_NEVER, target_kl=0.02),
}
SELS = [None, list(range(0, 150, 3)), [i for i in range(150) if i % 7 != 0], list(range(1, 150, 2))]


def check_identity(c, kw, grid=0):
    e_off = c.engine(lr=LR, weight_decay=2.0 ** -9, grid_limit=grid, **kw)
    e_on = c.engine(lr=LR, weight_decay=2.0 ** -9, grid_limit=grid, **kw)
    n = len(c.layout.slots)
    e_on.set_param_groups([LR] * n, [2.0 ** -9] * n, [True] * n)
    p_off, p_on = t(c.flat, c.dev).clone(), t(c.flat, c.dev).clone()
    seg = seg_of(c.layout)
    for k, sel in enumerate(SELS):
        step = two_call_step if kw.get("clip_mode") == _lib.CLIP_ALWAYS else fused_step
        g_off = step(e_off, c, p_off, sel)
        g_on = step(e_on, c, p_on, sel)
        steps = assert_same_state(e_off, p_off, g_off, e_on, p_on, g_on, (kw, k))
        assert e_on.get_tensor_steps().tolist() == [int(steps[1 + s]) for s in seg], k
    return e_on


@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_every_tensor_in_one_group_is_bit_identical_to_no_table(model, path, cases):
    eng = check_identity(cases[model], PATHS[path])
    if path == "target_kl":
        assert eng.get_opt_state()[2][0] < len(SELS)          # the stop came mid-sequence


@pytest.mark.parametrize("grid", XP.SGNN_GRIDS)
def test_identity_at_sgnn_fused_tail_grids(grid, cases):
    check_identity(cases["sgnn"], PATHS["fused"], grid)


@pytest.mark.parametrize("grid", XP.MLP_GRIDS)
def test_identity_at_mlp_fused_tail_grids(grid, cases):
    check_identity(cases["mlp"], PATHS["fused"], grid)


def guarded_step(eng, c, params, sel, two_call, bad):
    """One step on the graphs `sel`; bad: every return NaN, so the guard skips the step."""
    args = list(c.step_args(sel))
    if bad:
        args[2] = torch.full_like(args[2], float("nan"))
    g = nan_buffer(eng)
    if two_call:
        eng.ppo_grad(c.blob, params, *args, ids=c.ids(sel), out=g)
        eng.apply(params, g)
    else:
        eng.ppo_step(c.blob, params, *args, ids=c.ids(sel), out=g)
    return g


@pytest.mark.parametrize("path", ["skip_nonfinite", "two_call_skip_nonfinite"])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_a_skipped_nonfinite_step_keeps_every_count(model, path, cases):
    """The guard's skip with a table (the fused tail's, or k_apply's early return): nothing moves, every per-tensor count
    is kept, and the whole sequence is bit-identical to no table; a frozen encoder's counts stay 0 throughout."""
    c = cases[model]
    kw, two_call = PATHS[path], path.startswith("two_call")
    n = len(c.layout.slots)
    e_off = c.engine(lr=LR, **kw)
    e_on = c.engine(lr=LR, **kw)
    e_on.set_param_groups([LR] * n, [0.0] * n, [True] * n)
    e_fz = c.engine(lr=LR, **kw)
    n_enc = sum(1 for sl in c.layout.slots.values() if sl.owner == "enc")
    e_fz.set_param_groups([LR] * n, [0.0] * n, [k >= n_enc for k in range(n)])
    ps = {e: t(c.flat, c.dev).clone() for e in (e_off, e_on, e_fz)}
    seg = seg_of(c.layout)
    for k, (sel, bad) in enumerate([(SELS[1], False), (SELS[2], True), (SELS[3], False)]):
        before = {e: (ps[e].clone(), e.get_opt_state(), e.get_tensor_steps()) for e in (e_on, e_fz)}
        gs = {e: guarded_step(e, c, ps[e], sel, two_call, bad) for e in (e_off, e_on, e_fz)}
        torch.cuda.synchronize()
        a, b = gs[e_off].cpu().numpy(), gs[e_on].cpu().numpy()
        assert np.array_equal(a, b, equal_nan=True), (k, np.flatnonzero(~((a == b) | (np.isnan(a) & np.isnan(b))))[:8])
        assert torch.equal(ps[e_off], ps[e_on]), k
        for x, y in zip(e_off.get_opt_state(), e_on.get_opt_state()):
            assert np.array_equal(x, y), k
        steps = e_on.get_opt_state()[2]
        assert e_on.get_tensor_steps().tolist() == [int(steps[1 + s]) for s in seg], k
        assert not e_fz.get_tensor_steps()[:n_enc].any(), k
        for e in (e_on, e_fz):
            row = gs[e].cpu().numpy()
            assert (row[e.stat_offset + 19] == 1.0) == bad, k                 # the guard's mark
            if bad:
                p0, (m0, v0, s0), ts0 = before[e]
                m1, v1, s1 = e.get_opt_state()
                assert torch.equal(ps[e], p0) and np.array_equal(m0, m1) and np.array_equal(v0, v1), k
                assert s0.tolist() == s1.tolist() and e.get_tensor_steps().tolist() == ts0.tolist(), k


@pytest.mark.parametrize("path", ["fused", "two_call_clip_always"])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_frozen_tensor_columns_are_zero_and_unchanged(model, path, cases):
    """Engine level: a frozen encoder's gradient columns are 0 in every row and its parameters and moments do not move;
    the other tensors step."""
    c = cases[model]
    eng = c.engine(lr=LR, **PATHS[path])
    n = len(c.layout.slots)
    trained = [sl.owner != "enc" for sl in c.layout.slots.values()]
    eng.set_param_groups([LR] * n, [0.0] * n, trained)
    params = t(c.flat, c.dev).clone()
    enc = c.layout.encoder_end
    step = two_call_step if path != "fused" else fused_step
    for sel in SELS:
        g = step(eng, c, params, sel).cpu().numpy()
        assert not g[:enc].any() and g[enc:c.layout.num_params].any()
    torch.cuda.synchronize()
    p = params.cpu().numpy()
    m, v, steps = eng.get_opt_state()
    assert np.array_equal(p[:enc], c.flat[:enc]) and not m[:enc].any() and not v[:enc].any()
    assert not np.array_equal(p[enc:], c.flat[enc:])
    ts = eng.get_tensor_steps()
    assert ts[:sum(1 for x in trained if not x)].tolist() == [0] * sum(1 for x in trained if not x)
    assert steps[0] == len(SELS)


# ---- 2. against the oracle ports ---------------------------------------------------------------------------------------
def port_of(model, flat):
    return TP.PortAgent(flat) if model == "sgnn" else MP.MLPPortAgent(flat)


def regroup_port(port, groups):
    """port.opt rebuilt over `groups` [(slot names, lr, weight_decay)] with its state kept; tensors in no group get
    requires_grad_(False), so that clip_grad_norm_ and Adam.step skip them as torch does."""
    trained = {n for names, _, _ in groups for n in names}
    for n, p in port.P.items():
        p.requires_grad_(n in trained)
    old = port.opt.state
    port.opt = torch.optim.Adam([dict(params=[port.P[n] for n in names], lr=lr, weight_decay=wd)
                                 for names, lr, wd in groups], eps=1e-5)
    for p, s in old.items():
        port.opt.state[p] = s


def regroup_agent(ag, groups):
    """agent.optimizer rebuilt over the same groups of the agent's modules, requires_grad as the port's."""
    by_slot = {}
    for key, p in ag.actor_critic_net.named_parameters():
        for sl in layout_of(ag).slots.values():
            if PL.state_dict_keys(sl)[0] == key:
                by_slot[sl.name] = p
    trained = {n for names, _, _ in groups for n in names}
    for n, p in by_slot.items():
        p.requires_grad_(n in trained)
    ag.optimizer = torch.optim.Adam([dict(params=[by_slot[n] for n in names], lr=lr, weight_decay=wd)
                                     for names, lr, wd in groups], eps=ag.cfg.eps)


def layout_of(ag):
    return PL.MLP if getattr(ag.cfg, "agent", "rl-sgnn") == "rl-mlp" else PL.SGNN


def port_steps(port, lay):
    return [int(port.opt.state[port.P[n]]["step"]) if port.P[n] in port.opt.state else 0 for n in lay.slots]


def land_use_batch(seed):
    """T land-use graphs only (the road head is absent from every minibatch), rl-mlp-reproducible as batch()'s."""
    b = batch(seed)
    rng = np.random.default_rng(seed)
    b.states, b.actions = [], np.zeros((T, 2), np.float32)
    for i in range(T):
        n = int(rng.integers(8, SPEC.max_num_nodes + 1))
        e = int(rng.integers(n, min(2 * n, SPEC.max_num_edges) + 1))
        st, a = synth.make_exact_state(rng, SPEC, n, e, 1 + i % 2, 0)
        b.states.append(st)
        b.actions[i, 0] = a
    return b


def record_port_norms(port, lay):
    """port.norms gets, after every backward and before any clip, clip_grad_norm_'s norms over the tensors that have a
    gradient: (encoder + policy heads, encoder + value head, all), as diag/grad_norm_policy, _value and diag/grad_norm."""
    port.norms = []
    owner = {sl.name: sl.owner for sl in lay.slots.values()}
    backward = port.backward

    def recorded(*args):
        out = backward(*args)
        sq = dict(enc=0.0, pol=0.0, val=0.0)
        for name, p in port.P.items():
            if p.grad is not None:
                sq[owner[name]] += float((p.grad.double() ** 2).sum())
        port.norms.append((np.sqrt(sq["enc"] + sq["pol"]), np.sqrt(sq["enc"] + sq["val"]), np.sqrt(sum(sq.values()))))
        return out

    port.backward = recorded


def run_schedule(model, dev, schedule, seed=7, diagnostics=False, **kw):
    """update_params of use_b200_update(param_groups=True, **kw) and of the port, one update per entry of `schedule`
    (a list of groups, or (groups, batch) to give the update's rollout); yields (iteration, controller, port, got
    losses, want losses, the update's log) after each update.  With max_grad_norm the port does not clip (pass a bound
    the norms stay below)."""
    lay = layout(model)
    flat = flat_init(model, seed)
    logged = []
    ag = make_agent(model, dev, flat, logged)
    ctl = use_b200_update(ag, param_groups=True, diagnostics=diagnostics, **kw)
    port = port_of(model, flat)
    if kw.get("max_grad_norm"):
        port.steps_done = 1               # both ports clip on their first step only: never
    record_port_norms(port, lay)
    mod = TP if model == "sgnn" else MP
    epochs, B = ag.cfg.num_optim_epoch, ag.cfg.mini_batch_size
    for it, entry in enumerate(schedule):
        groups, b = entry if isinstance(entry, tuple) else (entry, batch(50 + it))
        regroup_agent(ag, groups)
        regroup_port(port, groups)
        start = len(logged)
        np.random.seed(it)
        ag.update_params(b, it)
        np.random.seed(it)
        want = port_iteration(port, mod, b, ag.gamma, ag.tau, epochs, B)
        got = update_losses(logged[start:])
        yield it, ctl, port, got, want, logged[start:]


def names(model, owners):
    return [sl.name for sl in layout(model).slots.values() if sl.owner in owners]


@pytest.mark.parametrize("clip", ["reference", "max_grad_norm"])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_frozen_encoder_follows_the_port(model, clip, dev):
    lay = layout(model)
    heads = [(names(model, ("pol", "val")), 4e-4, 0.0)]
    flat0 = flat_init(model, 7)
    enc = lay.encoder_end
    kw = dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=1e6) if clip == "max_grad_norm" else {}
    for it, ctl, port, got, want, logs in run_schedule(model, dev, [heads] * 3, diagnostics=True, **kw):
        assert np.allclose(got, want, rtol=2e-4, atol=2e-5), (it, np.abs(got - want).max())
        p = ctl.updater.flat_params()
        assert rel(p, port.flat()) < 2e-5, it
        assert np.array_equal(p[:enc], flat0[:enc]), it
        m, v, _ = ctl.updater.engine.get_opt_state()
        assert not m[:enc].any() and not v[:enc].any(), it
        assert ctl.updater.engine.get_tensor_steps().tolist() == port_steps(port, lay), it
        nb = T // ctl.updater.mini_batch_size
        assert not ctl.updater._grad_ring[:nb, :enc].any(), it
        # the gradient norms leave the frozen tensors out, as clip_grad_norm_ skips a grad that is None
        ref = np.array(port.norms[-nb:])
        tags = ["diag/grad_norm_policy", "diag/grad_norm_value"] + (["diag/grad_norm"] if kw else [])
        for j, tag in enumerate(tags):
            gn = np.array([v for name, v, s in logs if name == tag])
            assert gn.shape == (nb,), (it, tag)
            assert np.allclose(gn, ref[:, j], rtol=2e-4, atol=1e-7), (it, tag, gn, ref[:, j])


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_two_groups_follow_the_port(model, dev):
    groups = [(names(model, ("enc",)), 1e-4, 1e-4), (names(model, ("pol", "val")), 4e-4, 0.0)]
    lay = layout(model)
    for it, ctl, port, got, want, _ in run_schedule(model, dev, [groups] * 3):
        assert np.allclose(got, want, rtol=2e-4, atol=2e-5), (it, np.abs(got - want).max())
        assert rel(ctl.updater.flat_params(), port.flat()) < 2e-5, it
        assert ctl.updater.engine.get_tensor_steps().tolist() == port_steps(port, lay), it


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_freeze_then_unfreeze_keeps_each_tensor_count(model, dev):
    every = [(list(layout(model).slots), 4e-4, 0.0)]
    heads = [(names(model, ("pol", "val")), 4e-4, 0.0)]
    lay = layout(model)
    val_w0 = list(lay.slots).index("val_w0")
    road = [k for k, n in enumerate(lay.slots) if n.startswith("road_")]
    # the fourth and fifth updates see land-use graphs only: the road head is trained but absent, so it keeps its count
    # (the head rule) while the encoder is frozen in the fourth and trained again in the fifth
    lu = [land_use_batch(80), land_use_batch(81)]
    schedule = [every, every, heads, (heads, lu[0]), (every, lu[1]), every]
    prev = None
    for it, ctl, port, got, want, _ in run_schedule(model, dev, schedule):
        assert np.allclose(got, want, rtol=2e-4, atol=2e-5), (it, np.abs(got - want).max())
        assert rel(ctl.updater.flat_params(), port.flat()) < 2e-5, it
        ts = ctl.updater.engine.get_tensor_steps()
        assert ts.tolist() == port_steps(port, lay), it
        steps4 = ctl.updater.engine.get_opt_state()[2]
        assert ts[val_w0] == steps4[1], it                     # the value head never froze: its segment's count
        if it >= 2:                                            # the encoder missed the third update's steps
            assert ts[0] < ts[val_w0], (it, ts.tolist())
        if it in (3, 4):
            assert ts[road].tolist() == prev[road].tolist() and ts[road].tolist() == [steps4[3]] * len(road), it
            assert (ts[0] == prev[0]) == (it == 3), it            # frozen in the fourth update, trained in the fifth
        prev = ts


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_checkpoint_with_frozen_tensors_resumes_bit_identically(model, dev):
    lay = layout(model)
    heads = [(names(model, ("pol", "val")), 4e-4, 0.0)]
    flat = flat_init(model, 9)
    logs = [[], []]
    ag = make_agent(model, dev, flat, logs[0])
    ctl = use_b200_update(ag, param_groups=True, clip_mode=_lib.CLIP_NEVER)
    regroup_agent(ag, heads)
    for it in range(2):
        np.random.seed(it)
        ag.update_params(batch(60 + it), it)
    state = ctl.optimizer_state()
    assert "tensor_steps" in state and state["tensor_steps"][0] == 0
    ag2 = make_agent(model, dev, ctl.updater.flat_params(), logs[1])
    ctl2 = use_b200_update(ag2, param_groups=True, clip_mode=_lib.CLIP_NEVER)
    regroup_agent(ag2, heads)
    ctl2.load_optimizer_state(state, clip_like_new_process=False)
    ag2.loss_iter = ag.loss_iter
    for it in range(2, 4):
        for a in (ag, ag2):
            np.random.seed(it)
            a.update_params(batch(60 + it), it)
    torch.cuda.synchronize()
    assert np.array_equal(ctl.updater.flat_params(), ctl2.updater.flat_params())
    for x, y in zip(ctl.updater.engine.get_opt_state(), ctl2.updater.engine.get_opt_state()):
        assert np.array_equal(x, y)
    assert np.array_equal(ctl.updater.engine.get_tensor_steps(), ctl2.updater.engine.get_tensor_steps())


@pytest.mark.parametrize("frozen", ["val_w2", "val_b2"])
def test_value_norm_refuses_a_frozen_last_value_layer(frozen, dev):
    ag = make_agent("sgnn", dev, flat_init("sgnn", 3), [])
    ctl = use_b200_update(ag, param_groups=True, value_norm=True)
    regroup_agent(ag, [([n for n in PL.SGNN.slots if n != frozen], 4e-4, 0.0)])
    with pytest.raises(ValueError, match=f"value_norm rescales {frozen}"):
        ag.update_params(batch(70), 0)
    assert ctl.updater.engine.get_opt_state()[2][0] == 0
