"""GPU (H100): Adam options, both models: betas, eps, AMSGrad and decoupled weight decay (Engine.set_adam and
per-tensor settings in Engine.set_param_groups).

Teacher-forced: each step's reduced gradient is read from the gradient buffer, and the parameters, both moments and
AMSGrad's max_exp_avg_sq must equal the fp32 replay of tests/adamw_oracle.py bit for bit, on the fused step, the fused
step with max_grad_norm and with skip_nonfinite (the clip's tail at coefficient 1), the two-call path (k_apply's table),
the parameter-group tail with per-tensor settings, and the SGNN's fused tail at every grid size of the cross-path table.
Steps that change nothing (a KL stop, a non-finite step the guard skips, an absent head) neither decay nor touch the
max.  At the default settings the switch changes nothing, launches included, and an AMSGrad run resumed from its
checkpointed state is bit-identical to an uninterrupted one."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL
import adamw_oracle as AO
import cross_path as XP
from harness import Case, assert_same_state, dev, fused_step, nan_buffer, reproducible_states, t, two_call_step

pytestmark = pytest.mark.gpu

LR, WD = 3.7e-4, 0.05          # lr not an fp32 number: the step size is formed from the double

OPTIONS = {
    "adamw": ((0.9, 0.999), 1e-8, False, True),
    "amsgrad": ((0.8, 0.99), 1e-6, True, False),
    "adamw_amsgrad": ((0.5, 0.9), 1e-7, True, True),
}


@pytest.fixture(scope="module")
def cases(dev):
    states, actions = reproducible_states(43, 150)
    return {m: Case(dev, m, states, actions, 43) for m in ("sgnn", "mlp")}


def seg_of(lay):
    return [0 if sl.owner != "pol" else (1 if sl.name.startswith("lu_") else 2) for sl in lay.slots.values()]


def stat_offset(lay):
    return _lib.UPB_MLP_STAT_OFFSET if lay is PL.MLP else _lib.UPB_STAT_OFFSET


def snapshot(eng, params):
    torch.cuda.synchronize()
    m, v, steps = eng.get_opt_state()
    vmax = eng.get_amsgrad_state()
    return params.cpu().numpy(), m, v, (np.zeros_like(m) if vmax is None else vmax), steps


def replay(lay, before, grad, settings, lr, wd, counts):
    """The expected (params, m, v, vmax) after one step: each tensor k with its settings[k] = (betas, eps, amsgrad,
    decoupled), lr[k], wd[k] and count after the step counts[k] (None: not stepped)."""
    p, m, v, vmax, _ = (x.copy() for x in before)
    g = grad[:lay.num_params]
    for k, sl in enumerate(lay.slots.values()):
        if counts[k] is None:
            continue
        (b1, b2), eps, ams, dec = settings[k]
        s = slice(sl.offset, sl.offset + sl.size)
        p[s], m[s], v[s], vm = AO.adam32(p[s], g[s], m[s], v[s], vmax[s], counts[k], lr[k], wd[k], b1, b2, eps, ams,
                                         dec)
        if ams:
            vmax[s] = vm
    return p, m, v, vmax


def context_counts(lay, grad, steps_after):
    """Each tensor's count after a step of the context's table (its segment's), None where its head was absent."""
    st = grad[stat_offset(lay):]
    live = [True, st[5] > 0, st[6] > 0]
    return [int(steps_after[1 + s]) if live[s] else None for s in seg_of(lay)]


def assert_replayed(eng, params, want, what):
    got = snapshot(eng, params)
    for name, a, b in zip(("params", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"), got[:4], want):
        assert np.array_equal(a, b), (what, name, np.flatnonzero(a != b)[:8])


SELS = [None, list(range(0, 150, 3)), [i for i in range(150) if i % 7 != 0]]
# graphs of one stage only: the other head is absent from the minibatch (torch's grad None)
ONE_STAGE = "one_stage"


def run_context(c, opt, path_kw, step, sels=SELS, grid=0):
    n = len(c.layout.slots)
    eng = c.engine(lr=LR, weight_decay=WD, grid_limit=grid, **path_kw)
    eng.set_lr(LR)              # the double (upb_create keeps (double)(float)lr)
    betas, eps, ams, dec = OPTIONS[opt]
    eng.set_adam(betas, eps, ams, dec)
    params = t(c.flat, c.dev).clone()
    for k, sel in enumerate(sels):
        if sel == ONE_STAGE:
            sel = [i for i in range(c.count) if c.stage[i] == c.stage[0]]
        before = snapshot(eng, params)
        g = step(eng, c, params, sel)
        torch.cuda.synchronize()
        gh = g.cpu().numpy()
        counts = context_counts(c.layout, gh, eng.get_opt_state()[2])
        want = replay(c.layout, before, gh, [OPTIONS[opt]] * n, [LR] * n, [WD] * n, counts)
        assert_replayed(eng, params, want, (opt, path_kw, k))
    return eng


PATHS = {
    "fused": (dict(clip_mode=_lib.CLIP_NEVER), fused_step),
    "fused_max_grad_norm": (dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=1e6), fused_step),
    "fused_skip_nonfinite": (dict(clip_mode=_lib.CLIP_NEVER, skip_nonfinite=True), fused_step),
    "two_call": (dict(clip_mode=_lib.CLIP_NEVER), two_call_step),
}


@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("opt", sorted(OPTIONS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_context_settings_replay_bit_for_bit(model, opt, path, cases):
    kw, step = PATHS[path]
    run_context(cases[model], opt, kw, step, SELS + [ONE_STAGE])


@pytest.mark.parametrize("grid", XP.SGNN_GRIDS)
def test_sgnn_fused_tail_at_every_grid_size(grid, cases):
    run_context(cases["sgnn"], "adamw_amsgrad", dict(clip_mode=_lib.CLIP_NEVER), fused_step, grid=grid)


@pytest.mark.parametrize("grid", XP.MLP_GRIDS)
def test_mlp_fused_tail_at_every_grid_size(grid, cases):
    run_context(cases["mlp"], "adamw_amsgrad", dict(clip_mode=_lib.CLIP_NEVER), fused_step, grid=grid)


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


@pytest.mark.parametrize("opt", sorted(OPTIONS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_reference_first_step_clip_against_float64(model, opt, cases):
    """CLIP_REFERENCE's first step takes the two-call path with the reference's two-group clip (coefficients < 1) and
    k_apply's table.  Against float64: the two clip coefficients formed from the step's unclipped gradient buffer, then
    adam64 per tensor.  Each parameter step within 1e-4 of float64's plus 2 ulps; the moments and the max within 1e-4
    of the size of their gradient terms plus 2 ulps."""
    c = cases[model]
    lay, n = c.layout, len(c.layout.slots)
    eng = c.engine(lr=LR, weight_decay=WD, clip_mode=_lib.CLIP_REFERENCE)
    eng.set_lr(LR)
    eng.set_adam(*OPTIONS[opt])
    params = t(c.flat, c.dev).clone()
    # advantages and returns scaled up so that both groups' norms exceed 1 and the clip acts
    act, adv, ret, fixed, exps = c.dev_args
    g = nan_buffer(eng)
    eng.ppo_step(c.blob, params, act, adv * 100.0, ret * 100.0, fixed, exps, *c.step_args()[5:], out=g)   # clips:
    torch.cuda.synchronize()                    # ppo_grad + apply inside the library
    gh = g.cpu().numpy()
    g64 = gh[:lay.num_params].astype(np.float64)
    enc, pol = lay.encoder_end, lay.policy_end
    se, sp, sv = (float((g64[a:b] ** 2).sum()) for a, b in ((0, enc), (enc, pol), (pol, lay.num_params)))
    k1 = min(1.0 / (np.sqrt(se + sp) + 1e-6), 1.0)
    k2 = min(1.0 / (np.sqrt(k1 * k1 * se + sv) + 1e-6), 1.0)
    assert k1 < 0.5 or k2 < 0.5, (k1, k2)              # the clip acts
    coef = np.concatenate([np.full(enc, k1 * k2), np.full(pol - enc, k1), np.full(lay.num_params - pol, k2)])
    counts = context_counts(lay, gh, eng.get_opt_state()[2])
    (b1, b2), eps, ams, dec = OPTIONS[opt]
    p0 = c.flat.astype(np.float64)
    got_p, got_m, got_v, got_x = snapshot(eng, params)[:4]
    zero = np.zeros(lay.num_params)
    want_p, want_m, want_v, want_x = p0.copy(), zero.copy(), zero.copy(), zero.copy()
    for k, sl in enumerate(lay.slots.values()):
        if counts[k] is None:
            continue
        s = slice(sl.offset, sl.offset + sl.size)
        want_p[s], want_m[s], want_v[s], want_x[s] = AO.adam64(p0[s], g64[s] * coef[s], zero[s], zero[s], zero[s],
                                                                counts[k], LR, WD, b1, b2, eps, ams, dec)
    d_got, d_want = got_p.astype(np.float64) - p0, want_p - p0
    assert (np.abs(d_got - d_want) <= 1e-4 * np.abs(d_want) + 2 * ulp(c.flat)).all(), np.abs(d_got - d_want).max()
    # the moments against the size of the gradient's terms (the clipped gradient and the coupled decay may cancel)
    g_size = np.abs(g64 * coef) + (0.0 if dec else WD * np.abs(p0))
    assert (np.abs(got_m - want_m) <= 1e-4 * (1 - b1) * g_size + 2 * ulp(want_m)).all()
    assert (np.abs(got_v - want_v) <= 1e-4 * (1 - b2) * g_size ** 2 + 2 * ulp(want_v)).all()
    if ams:
        assert (np.abs(got_x - want_x) <= 1e-4 * (1 - b2) * g_size ** 2 + 2 * ulp(want_x)).all()
    assert not np.array_equal(got_p, c.flat)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_per_tensor_settings_in_the_parameter_group_tail(model, cases):
    c = cases[model]
    lay, n = c.layout, len(c.layout.slots)
    rng = np.random.default_rng(5)
    opts = list(OPTIONS.values()) + [((0.9, 0.999), 1e-5, False, False)]
    settings = [opts[k % len(opts)] for k in range(n)]
    lr = [LR * (1 + k / 32) for k in range(n)]
    wd = [float(x) for x in rng.choice([0.0, 0.01, 0.1], n)]
    trained = [k % 5 != 3 for k in range(n)]
    for path, step in (("fused", fused_step), ("two_call", two_call_step)):
        eng = c.engine(lr=LR, clip_mode=_lib.CLIP_NEVER)
        eng.set_param_groups(lr, wd, trained, adam=[(*b, e, a, d) for b, e, a, d in settings])
        params = t(c.flat, c.dev).clone()
        for k, sel in enumerate(SELS):
            before = snapshot(eng, params)
            ts0 = eng.get_tensor_steps()
            g = step(eng, c, params, sel)
            torch.cuda.synchronize()
            ts1 = eng.get_tensor_steps()
            counts = [int(ts1[j]) if ts1[j] != ts0[j] else None for j in range(n)]
            assert all(counts[j] is None for j in range(n) if not trained[j])
            want = replay(lay, before, g.cpu().numpy(), settings, lr, wd, counts)
            assert_replayed(eng, params, want, (path, k))


def _poisoned(c):
    """A NaN return: the value gradient is NaN, so the guard skips the step."""
    ret = c.dev_args[2].clone()
    ret[3] = float("nan")
    return c.dev_args[:2] + (ret,) + c.dev_args[3:]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_steps_that_change_nothing_neither_decay_nor_touch_the_max(model, cases):
    c = cases[model]
    for kw in (dict(skip_nonfinite=True), dict(target_kl=1e-12)):
        for step in ("fused", "two_call"):
            eng = c.engine(lr=LR, weight_decay=WD, clip_mode=_lib.CLIP_NEVER, **kw)
            eng.set_adam(*OPTIONS["adamw_amsgrad"])
            params = t(c.flat, c.dev).clone()
            rng = np.random.default_rng(2)
            eng.set_amsgrad_state(rng.uniform(0, 1e-3, eng.num_params).astype(np.float32))
            before = snapshot(eng, params)
            args = _poisoned(c) if "skip_nonfinite" in kw else c.dev_args
            inv = (1.0 / c.count, 1.0 / max(int((c.exps != 0).sum()), 1))
            g = nan_buffer(eng)
            if step == "fused":
                eng.ppo_step(c.blob, params, *args, *inv, out=g)
            else:
                eng.ppo_grad(c.blob, params, *args, *inv, out=g)
                eng.apply(params, g)
            after = snapshot(eng, params)
            for a, b in zip(before[:4], after[:4]):
                assert np.array_equal(a, b), (kw, step)
            assert after[4].tolist() == before[4].tolist()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_default_settings_are_the_untouched_path(model, cases):
    """set_adam at the engine's own betas and eps (coupled, no AMSGrad, and decoupled with weight decay 0) leaves every
    launch and every bit as an engine that never called it."""
    c = cases[model]
    for kw, step in ((dict(clip_mode=_lib.CLIP_NEVER), fused_step), (dict(clip_mode=_lib.CLIP_REFERENCE), fused_step),
                     (dict(clip_mode=_lib.CLIP_ALWAYS), two_call_step)):
        for wd, dec in ((WD, False), (0.0, True)):
            e_off = c.engine(lr=LR, weight_decay=wd, **kw)
            e_on = c.engine(lr=LR, weight_decay=wd, **kw)
            e_on.set_adam(e_on.betas, e_on.eps, False, dec)
            p_off, p_on = t(c.flat, c.dev).clone(), t(c.flat, c.dev).clone()
            for sel in SELS:
                l_off, l_on = e_off.launches, e_on.launches
                g_off = step(e_off, c, p_off, sel)
                g_on = step(e_on, c, p_on, sel)
                assert e_on.launches - l_on == e_off.launches - l_off
                assert_same_state(e_off, p_off, g_off, e_on, p_on, g_on, (kw, wd, dec))
            assert e_on.get_amsgrad_state() is None
            with pytest.raises(_lib.UpbError, match="no parameter groups"):      # no table was synthesised
                e_on.get_tensor_steps()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_amsgrad_checkpoint_resumes_bit_identically(model, cases):
    c = cases[model]
    mk = lambda: c.engine(lr=LR, weight_decay=WD, clip_mode=_lib.CLIP_NEVER)
    whole = mk()
    whole.set_adam(*OPTIONS["adamw_amsgrad"])
    p_whole = t(c.flat, c.dev).clone()
    for sel in SELS:
        fused_step(whole, c, p_whole, sel)
    first = mk()
    first.set_adam(*OPTIONS["adamw_amsgrad"])
    p = t(c.flat, c.dev).clone()
    for sel in SELS[:2]:
        fused_step(first, c, p, sel)
    m, v, steps = first.get_opt_state()
    vmax = first.get_amsgrad_state()
    resumed = mk()
    resumed.set_adam(*OPTIONS["adamw_amsgrad"])
    resumed.set_opt_state(m, v, steps)
    resumed.set_amsgrad_state(vmax)
    g = fused_step(resumed, c, p, SELS[2])
    torch.cuda.synchronize()
    assert np.array_equal(p.cpu().numpy(), p_whole.cpu().numpy())
    for a, b in zip(whole.get_opt_state(), resumed.get_opt_state()):
        assert np.array_equal(a, b)
    assert np.array_equal(whole.get_amsgrad_state(), resumed.get_amsgrad_state())
    assert np.isfinite(g.cpu().numpy()).all()


# ---- the user-facing path: use_b200_update(adam_options=True) against the oracle ports with torch's AdamW ----------------
def _by_slot(ag, lay):
    keys = {PL.state_dict_keys(sl)[0]: sl.name for sl in lay.slots.values()}
    return {keys[key]: p for key, p in ag.actor_critic_net.named_parameters()}


def _adamw_groups(model, grouped):
    """[(slot names, AdamW group keywords)]: one group of every tensor with AMSGrad, or the shared encoder at its own
    betas, eps, weight decay and AMSGrad beside the heads at AdamW's defaults and another lr."""
    lay = PL.MLP if model == "mlp" else PL.SGNN
    if not grouped:
        return [(list(lay.slots), dict(amsgrad=True))]
    enc = [n for n, sl in lay.slots.items() if sl.owner == "enc"]
    return [(enc, dict(betas=(0.8, 0.99), eps=1e-6, weight_decay=0.02, amsgrad=True)),
            ([n for n in lay.slots if n not in enc], dict(lr=3e-4))]


def _adamw(params_by_slot, groups):
    return torch.optim.AdamW([dict(params=[params_by_slot[n] for n in names], **kw) for names, kw in groups], lr=4e-4)


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_adamw_updates_follow_the_port(model, grouped, dev):
    """Three update_params of use_b200_update(adam_options=True[, param_groups=True]) with agent.optimizer an AdamW,
    against the oracle port whose optimizer is the same AdamW over its own tensors: the logged losses, the parameters
    and AMSGrad's max follow the port (the first step of each clips, as the reference's does)."""
    from drl_urban_planning_b200.agent import use_b200_update
    from oracle import mlp_port as MP, torch_port as TP
    from harness import rel, update_losses
    from test_gpu_live_hyperparams import batch, flat_init, make_agent, port_iteration
    lay = PL.MLP if model == "mlp" else PL.SGNN
    flat = flat_init(model, 7)
    logged = []
    ag = make_agent(model, dev, flat, logged)
    ctl = use_b200_update(ag, adam_options=True, param_groups=grouped)
    port = TP.PortAgent(flat) if model == "sgnn" else MP.MLPPortAgent(flat)
    groups = _adamw_groups(model, grouped)
    ag.optimizer = _adamw(_by_slot(ag, lay), groups)
    port.opt = _adamw(port.P, groups)
    ams = [n for names, kw in groups if kw.get("amsgrad") for n in names]
    mod = TP if model == "sgnn" else MP
    for it in range(3):
        b = batch(50 + it)
        start = len(logged)
        np.random.seed(it)
        ag.update_params(b, it)
        np.random.seed(it)
        want = port_iteration(port, mod, b, ag.gamma, ag.tau, ag.cfg.num_optim_epoch, ag.cfg.mini_batch_size)
        got = update_losses(logged[start:])
        assert np.allclose(got, want, rtol=2e-4, atol=2e-5), (it, np.abs(got - want).max())
        assert rel(ctl.updater.flat_params(), port.flat()) < 2e-5, it
        vmax = ctl.updater.engine.get_amsgrad_state()
        for name in ams:
            sl = lay.slots[name]
            ref = port.opt.state[port.P[name]]["max_exp_avg_sq"].detach().cpu().numpy().reshape(-1)
            assert rel(vmax[sl.offset:sl.offset + sl.size], ref) < 1e-3, (it, name)
    if not grouped:
        assert ctl.updater.hyperparameters()["eps"] == 1e-8 and ctl.updater.hyperparameters()["decoupled_weight_decay"]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_agent_amsgrad_checkpoint_resumes_bit_identically(model, dev):
    """B200Update.optimizer_state carries max_exp_avg_sq; a second agent that loads it continues bit-identically; a
    checkpoint without the key starts the buffer from zeros."""
    from drl_urban_planning_b200.agent import use_b200_update
    from test_gpu_live_hyperparams import batch, flat_init, make_agent
    lay = PL.MLP if model == "mlp" else PL.SGNN
    groups = _adamw_groups(model, False)

    def agent(flat, logs):
        ag = make_agent(model, dev, flat, logs)
        ctl = use_b200_update(ag, adam_options=True, clip_mode=_lib.CLIP_NEVER)
        ag.optimizer = _adamw(_by_slot(ag, lay), groups)
        return ag, ctl

    ag, ctl = agent(flat_init(model, 9), [])
    for it in range(2):
        np.random.seed(it)
        ag.update_params(batch(60 + it), it)
    state = ctl.optimizer_state()
    assert "max_exp_avg_sq" in state and state["max_exp_avg_sq"].any()
    ag2, ctl2 = agent(ctl.updater.flat_params(), [])
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
    assert np.array_equal(ctl.updater.engine.get_amsgrad_state(), ctl2.updater.engine.get_amsgrad_state())
    without = {k: v for k, v in state.items() if k != "max_exp_avg_sq"}
    ctl2.load_optimizer_state(without, clip_like_new_process=False)
    assert not ctl2.updater.engine.get_amsgrad_state().any()
