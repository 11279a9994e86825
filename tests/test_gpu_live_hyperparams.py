"""GPU (H100): training with the agent's live hyperparameters, both models.

1. Values that never change issue no call and move nothing: use_b200_update reading an untouched optimizer and agent is
   bit-identical to a controller that never reads them (parameters, moments, counters, statistics rows, log, launches).
2. upb_set_lr: the step size is (float)(lr / bc1) with the double lr, bit for bit against a host replay of the Adam tail,
   on upb_apply and on the fused step at every fused-tail grid size.
3. A LambdaLR (CleanRL's linear anneal) or a ReduceLROnPlateau on agent.optimizer, with entropy_coef, clip_epsilon,
   mini_batch_size and opt_num_epochs changed between iterations, against the oracle ports replaying the same schedule.
4. The live values together with max_grad_norm, skip_nonfinite, target_kl and the KL penalty, a weight decay changed
   through the param group, and lr = 0: the update after the change is bit-identical to that of a controller built with
   the new values (fp32 numbers, so both hold the same ones) from the same parameters and Adam state."""
import math
import types
import warnings

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.agent import B200Update, use_b200_update
import cross_path as XP
from harness import (SHIPPED_CFG, Agent, Case, Cfg, dev, fused_step, nan_buffer, rel, reproducible_states, sgnn_agent, t,
                     update_losses)
from oracle import mlp_port as MP, torch_port as TP

pytestmark = pytest.mark.gpu

SPEC = synth.COMMUNITIES["small"]            # the graphs of harness.reproducible_states
N_CAP, E_CAP = SPEC.max_num_nodes, SPEC.max_num_edges
T = 48


def make_agent(model, dev, flat, logged, with_optimizer=True, **cfg):
    """A reference-shaped agent of `model` holding `flat`: cfg (SHIPPED_CFG unless `cfg` says otherwise), tb_logger into
    `logged`, and with_optimizer the attributes UrbanPlanningAgent.__init__ sets plus setup_optimizer's Adam."""
    if model == "sgnn":
        ag = sgnn_agent(dev, N_CAP, E_CAP, flat, logged, **cfg)
    else:
        from drl_urban_planning_b200.mlp import ActorCritic, create_mlp_model
        c = Cfg(N_CAP, E_CAP)
        c.agent, c.agent_specs = "rl-mlp", {}
        for k, v in {**SHIPPED_CFG, **cfg}.items():
            setattr(c, k, v)
        torch.manual_seed(5)
        p, v = create_mlp_model(c, Agent())
        ag = types.SimpleNamespace(cfg=c, device=dev, loss_iter=0, actor_critic_net=ActorCritic(p, v),
                                   tb_logger=types.SimpleNamespace(add_scalar=lambda tag, x, s: logged.append((tag, x, s))))
        ag.actor_critic_net.load_state_dict({k: torch.as_tensor(x) for k, x in PL.MLP.to_state_dict(flat).items()})
    if with_optimizer:
        c = ag.cfg
        ag.gamma, ag.tau, ag.clip_epsilon = c.gamma, c.tau, c.clip_epsilon
        ag.value_pred_coef, ag.entropy_coef = c.value_pred_coef, c.entropy_coef
        ag.opt_num_epochs, ag.mini_batch_size = c.num_optim_epoch, c.mini_batch_size
        ag.optimizer = torch.optim.Adam(ag.actor_critic_net.parameters(), lr=c.lr, eps=c.eps,
                                        weight_decay=getattr(c, "weightdecay", 0.0))
    return ag


def flat_init(model, seed):
    return PL.MLP.default_init(seed) if model == "mlp" else PL.default_init(seed)


def batch(seed):
    """T graphs whose rl-mlp gradient rows are run-to-run reproducible (harness.reproducible_states), and their rollout."""
    states, actions = reproducible_states(seed, T)
    rng = np.random.default_rng(seed)
    masks = np.ones(T, np.float32)
    masks[9::10] = 0.0
    exps = np.ones(T, np.float32)
    exps[3] = 0.0
    return types.SimpleNamespace(states=states, actions=actions, rewards=rng.standard_normal(T).astype(np.float32),
                                 masks=masks, exps=exps)


def fixed_update(ctl, b, iteration):
    """B200Update.update_params without reading the agent's values: what a run that never changes them computes."""
    agent = ctl.agent
    ctl.push_weights()
    ctl.updater.loss_iter = getattr(agent, "loss_iter", 0)
    ctl.updater.update_params(b.states, b.actions, b.rewards, b.masks, b.exps,
                              log_fn=lambda tag, v, s: agent.tb_logger.add_scalar(tag, v, s), iteration=iteration)
    agent.loss_iter = ctl.updater.loss_iter
    ctl.pull_weights()


def same_state(c1, c2, what):
    u1, u2 = c1.updater, c2.updater
    torch.cuda.synchronize()
    assert np.array_equal(u1.flat_params(), u2.flat_params()), what
    for a, b in zip(u1.engine.get_opt_state(), u2.engine.get_opt_state()):
        assert np.array_equal(a, b), what
    assert np.array_equal(u1._grad_ring.cpu().numpy(), u2._grad_ring.cpu().numpy()), what


# ---- 1. nothing changes, nothing moves ---------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_untouched_values_are_bit_identical_to_never_reading_them(model, dev):
    flat = flat_init(model, 3)
    log_live, log_fixed = [], []
    live = use_b200_update(make_agent(model, dev, flat, log_live))
    fixed = B200Update(make_agent(model, dev, flat, log_fixed, with_optimizer=False))
    for it in range(3):
        b = batch(10 + it)
        np.random.seed(it)
        live.agent.update_params(b, it)
        np.random.seed(it)
        fixed_update(fixed, b, it)
        same_state(live, fixed, it)
        assert log_live == log_fixed, it
        assert live.updater.engine.launches == fixed.updater.engine.launches, it
    sd1, sd2 = live.agent.actor_critic_net.state_dict(), fixed.agent.actor_critic_net.state_dict()
    assert all(torch.equal(sd1[k], sd2[k]) for k in sd1)                  # the weights written back too


# ---- 2. the step size ----------------------------------------------------------------------------------------------
def ipow(b, n):
    """layout.h ipow: the bias corrections' powers, by squaring."""
    r = 1.0
    while n > 0:
        if n & 1:
            r *= b
        b *= b
        n >>= 1
    return r


def adam_replay(layout, p, m, v, steps, grad, lr, b1=0.9, b2=0.999, eps=1e-5):
    """The Adam tail of k_apply / the fused tails on the host, in its fp32 operations (numpy float32 rounds each one as
    __fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn do), with the step size (float)(lr / bc1) formed in float64 from the
    double lr; bc1 and bc2 from the fp32 betas, per segment (encoder + value, land-use head, road head).  No clip, no
    decay.  Returns the parameters after the step."""
    f = np.float32
    n = layout.num_params
    g = grad[:n].astype(f)
    st = grad[layout_stat_offset(layout):]
    lu, rd = layout.slots["lu_w0"].offset, layout.slots["road_w0"].offset
    seg = np.zeros(n, np.int64)
    seg[lu:rd], seg[rd:layout.policy_end] = 1, 2
    live = [True, st[5] > 0, st[6] > 0]
    step_size, bc2s = np.zeros(3, f), np.ones(3, f)
    for s in range(3):
        stp = int(steps[1 + s]) + int(live[s])
        step_size[s] = f(lr / (1.0 - ipow(float(f(b1)), max(stp, 1))))
        bc2s[s] = f(math.sqrt(1.0 - ipow(float(f(b2)), max(stp, 1))))
    w1, w2 = f(1) - f(b1), f(1) - f(b2)
    m1 = m + w1 * (g - m)
    v1 = v * f(b2) + (w2 * g) * g
    denom = np.sqrt(v1) / bc2s[seg] + f(eps)
    out = p + (-step_size[seg]) * (m1 / denom)
    keep = ~np.array(live)[seg]
    out[keep] = p[keep]
    return out


def layout_stat_offset(layout):
    return _lib.UPB_MLP_STAT_OFFSET if layout is PL.MLP else _lib.UPB_STAT_OFFSET


LRS = [3.7e-4, 1.234567e-3, 0.0, 2.5e-4]          # not fp32 numbers (but 0); 0 moves nothing


@pytest.fixture(scope="module")
def cases(dev):
    states, actions = reproducible_states(29, 150)
    return {m: Case(dev, m, states, actions, 29) for m in ("sgnn", "mlp")}


def check_step_size(c, path, grid=0):
    eng = c.engine(clip_mode=_lib.CLIP_NEVER, grid_limit=grid)
    params = t(c.flat, c.dev).clone()
    for k, lr in enumerate(LRS):
        assert lr == 0.0 or float(np.float32(lr)) != lr
        eng.set_lr(lr)
        m, v, steps = eng.get_opt_state()
        p_old = params.cpu().numpy()
        if path == "fused":
            before = eng.launches
            g = fused_step(eng, c, params)
            assert eng.launches == before + 1
        else:
            g = nan_buffer(eng)
            eng.ppo_grad(c.blob, params, *c.step_args(), out=g)
            eng.apply(params, g)
        torch.cuda.synchronize()
        want = adam_replay(c.layout, p_old, m, v, steps, g.cpu().numpy(), lr)
        got = params.cpu().numpy()
        assert np.array_equal(got, want), (k, np.flatnonzero(got != want)[:8])
        assert np.array_equal(got, p_old) == (lr == 0.0), k
        assert eng.get_opt_state()[2][0] == k + 1                      # lr = 0 still counts the step


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_set_lr_step_size_on_upb_apply(model, cases):
    check_step_size(cases[model], "apply")


@pytest.mark.parametrize("grid", XP.SGNN_GRIDS)
def test_set_lr_step_size_on_the_sgnn_fused_step(grid, cases):
    check_step_size(cases["sgnn"], "fused", grid)


@pytest.mark.parametrize("grid", XP.MLP_GRIDS)
def test_set_lr_step_size_on_the_mlp_fused_step(grid, cases):
    check_step_size(cases["mlp"], "fused", grid)


def test_set_lr_and_set_loss_coefs_refuse_invalid_values(cases):
    eng = cases["sgnn"].engine()
    L = _lib.lib()
    for bad in (-1e-4, float("nan"), float("inf")):
        assert L.upb_set_lr(eng._ctx, bad) == -1                          # UPB_ERR_ARG
    for bad in (float("nan"), float("inf"), float("-inf")):
        assert L.upb_set_loss_coefs(eng._ctx, bad, 0.01) == -1 and L.upb_set_loss_coefs(eng._ctx, 0.5, bad) == -1
    assert L.upb_set_lr(eng._ctx, 0.0) == 0 and L.upb_set_loss_coefs(eng._ctx, -1.0, -0.5) == 0


def test_read_losses_use_the_coefficients_current_at_the_read(cases):
    c = cases["sgnn"]
    eng = c.engine(clip_mode=_lib.CLIP_NEVER)
    g = eng.ppo_grad(c.blob, t(c.flat, c.dev).clone(), *c.step_args())
    st = g[_lib.UPB_STAT_OFFSET:].cpu().numpy().astype(np.float32)
    for cv, ce in [(0.5, 0.01), (1.0, 0.25), (-2.0, 0.0)]:
        eng.set_loss_coefs(cv, ce)
        loss, vl, sl, el = eng.read_losses(g)
        assert vl == np.float32(st[0] / st[3]) and el == np.float32(st[2] / st[4])
        assert loss == np.float32(np.float32(sl + np.float32(cv) * vl) + np.float32(ce) * el)


# ---- 3. trajectories against the oracle ports --------------------------------------------------------------------------
def port_iteration(port, mod, b, gamma, tau, epochs, B):
    """The reference's update_params / update_policy on an oracle port (CPU), np.random drawn as PPOUpdater draws it."""
    b_all = mod.stack_states(b.states)
    act = torch.tensor(b.actions)
    with torch.no_grad():
        values = mod.value(port.P, b_all).reshape(-1, 1)
    adv, ret = TP.estimate_advantages(torch.tensor(b.rewards), torch.tensor(b.masks), values, gamma, tau)
    with torch.no_grad():
        fixed, _ = mod.log_prob_entropy(port.P, b_all, act)
    exps_t = torch.tensor(b.exps)
    order, losses = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(T // B):
            idx = order[i * B:(i + 1) * B]
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(port.step(mod.stack_states([b.states[j] for j in idx]), act[idx], adv[idx], ret[idx],
                                    fixed[idx], ind))
    return np.array(losses)


# per iteration: the agent attributes set before it (the same on the port); lr comes from the scheduler
CHANGES = [{}, dict(entropy_coef=0.05, clip_epsilon=0.1, mini_batch_size=12, opt_num_epochs=2),
           dict(entropy_coef=0.0, clip_epsilon=0.3, value_pred_coef=1.0)]


@pytest.mark.parametrize("sched", ["lambda", "plateau"])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_scheduled_trajectory_matches_the_oracle_port(model, sched, dev):
    flat = flat_init(model, 7)
    logged = []
    ag = make_agent(model, dev, flat, logged)
    ctl = use_b200_update(ag)
    port = TP.PortAgent(flat) if model == "sgnn" else MP.MLPPortAgent(flat)
    mod = TP if model == "sgnn" else MP

    def scheduler(opt):
        if sched == "lambda":                     # CleanRL's anneal_lr over the three iterations
            return torch.optim.lr_scheduler.LambdaLR(opt, lambda it: 1.0 - it / 3.0)
        return torch.optim.lr_scheduler.ReduceLROnPlateau(opt, factor=0.2, patience=0)

    scheds = [scheduler(ag.optimizer), scheduler(port.opt)]
    epochs, B = ag.cfg.num_optim_epoch, ag.cfg.mini_batch_size
    for it, change in enumerate(CHANGES):
        for k, v in change.items():
            setattr(ag, k, v)
            if k in ("entropy_coef", "clip_epsilon", "value_pred_coef"):
                setattr(port, k, v)
        epochs, B = change.get("opt_num_epochs", epochs), change.get("mini_batch_size", B)
        b = batch(20 + it)
        start = len(logged)
        np.random.seed(it)
        ag.update_params(b, it)
        np.random.seed(it)
        want = port_iteration(port, mod, b, ag.gamma, ag.tau, epochs, B)
        got = update_losses(logged[start:])
        assert got.shape == want.shape == (epochs * (T // B), 4), it
        assert np.allclose(got, want, rtol=2e-4, atol=2e-5), (it, np.abs(got - want).max())
        assert rel(ctl.updater.flat_params(), port.flat()) < 2e-5, it
        assert ctl.updater.engine.lr == port.opt.param_groups[0]["lr"] == ag.optimizer.param_groups[0]["lr"], it
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")       # the agent's optimizer never steps: the H100 path trains
            for s in scheds:
                if sched == "lambda":
                    s.step()
                else:
                    s.step([1.0, 2.0, 3.0][it])   # no improvement after the first iteration: lr * 0.2 each time
    assert ctl.updater.engine.lr < SHIPPED_CFG["lr"] * 0.5


# ---- 4. together with the other options --------------------------------------------------------------------------------
OPTIONS = {"max_grad_norm": dict(max_grad_norm=0.5), "skip_nonfinite": dict(skip_nonfinite=True),
           "target_kl": dict(target_kl=0.002), "kl_penalty": dict(kl_coef=0.2, kl_target=0.01)}
# fp32 numbers, so that a controller built with them holds the very values the live change passes
NEW = dict(lr=2.0 ** -11, weightdecay=2.0 ** -7, entropy_coef=2.0 ** -5, value_pred_coef=0.75, clip_epsilon=0.25,
           gamma=0.5, num_optim_epoch=2, mini_batch_size=12)
ATTR = dict(entropy_coef="entropy_coef", value_pred_coef="value_pred_coef", clip_epsilon="clip_epsilon", gamma="gamma",
            num_optim_epoch="opt_num_epochs", mini_batch_size="mini_batch_size")


@pytest.mark.parametrize("zero_lr", [False, True])
@pytest.mark.parametrize("option", sorted(OPTIONS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_live_changes_work_with_the_other_options(model, option, zero_lr, dev):
    kw = dict(OPTIONS[option], clip_mode=_lib.CLIP_NEVER)
    new = dict(NEW, lr=0.0 if zero_lr else NEW["lr"])
    flat = flat_init(model, 11)
    logged = []
    ag = make_agent(model, dev, flat, logged)
    ctl = use_b200_update(ag, **kw)
    np.random.seed(0)
    ag.update_params(batch(30), 0)
    # the changes, through the param group (lr, weight_decay) and the agent's attributes
    for g in ag.optimizer.param_groups:
        g["lr"], g["weight_decay"] = new["lr"], new["weightdecay"]
    for k, a in ATTR.items():
        setattr(ag, a, new[k])
    # the same state, in a controller built with the new values
    log2 = []
    ag2 = make_agent(model, dev, ctl.updater.flat_params(), log2, **new)
    ctl2 = use_b200_update(ag2, **kw)
    m, v, steps = ctl.updater.engine.get_opt_state()
    ctl2.updater.engine.set_opt_state(m, v, steps)
    if ctl.updater.kl_coef is not None:
        ctl2.updater.set_kl_coef(ctl.updater.kl_coef)
    ag2.loss_iter = ag.loss_iter
    p_before = ctl.updater.flat_params()
    b = batch(31)
    start = len(logged)
    np.random.seed(1)
    ag.update_params(b, 1)
    np.random.seed(1)
    ag2.update_params(b, 1)
    same_state(ctl, ctl2, option)
    assert logged[start:] == log2, option
    e = ctl.updater.engine
    assert (e.lr, e.weight_decay, e.clip_epsilon, ctl.updater.opt_num_epochs) == (new["lr"], new["weightdecay"], 0.25, 2)
    steps_after = e.get_opt_state()[2]
    assert steps_after[0] > steps[0]
    if zero_lr:
        assert np.array_equal(ctl.updater.flat_params(), p_before)     # lr = 0: counters advance, nothing moves
    else:
        assert not np.array_equal(ctl.updater.flat_params(), p_before)
