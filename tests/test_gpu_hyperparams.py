"""GPU (H100): both models' training paths at clip, loss-coefficient and Adam settings away from the shipped ones.

Each setting reaches the device through its own path: clip range, value_pred_coef and entropy_coef through StepArgs into
softmax_seeds (and the SGNN's value-backward seed); lr, betas and eps through StepArgs into the fused tails and through
ApplyArgs into k_apply; the coefficients again in read_losses.  References: golden vectors recorded by the unmodified
reference at other settings (tests/golden/*_hp*.npz), the two-call path against the fused step at the fused-tail grid
sizes, the float64 Adam and torch.optim.Adam at other betas, and torch.clamp's clip bounds read back exactly from
statistics slot 1."""
import os
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine, clip_range
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from oracle import sgnn_numpy as ON
from test_gpu_mlp_step import HEADS as MLP_HEADS, Case, assert_same_state, fused_step, reproducible_states, two_call_step
from test_gpu_parity import per_tensor_rel, rel, t
from test_mlp import per_tensor_rel as mlp_per_tensor_rel

pytestmark = pytest.mark.gpu

TOL = 1e-4
SGNN_HEADS = {0: slice(PL.SLOTS["lu_w0"].offset, PL.SLOTS["road_w0"].offset),
              1: slice(PL.SLOTS["road_w0"].offset, PL.POLICY_END)}
VALUE_HEAD = slice(PL.POLICY_END, PL.NUM_PARAMS)
EPSILONS = [k / 100 for k in range(1, 100)]
# lr, betas, eps and the loss settings of the fused-against-two-call tests: none of them the shipped value
ODD = dict(lr=1e-3, betas=(0.8, 0.99), eps=1e-7, clip_epsilon=0.18, value_pred_coef=1.0, entropy_coef=0.05)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need an H100"
    return torch.device("cuda", 0)


def load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def settings(z):
    return {k: float(z[k]) for k in ("clip_epsilon", "value_pred_coef", "entropy_coef", "lr", "eps")}


def step_bar(h, bar):
    """A parameter-trajectory bar set at lr 4e-4, scaled to the fixture's lr (test_hyperparams.step_bar)."""
    return bar * max(1.0, h["lr"] / 4e-4)


# ---- golden trajectories of the reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("name", ["small_mixed_hp", "small_mixed_hp0", "mlp_small_hp"])
def test_steps_match_reference_golden_at_other_settings(name, fused, golden_dir, dev):
    """Values and log-probs, then three steps: the first clips (two-call path on both), the next two run through
    upb_apply or the fused tail.  Losses from read_losses, every gradient tensor and the parameters after each step, with
    test_gpu_parity's bars (the parameter bar scaled to the lr)."""
    z = load(golden_dir, name)
    h = settings(z)
    mlp = name.startswith("mlp")
    layout = PL.MLP if mlp else PL.SGNN
    ptr = mlp_per_tensor_rel if mlp else per_tensor_rel
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE, model="mlp" if mlp else "sgnn", **h)
    assert eng.clip_range == (float(np.float32(1.0 - h["clip_epsilon"])), float(np.float32(1.0 + h["clip_epsilon"])))
    params = t(z["params"], dev).clone()
    value, logp, _ = eng.forward(blob, params, t(z["actions"], dev))
    assert rel(value.cpu().numpy(), z["values"].ravel()) < TOL
    assert rel(logp.cpu().numpy(), z["log_probs"].ravel()) < TOL
    n_ind = int((z["exps"] != 0).sum())
    args = tuple(t(z[k], dev) for k in ("actions", "advantages", "returns", "fixed_log_probs", "exps"))
    for k in range(3):
        before = eng.launches
        if fused:
            grad = eng.ppo_step(blob, params, *args, 1.0 / B, 1.0 / n_ind)
        else:
            grad = eng.ppo_grad(blob, params, *args, 1.0 / B, 1.0 / n_ind)
            eng.apply(params, grad)
        torch.cuda.synchronize()
        if fused:
            assert (eng.launches - before == 1) == (k > 0), k
        losses = eng.read_losses(grad)
        assert np.allclose(losses, z["losses"][k], rtol=1e-4, atol=1e-5), (k, losses, z["losses"][k])
        worst, where = ptr(grad.cpu().numpy()[:layout.num_params], z["grads"][k])
        assert worst < TOL, (k, worst, where)
        assert rel(params.cpu().numpy(), z["params_after"][k]) < step_bar(h, 1e-5), k
    if name == "small_mixed_hp0":
        # value_pred_coef = 0: a zero value-head gradient, not an absent one -- the head keeps its weights and zero
        # moments while its step counter (shared with the encoder) advances, as the reference's Adam counts its steps
        p = params.cpu().numpy()
        assert not grad.cpu().numpy()[VALUE_HEAD].any()
        assert np.array_equal(p[VALUE_HEAD], z["params"][VALUE_HEAD])
        m, v, steps = eng.get_opt_state()
        assert not m[VALUE_HEAD].any() and not v[VALUE_HEAD].any()
        assert steps.tolist() == [3, 3, 3, 3] and z["value_adam_steps"].tolist() == [3] * len(z["value_adam_steps"])


def update_losses(logged):
    return np.array([[v for tag, v, s in logged if tag == k] for k in
                     ("loss/loss", "loss/value_loss", "loss/surr_loss", "loss/entropy_loss")]).T


def test_update_params_matches_reference_at_other_settings(golden_dir, dev):
    """The reference's whole update_params iteration at gamma 1, tau 0, eps 0.09, c_v 0.25, c_e 0.02 and lr 3e-4
    (update_small_hp) through PPOUpdater, with the update_small test's tolerances."""
    from drl_urban_planning_b200.ppo import PPOUpdater
    z = load(golden_dir, "update_small_hp")
    h = settings(z)
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    up = PPOUpdater(z["params"], int(z["n_cap"]), int(z["e_cap"]), dev, gamma=float(z["gamma"]), tau=float(z["tau"]),
                    opt_num_epochs=epochs, mini_batch_size=B, clip_mode=_lib.CLIP_REFERENCE, **h)
    logged = []
    np.random.seed(np_seed)
    out = up.update_params(expand_states(z), z["actions"], z["rewards"], z["masks"], z["exps"],
                           log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    got = update_losses(logged)
    assert got.shape == z["losses"].shape == (epochs * (T // B), 4)
    assert np.allclose(got, z["losses"], rtol=2e-4, atol=2e-5), np.abs(got - z["losses"]).max()
    totals = np.array([out["total_loss"], out["total_value_loss"], out["total_surr_loss"], out["total_entropy_loss"]])
    assert np.allclose(totals, z["totals"], rtol=2e-4, atol=2e-5)
    assert rel(up.flat_params(), z["params_after"]) < 2e-5


def test_use_b200_update_honours_the_cfg_settings(golden_dir, dev):
    """use_b200_update on a reference-shaped agent whose cfg carries update_small_hp's settings reproduces the
    reference's update_params with that cfg, and writes the parameters back into the modules."""
    from drl_urban_planning_b200.agent import use_b200_update
    from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
    from test_model_dropin import Agent, Cfg
    z = load(golden_dir, "update_small_hp")
    h = settings(z)
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    cfg = Cfg(int(z["n_cap"]), int(z["e_cap"]))
    cfg.lr, cfg.eps, cfg.clip_epsilon = h["lr"], h["eps"], h["clip_epsilon"]
    cfg.value_pred_coef, cfg.entropy_coef = h["value_pred_coef"], h["entropy_coef"]
    cfg.gamma, cfg.tau = float(z["gamma"]), float(z["tau"])
    cfg.num_optim_epoch, cfg.mini_batch_size = epochs, B
    cfg.agent_specs, cfg.agent = {}, "rl-sgnn"
    ag = Agent()
    ag.cfg, ag.device, ag.loss_iter = cfg, dev, 0
    logged = []
    ag.tb_logger = types.SimpleNamespace(add_scalar=lambda tag, v, s: logged.append((tag, v, s)))
    torch.manual_seed(0)
    p, v = create_sgnn_model(cfg, ag)
    ag.policy_net, ag.value_net, ag.actor_critic_net = p, v, ActorCritic(p, v)
    ag.actor_critic_net.load_flat_parameters(z["params"])
    ctl = use_b200_update(ag)
    assert ctl.updater.engine.clip_range == clip_range(h["clip_epsilon"])
    batch = types.SimpleNamespace(states=expand_states(z), actions=z["actions"], rewards=z["rewards"], masks=z["masks"],
                                  exps=z["exps"])
    np.random.seed(np_seed)
    ag.update_params(batch, 0)
    assert np.allclose(update_losses(logged), z["losses"], rtol=2e-4, atol=2e-5)
    assert rel(ctl.updater.flat_params(), z["params_after"]) < 2e-5
    assert rel(ag.actor_critic_net.flat_parameters(), z["params_after"]) < 2e-5


# ---- fused tail vs two-call path at other lr, betas and eps ------------------------------------------------------------
@pytest.fixture(scope="module")
def sgnn_batch(dev):
    """140 hlg-sized graphs of both stages (one in three a road graph): more than the 132 CTAs of a full grid."""
    count = 140
    states, actions = synth.make_states(19, "hlg", count, stages=[int(i % 3 == 1) for i in range(count)])
    adv, ret, exps = synth.make_ppo_targets(19, count)
    exps[7] = 0.0
    fixed = np.random.default_rng(19).normal(-3.0, 0.3, size=(count, 1)).astype(np.float32)
    blob = pack_states(states).to(dev)
    return types.SimpleNamespace(states=states, count=count, blob=blob, exps=exps, actions=actions, adv=adv, ret=ret,
                                 fixed=fixed, args=tuple(t(x, dev) for x in (actions, adv, ret, fixed, exps)),
                                 flat=PL.default_init(19))


@pytest.mark.parametrize("grid", [1, 2, 7, 113, 114, 115, 132])
def test_sgnn_fused_step_matches_two_call_path_at_other_settings(grid, sgnn_batch, dev):
    """StepArgs (fused tail) and ApplyArgs (k_apply) must carry the same lr, betas and eps: 4 steps (the first clips),
    the tolerances of test_fused_step_matches_two_call_path, and far from an engine at the shipped settings."""
    b = sgnn_batch
    n_ind = int((b.exps != 0).sum())
    e1 = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid, **ODD)
    e2 = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid, **ODD)
    e0 = Engine(dev, b.blob.n_cap, b.blob.e_cap, grid_limit=grid)
    p1, p2, p0 = (t(b.flat, dev).clone() for _ in range(3))
    for step in range(4):
        g1 = e1.ppo_grad(b.blob, p1, *b.args, 1.0 / b.count, 1.0 / n_ind)
        e1.apply(p1, g1)
        before = e2.launches
        g2 = e2.ppo_step(b.blob, p2, *b.args, 1.0 / b.count, 1.0 / n_ind)
        e0.ppo_step(b.blob, p0, *b.args, 1.0 / b.count, 1.0 / n_ind)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (step > 0), step
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (step, worst, where)
        assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
        # the two paths sum the gradient columns in different orders; Adam turns that last-bit noise into parameter
        # differences that grow with lr (the weight-decay test's 1e-6 is at 4e-4)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < step_bar(ODD, 1e-6), step
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    assert s1.tolist() == s2.tolist() == [4, 4, 4, 4]
    assert rel(m2, m1) < 1e-5 and rel(v2, v1) < 1e-5
    assert rel(p2.cpu().numpy(), p0.cpu().numpy()) > 1e-3


@pytest.fixture(scope="module")
def mlp_case(dev):
    states, actions = reproducible_states(29, 150)
    stage = np.array([int(s[8].argmax()) for s in states])
    return Case(dev, states, actions, 29, zero_exps=(int(np.flatnonzero(stage == 0)[1]),))


@pytest.mark.parametrize("grid", [1, 2, 80, 81, 82, 132])
def test_mlp_fused_step_is_bit_identical_to_two_call_path_at_other_settings(grid, mlp_case, dev):
    """On reproducible batches the rl-mlp fused tail and k_apply stay bit-identical at other lr, betas and eps:
    parameters, gradient buffer, moments and step counters."""
    c = mlp_case
    lu, allg = np.flatnonzero(c.stage == 0), np.arange(c.count)
    e1 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid, **ODD)
    e2 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid, **ODD)
    e0 = Engine(dev, c.blob.n_cap, c.blob.e_cap, model="mlp", grid_limit=grid)
    p1, p2, p0 = (t(c.flat, dev).clone() for _ in range(3))
    for step, sel in enumerate([allg, allg, lu, allg]):
        g1 = two_call_step(e1, c, p1, sel)
        before = e2.launches
        g2 = fused_step(e2, c, p2, sel)
        fused_step(e0, c, p0, sel)
        assert e2.launches - before == (3 if step == 0 else 1), step
        steps = assert_same_state(e1, p1, g1, e2, p2, g2, (grid, step))
    assert steps.tolist() == [4, 4, 4, 3]
    assert rel(p2.cpu().numpy(), p0.cpu().numpy()) > 1e-3


# ---- betas -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_betas_against_float64_adam_and_torch_adam(model, sgnn_batch, mlp_case, dev):
    """Engine(betas=(0.8, 0.99)): three fused steps, each against sgnn_numpy.adam_step(b1, b2) and torch.optim.Adam(betas)
    applied to the step's own gradient buffer (no clipping; both policy heads live on every step)."""
    b1, b2, lr, eps = 0.8, 0.99, 1e-3, 1e-5
    if model == "sgnn":
        blob, flat, args = sgnn_batch.blob, sgnn_batch.flat, sgnn_batch.args
        count, n_ind = sgnn_batch.count, int((sgnn_batch.exps != 0).sum())
    else:
        blob, flat, args = mlp_case.blob, mlp_case.flat, mlp_case.dev_args
        count, n_ind = mlp_case.count, int((mlp_case.exps != 0).sum())
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model, clip_mode=_lib.CLIP_NEVER, lr=lr, betas=(b1, b2), eps=eps)
    n = eng.num_params
    params = t(flat, dev).clone()
    ref = torch.tensor(flat, dtype=torch.float32, requires_grad=True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps)
    f64, m, v, tt = flat.astype(np.float64), np.zeros(n), np.zeros(n), np.zeros(n)
    live = np.ones(n, bool)
    for step in range(3):
        p_old = params.cpu().numpy()
        grad = eng.ppo_step(blob, params, *args, 1.0 / count, 1.0 / n_ind)
        torch.cuda.synchronize()
        g = grad.cpu().numpy()[:n]
        ref.grad = torch.tensor(g)
        opt.step()
        # the float64 Adam steps from the device's parameters, so each step is judged on its own
        f64, m, v, tt = ON.adam_step(p_old, m, v, tt, g, live, lr=lr, b1=b1, b2=b2, eps=eps)
        p = params.cpu().numpy()
        assert rel(p, f64) < 1e-6, step
        assert rel(p - p_old, f64 - p_old) < 1e-3, step                    # the step itself, not only the parameter
        assert rel(p, ref.detach().numpy()) < 1e-6, step
        _, _, steps = eng.get_opt_state()
        assert steps.tolist()[0] == step + 1
    mm, vv, _ = eng.get_opt_state()
    assert rel(mm, m) < 1e-5 and rel(vv, v) < 1e-5
    st = opt.state[ref]
    assert rel(mm, st["exp_avg"].numpy()) < 1e-5 and rel(vv, st["exp_avg_sq"].numpy()) < 1e-5


# ---- the clip range, read back exactly ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def one_graph(dev):
    states, actions = synth.make_states(31, "small", 1, stages=[0])
    blob = pack_states(states).to(dev)
    return types.SimpleNamespace(blob=blob, actions=t(actions, dev))


def launch_one(eng, g, params, logp, adv, dlp, fused):
    """One graph in ind with advantage `adv` and fixed log-prob logp - dlp, on ppo_grad or on a fused ppo_step (from a
    copy of params); the gradient / statistics buffer."""
    dev = eng.device
    fixed = torch.tensor([[np.float32(logp - dlp)]], device=dev)
    one = torch.ones(1, 1, device=dev)
    a = (g.actions, one * adv, torch.zeros(1, 1, device=dev), fixed, one)
    if fused:
        before = eng.launches
        grad = eng.ppo_step(g.blob, params.clone(), *a, 1.0, 1.0)
        assert eng.launches - before == 1
    else:
        grad = eng.ppo_grad(g.blob, params, *a, 1.0, 1.0)
    torch.cuda.synchronize()
    return grad.cpu().numpy()


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_clip_range_is_torch_clamps(model, fused, one_graph, dev):
    """surr = -min(r A, clamp(r, lo, hi) A) of one graph far outside the range: A = +1, r = e^8 gives statistics slot 1 =
    -hi, and A = -1, r = e^-8 gives lo -- both exactly np.float32(1 +/- eps), torch.clamp's bounds, for every
    eps = k/100.  Slot 9 counts the graph as clipped.  With entropy_coef = 0 the A = +1 case leaves the land-use head
    an exactly zero gradient (the surrogate passes none through the clamped branch)."""
    g = one_graph
    flat = PL.MLP.default_init(31) if model == "mlp" else PL.default_init(31)
    params = t(flat, dev)
    s = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    head = (MLP_HEADS if model == "mlp" else SGNN_HEADS)[0]
    logp = None
    wrong = []
    for eps in EPSILONS:
        lo, hi = np.float32(1.0 - eps), np.float32(1.0 + eps)
        kw = dict(model=model, clip_mode=_lib.CLIP_NEVER, clip_epsilon=eps, diagnostics=True)
        eng = Engine(dev, g.blob.n_cap, g.blob.e_cap, **kw)
        if logp is None:
            logp = float(eng.forward(g.blob, params, g.actions)[1].cpu().numpy()[0])
        up = launch_one(eng, g, params, logp, 1.0, 8.0, fused)
        down = launch_one(eng, g, params, logp, -1.0, -8.0, fused)
        assert up[s + 4] == down[s + 4] == 1 and up[s + 9] == down[s + 9] == 1, eps
        if up[s + 1] != -hi or down[s + 1] != lo:
            wrong.append((eps, float(up[s + 1]), float(-hi), float(down[s + 1]), float(lo)))
        e0 = Engine(dev, g.blob.n_cap, g.blob.e_cap, entropy_coef=0.0, **kw)
        g0 = launch_one(e0, g, params, logp, 1.0, 8.0, fused)
        assert g0[s + 1] == -hi and not g0[head].any(), eps
        assert np.abs(up[head]).max() > 0, eps                    # the entropy term alone moves the head
    assert not wrong, wrong


def test_set_clip_range_rejects_invalid_ranges(dev):
    """The C entry point refuses non-finite bounds and lo > hi, and accepts a point range."""
    eng = Engine(dev, 64, 64)
    L = _lib.lib()
    for lo, hi in ((float("nan"), 1.2), (0.8, float("inf")), (-float("inf"), 1.2), (1.2, 0.8)):
        assert L.upb_set_clip_range(eng._ctx, lo, hi) == -1, (lo, hi)                  # UPB_ERR_ARG
        assert b"set_clip_range" in L.upb_last_error()
    assert L.upb_set_clip_range(eng._ctx, 1.0, 1.0) == 0 and L.upb_set_clip_range(eng._ctx, 0.8, 1.2) == 0
