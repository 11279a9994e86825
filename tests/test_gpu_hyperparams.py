"""GPU (H100): both models' training paths at clip, loss-coefficient and Adam settings away from the shipped ones (the
`hp` row of cross_path.SETTINGS), and the checks of the clip range and the betas alone.

Each setting reaches the device through its own path: clip range, value_pred_coef and entropy_coef through StepArgs into
softmax_seeds (and the SGNN's value-backward seed); lr, betas and eps through StepArgs into the fused tails
and through ApplyArgs into k_apply; the coefficients again in read_losses.  References: golden vectors recorded by the
unmodified reference at other settings (tests/golden/*_hp*.npz), the two-call path against the fused step at
the fused-tail grid sizes, the float64 Adam and torch.optim.Adam at other betas, and torch.clamp's clip bounds read back
exactly from statistics slot 1."""
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
import cross_path as XP
from harness import Case, dev, heads, load, rel, reproducible_states, t
from oracle import sgnn_numpy as ON

pytestmark = pytest.mark.gpu

EPSILONS = [k / 100 for k in range(1, 100)]


# ---- golden trajectories of the reference ----------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("name", ["small_mixed_hp", "small_mixed_hp0", "mlp_small_hp"])
def test_steps_match_reference_golden_at_other_settings(name, fused, golden_dir, dev):
    """cross_path.check_golden_trajectory: values, log-probs and three steps (the first clips), both models."""
    XP.check_golden_trajectory(load(golden_dir, name), name, fused, dev)


def test_update_params_matches_reference_at_other_settings(golden_dir, dev):
    """The reference's whole update_params iteration at gamma 1, tau 0, eps 0.09, c_v 0.25, c_e 0.02 and lr 3e-4
    (update_small_hp) through PPOUpdater."""
    XP.check_update_params(load(golden_dir, "update_small_hp"), dev)


def test_use_b200_update_honours_the_cfg_settings(golden_dir, dev):
    """use_b200_update on a reference-shaped agent whose cfg carries update_small_hp's settings."""
    XP.check_use_b200_update(load(golden_dir, "update_small_hp"), dev)


# ---- fused tail vs two-call path at other lr, betas and eps ------------------------------------------------------------
@pytest.fixture(scope="module")
def sgnn_batch(dev):
    return XP.hlg_case(dev, 19)


@pytest.fixture(scope="module")
def mlp_case(dev):
    states, actions = reproducible_states(29, 150)
    stage = np.array([int(s[8].argmax()) for s in states])
    return Case(dev, "mlp", states, actions, 29, zero_exps=(int(np.flatnonzero(stage == 0)[1]),))


@pytest.mark.parametrize("grid", XP.SGNN_GRIDS)
def test_sgnn_fused_step_matches_two_call_path_at_other_settings(grid, sgnn_batch, dev):
    """StepArgs (fused tail) and ApplyArgs (k_apply) must carry the same lr, betas, eps and loss settings
    (cross_path.check_sgnn_fused_against_two_call at the `hp` row)."""
    XP.check_sgnn_fused_against_two_call(sgnn_batch, "hp", grid)


@pytest.mark.parametrize("grid", XP.MLP_GRIDS)
def test_mlp_fused_step_is_bit_identical_to_two_call_path_at_other_settings(grid, mlp_case, dev):
    """The rl-mlp fused tail and k_apply stay bit-identical at the `hp` row (cross_path.check_mlp_fused_bit_identical)."""
    XP.check_mlp_fused_bit_identical(mlp_case, "hp", grid)


# ---- betas -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_betas_against_float64_adam_and_torch_adam(model, sgnn_batch, mlp_case, dev):
    """Engine(betas=(0.8, 0.99)): three fused steps, each against sgnn_numpy.adam_step(b1, b2) and torch.optim.Adam(betas)
    applied to the step's own gradient buffer (no clipping; both policy heads live on every step)."""
    b1, b2, lr, eps = 0.8, 0.99, 1e-3, 1e-5
    c = sgnn_batch if model == "sgnn" else mlp_case
    eng = c.engine(clip_mode=_lib.CLIP_NEVER, lr=lr, betas=(b1, b2), eps=eps)
    n = eng.num_params
    params = t(c.flat, dev).clone()
    ref = torch.tensor(c.flat, dtype=torch.float32, requires_grad=True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps)
    f64, m, v, tt = c.flat.astype(np.float64), np.zeros(n), np.zeros(n), np.zeros(n)
    live = np.ones(n, bool)
    for step in range(3):
        p_old = params.cpu().numpy()
        grad = eng.ppo_step(c.blob, params, *c.step_args())
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


# ---- the clip range, read back exactly -------------------------------------------------------------------------------
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
    layout = PL.MLP if model == "mlp" else PL.SGNN
    params = t(PL.MLP.default_init(31) if model == "mlp" else PL.default_init(31), dev)
    s = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
    head = heads(layout)[0]
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
