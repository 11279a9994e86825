"""The checks that hold every implementation of the update together, written once and run at each optimiser setting.

A setting is a set of `Engine` keyword arguments (SETTINGS; a golden fixture carries its own, read by `settings`).  The
test modules of each feature call these checks with their setting, so a new setting needs only a table entry and the
test entry points that name it:
  * CPU: the float64 oracle, the torch port and the rl-mlp port against the golden vectors the unmodified reference
    recorded at that setting, and the fixture's distance from its shipped-settings namesake;
  * GPU: the golden trajectories (two-call and fused), PPOUpdater and use_b200_update against the reference, and the
    fused step against ppo_grad + apply at the grid sizes where the fused tails own their gradient slices differently
    (the rl-mlp bit for bit)."""
import math
import types

import numpy as np
import torch

import decay_oracle as DO
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine, clip_range
from drl_urban_planning_b200.packing import pack_states
from fixtures_io import expand_states
from harness import (Case, assert_same_state, fused_step, heads, load, per_tensor_rel, rel, sgnn_agent, t,
                     two_call_step, update_losses)
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP

# Engine keyword arguments of the optimiser settings the fused-against-two-call checks run at
SETTINGS = {
    "shipped": {},
    "wd": dict(weight_decay=1e-2),
    "hp": dict(lr=1e-3, betas=(0.8, 0.99), eps=1e-7, clip_epsilon=0.18, value_pred_coef=1.0, entropy_coef=0.05),
}
# grid sizes that change how the fused tails own their gradient slices: one CTA owning every slice, several per CTA,
# one each with idle CTAs, and the full H100 grid
SGNN_GRIDS = [1, 2, 3, 7, 57, 113, 114, 115, 132]             # 114 slices of 128 columns (sgnn_kernel.cuh)
M_NSLICE = 81              # csrc/mlp_kernel.cuh (static_assert): 10,304 columns in slices of 128, the last one half
MLP_GRIDS = [1, 2, 3, 7, 8, M_NSLICE - 1, M_NSLICE, M_NSLICE + 1, 132]
TOL = 1e-4
VALUE_HEAD = slice(PL.POLICY_END, PL.NUM_PARAMS)


def settings(z):
    """The Engine keyword arguments a golden fixture was recorded at (the shipped value where it has no key)."""
    return {k: float(z[k]) for k in ("clip_epsilon", "value_pred_coef", "entropy_coef", "lr", "eps", "weight_decay")
            if k in z.files}


def loss_kw(h):
    return {k: h[k] for k in ("clip_epsilon", "value_pred_coef", "entropy_coef") if k in h}


def adam_kw(h):
    return {k: h[k] for k in ("lr", "eps") if k in h}


def step_bar(h, bar):
    """A parameter-trajectory bar set at lr 4e-4, scaled to the setting's lr: gradients that differ in the last bits
    (oracle against reference, or two summation orders) become parameter differences that Adam scales with lr."""
    return bar * max(1.0, h.get("lr", 4e-4) / 4e-4)


# ---- CPU: the oracles against the reference's golden vectors ---------------------------------------------------------
def check_away_from_shipped(golden_dir, name, shipped_name):
    """The fixture starts where its shipped-settings namesake does and ends far outside the parity bars (5e-6 on the
    CPU, 2e-5 on the GPU), so a path that ran at the shipped settings could not match it."""
    z, base = load(golden_dir, name), load(golden_dir, shipped_name)
    h = settings(z)
    if "weight_decay" in h:
        assert h["weight_decay"] > 0.0
    else:
        assert (h["clip_epsilon"], h["value_pred_coef"], h["entropy_coef"]) != (0.2, 0.5, 0.01)
    assert np.array_equal(z["params"], base["params"]) and np.array_equal(z["actions"], base["actions"])
    a, b = z["params_after"], base["params_after"]
    assert a.shape == b.shape
    assert rel(a.reshape(-1, a.shape[-1])[-1], b.reshape(-1, b.shape[-1])[-1]) > 10 * 1e-4
    if loss_kw(h) and not name.startswith("update"):
        assert not np.allclose(z["losses"][0], base["losses"][0], rtol=1e-3, atol=1e-4)


def port_step_args(z, stack):
    b = stack(expand_states(z))
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    return (b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
            torch.tensor(z["fixed_log_probs"]), ind)


def check_numpy_oracle_steps(z):
    """The float64 oracle with the fixture's coefficients, clip range, Adam lr / eps and decay (on the live entries
    only): losses, every gradient and the three-step trajectory (first step clipped); the parameters of an absent head
    never move.  Away from the shipped loss settings, the oracle at the shipped ones misses the same fixture."""
    h = settings(z)
    states = expand_states(z)
    live = ON.live_mask(states)
    args = (states, z["actions"], z["advantages"], z["returns"], z["fixed_log_probs"], z["exps"])
    flat = z["params"].astype(np.float64)
    m = v = tt = np.zeros(PL.NUM_PARAMS)
    for k in range(3):
        r = ON.ppo_minibatch(flat, *args, **loss_kw(h))
        got = [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]]
        assert np.allclose(got, z["losses"][k], rtol=2e-5, atol=2e-6), (k, got, z["losses"][k])
        assert rel(r["grad"], z["grads"][k]) < 1e-4, k
        g = ON.clip_groups(r["grad"]) if k == 0 else r["grad"]
        flat, m, v, tt = DO.adam_step(flat, m, v, tt, g, live, h.get("weight_decay", 0.0), **adam_kw(h))
        assert rel(flat, z["params_after"][k]) < step_bar(h, 5e-6), k
    assert np.array_equal(flat[~live].astype(np.float32), z["params"][~live])
    if loss_kw(h):
        r0 = ON.ppo_minibatch(z["params"].astype(np.float64), *args)
        assert rel(r0["grad"], z["grads"][0]) > 1e-2


def check_torch_port_steps(z):
    """The torch port: three steps, the first one clipped by the reference's clip_policy_grad, then torch.optim.Adam
    with the fixture's lr, eps and (coupled) decay."""
    h = settings(z)
    agent = DO.port_agent(z["params"], h.get("weight_decay", 0.0), **adam_kw(h), **loss_kw(h))
    args = port_step_args(z, TP.stack_states)
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < step_bar(h, 5e-6), k


def check_mlp_port(z):
    """The rl-mlp port at the fixture's settings: losses and parameters of three steps, the first step's gradient,
    and the port at the shipped settings missing the first step."""
    h = settings(z)
    args = port_step_args(z, MP.stack_states)
    agent = DO.mlp_port_agent(z["params"], h.get("weight_decay", 0.0), **adam_kw(h), **loss_kw(h))
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < step_bar(h, 5e-6), k
    first = DO.mlp_port_agent(z["params"], h.get("weight_decay", 0.0), **adam_kw(h), **loss_kw(h))
    first.backward(*args)
    assert rel(first.flat_grad(), z["grads"][0]) < 5e-5
    base = MP.MLPPortAgent(z["params"])
    base.step(*args)
    assert rel(base.flat(), z["params_after"][0]) > 1e-4


def check_torch_port_update(z):
    """The reference's whole update_params iteration (GAE, fixed log-probs, the np.random permutations, Adam) at the
    fixture's settings, driven through the torch port."""
    h = settings(z)
    agent = DO.port_agent(z["params"], h.get("weight_decay", 0.0), **adam_kw(h), **loss_kw(h))
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    states = expand_states(z)
    b_all = TP.stack_states(states)
    act = torch.tensor(z["actions"])
    with torch.no_grad():
        values = TP.value(agent.params(), b_all)
    adv, ret = TP.estimate_advantages(torch.tensor(z["rewards"]), torch.tensor(z["masks"]), values,
                                      *(float(x) for x in z["gamma_tau"]))
    with torch.no_grad():
        fixed, _ = TP.log_prob_entropy(agent.params(), b_all, act)
    exps_t = torch.tensor(z["exps"])
    np.random.seed(np_seed)
    order, losses = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(int(math.floor(T / B))):
            idx = order[i * B:(i + 1) * B]
            b = TP.stack_states([states[j] for j in idx])
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(agent.step(b, act[idx], adv[idx], ret[idx], fixed[idx], ind))
    assert np.allclose(np.array(losses), z["losses"], rtol=2e-5, atol=2e-6)
    assert rel(agent.flat(), z["params_after"]) < 5e-6


# ---- GPU: the CUDA paths against the reference -----------------------------------------------------------------------
def check_golden_trajectory(z, name, fused, dev):
    """Values and log-probs, then three steps: the first clips (two-call path on both), the next two run through
    upb_apply or the fused tail.  Losses from read_losses, every gradient tensor (the undecayed gradient) and the
    parameters after each step, with test_gpu_parity's bars (the parameter bar scaled to the lr)."""
    h = settings(z)
    mlp = name.startswith("mlp")
    layout = PL.MLP if mlp else PL.SGNN
    states = expand_states(z)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE, model="mlp" if mlp else "sgnn", **h)
    eps = h.get("clip_epsilon", 0.2)
    assert eng.clip_range == (float(np.float32(1.0 - eps)), float(np.float32(1.0 + eps)))
    assert eng.weight_decay == h.get("weight_decay", 0.0)
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
        worst, where = per_tensor_rel(grad.cpu().numpy()[:layout.num_params], z["grads"][k], layout)
        assert worst < TOL, (k, worst, where)
        assert rel(params.cpu().numpy(), z["params_after"][k]) < step_bar(h, 1e-5), k
    if name == "hlg_wd":
        # land-use only: the road head has no gradient, so it is neither stepped nor decayed
        road = heads(PL.SGNN)[1]
        assert np.array_equal(params.cpu().numpy()[road], z["params"][road])
        m, v, steps = eng.get_opt_state()
        assert not m[road].any() and not v[road].any() and steps.tolist() == [3, 3, 3, 0]
    if name == "small_mixed_hp0":
        # value_pred_coef = 0: a zero value-head gradient, not an absent one -- the head keeps its weights and zero
        # moments while its step counter (shared with the encoder) advances, as the reference's Adam counts its steps
        p = params.cpu().numpy()
        assert not grad.cpu().numpy()[VALUE_HEAD].any()
        assert np.array_equal(p[VALUE_HEAD], z["params"][VALUE_HEAD])
        m, v, steps = eng.get_opt_state()
        assert not m[VALUE_HEAD].any() and not v[VALUE_HEAD].any()
        assert steps.tolist() == [3, 3, 3, 3] and z["value_adam_steps"].tolist() == [3] * len(z["value_adam_steps"])


def check_update_params(z, dev):
    """The reference's whole update_params iteration at the fixture's settings through PPOUpdater, with the
    update_small test's tolerances."""
    from drl_urban_planning_b200.ppo import PPOUpdater
    h = settings(z)
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    gamma, tau = (float(x) for x in z["gamma_tau"])
    up = PPOUpdater(z["params"], int(z["n_cap"]), int(z["e_cap"]), dev, gamma=gamma, tau=tau, opt_num_epochs=epochs,
                    mini_batch_size=B, clip_mode=_lib.CLIP_REFERENCE, **h)
    assert up.engine.weight_decay == h.get("weight_decay", 0.0)
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


def check_use_b200_update(z, dev):
    """use_b200_update on a reference-shaped agent whose cfg carries the fixture's settings (`weightdecay` for the
    decay) reproduces the reference's update_params with that cfg, and writes the parameters back into the modules."""
    from drl_urban_planning_b200.agent import use_b200_update
    h = settings(z)
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    cfg = {k: v for k, v in h.items() if k != "weight_decay"}
    gamma, tau = (float(x) for x in z["gamma_tau"])
    logged = []
    ag = sgnn_agent(dev, int(z["n_cap"]), int(z["e_cap"]), z["params"], logged, gamma=gamma, tau=tau,
                    num_optim_epoch=epochs, mini_batch_size=B, weightdecay=h.get("weight_decay", 0.0), **cfg)
    ctl = use_b200_update(ag)
    assert ctl.updater.engine.weight_decay == h.get("weight_decay", 0.0)
    assert ctl.updater.engine.clip_range == clip_range(h.get("clip_epsilon", 0.2))
    batch = types.SimpleNamespace(states=expand_states(z), actions=z["actions"], rewards=z["rewards"], masks=z["masks"],
                                  exps=z["exps"])
    np.random.seed(np_seed)
    ag.update_params(batch, 0)
    assert np.allclose(update_losses(logged), z["losses"], rtol=2e-4, atol=2e-5)
    assert rel(ctl.updater.flat_params(), z["params_after"]) < 2e-5
    assert rel(ag.actor_critic_net.flat_parameters(), z["params_after"]) < 2e-5       # written back into the modules


# ---- GPU: the fused step against the two-call path -------------------------------------------------------------------
def hlg_case(dev, seed):
    """140 hlg-sized graphs of both stages (one in three a road graph): more than the 132 CTAs of a full grid."""
    states, actions = synth.make_states(seed, "hlg", 140, stages=[int(i % 3 == 1) for i in range(140)])
    return Case(dev, "sgnn", states, actions, seed)


def check_sgnn_fused_against_two_call(c, setting, grid):
    """upb_ppo_step (gradient + in-kernel reduction + Adam, one cooperative launch) against upb_ppo_grad + upb_apply
    over 4 steps, the first of which clips and takes the two-call path inside upb_ppo_step.  StepArgs (fused tail) and
    ApplyArgs (k_apply) must carry the same settings: every gradient tensor, the losses, the parameter trajectory,
    both moments and the step counters agree, one launch per non-clipping step, and away from the shipped settings the
    trajectory is far from theirs."""
    kw = SETTINGS[setting]
    e1, e2 = c.engine(grid_limit=grid, **kw), c.engine(grid_limit=grid, **kw)
    e0 = c.engine(grid_limit=grid)                                               # the shipped settings, for contrast
    p1, p2, p0 = (t(c.flat, c.dev).clone() for _ in range(3))
    for step in range(4):
        g1 = two_call_step(e1, c, p1)
        before = e2.launches
        g2 = fused_step(e2, c, p2)
        fused_step(e0, c, p0)
        torch.cuda.synchronize()
        assert (e2.launches - before == 1) == (step > 0), step
        worst, where = per_tensor_rel(g2.cpu().numpy()[:PL.NUM_PARAMS], g1.cpu().numpy()[:PL.NUM_PARAMS])
        assert worst < 1e-5, (step, worst, where)
        assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
        assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < step_bar(kw, 1e-6), step
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    live_heads = [int((c.stage == s).any()) for s in (0, 1)]
    assert s1.tolist() == s2.tolist() == [4, 4, 4 * live_heads[0], 4 * live_heads[1]]
    assert rel(m2, m1) < 1e-5 and rel(v2, v1) < 1e-5
    if kw:
        assert rel(p2.cpu().numpy(), p0.cpu().numpy()) > 1e-3


def check_mlp_fused_bit_identical(c, setting, grid):
    """On one GPU the rl-mlp fused step (upb_mlp_ppo_step, mlp_fused_tail in csrc/mlp_kernel.cuh) reduces every
    gradient column in k_mlp_reduce's order and applies k_apply's Adam (the decay the same fused multiply-add on the
    same old parameter), so on reproducible batches (harness.reproducible_states) it is bit-identical to
    upb_mlp_ppo_grad + upb_mlp_apply: parameters, the whole gradient / statistics buffer, both moments and the four step
    counters.  4 steps: mixed (clips in CLIP_REFERENCE mode: the library's two-call fallback), mixed, land-use only
    (the road head never fires), mixed; away from the shipped settings the trajectory is far from theirs."""
    kw = SETTINGS[setting]
    lu, allg = np.flatnonzero(c.stage == 0), np.arange(c.count)
    assert (c.stage == 1).any() and len(lu) > 0 and (c.exps[allg] == 0).any() and (c.exps[lu] == 0).any()
    e1, e2 = c.engine(grid_limit=grid, **kw), c.engine(grid_limit=grid, **kw)
    e0 = c.engine(grid_limit=grid)
    assert e2.grid == min(grid, torch.cuda.get_device_properties(c.dev).multi_processor_count)
    p1, p2, p0 = (t(c.flat, c.dev).clone() for _ in range(3))
    for step, sel in enumerate([allg, allg, lu, allg]):
        assert e2.next_step_fused() == (step > 0)
        g1 = two_call_step(e1, c, p1, sel)
        before = e2.launches
        g2 = fused_step(e2, c, p2, sel)
        fused_step(e0, c, p0, sel)
        assert e2.launches - before == (3 if step == 0 else 1), step
        steps = assert_same_state(e1, p1, g1, e2, p2, g2, (grid, step))
    assert steps.tolist() == [4, 4, 4, 3]
    if kw:
        assert rel(p2.cpu().numpy(), p0.cpu().numpy()) > 1e-3
