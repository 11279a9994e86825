"""GPU: value-target normalisation (`value_norm`, upb_set_value_norm) on both models.

  a. k_value_norm from its own inputs against tests/vnorm_oracle.py: the float64 state within 1e-12, the rescaled
     val_w2 / val_b2 and every normalised return and old value bit for bit, deterministic, with returns scaled x1e3 and
     a non-finite return (state and head unchanged); k_value_denorm bit for bit;
  b. the first update (d == 0): denormalised values, and so GAE, bit-identical to an updater with the option off;
  c. PopArt on the device: a forward pass after the rescale, denormalised with the new statistics, is the pre-pass
     denormalised with the old ones;
  d. three consecutive update_params iterations: each update from its own inputs against the oracle, and sampled steps
     teacher-forced against the float64 oracles fed the kernel's own normalised returns / old values (the SGNN also with
     value_clip, normalize_advantage, max_grad_norm, the KL penalty and diagnostics);
  e. resuming through B200Update.save_checkpoint / load_checkpoint gives the next update bit for bit;
  f. off: no launch and no change; on: two launches per update more."""
import os
import pickle
import types

import numpy as np
import pytest
import torch

import decay_oracle as DO
import gclip_oracle as GO
import klpen_oracle as KO
import ppo_oracle as PPO
import scale_cases as SC
import vnorm_oracle as VN
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.agent import use_b200_update
from drl_urban_planning_b200.packing import pack_states
from drl_urban_planning_b200.ppo import GCLIP_NORM_SLOT, KLPEN_SLOT, VCLIP_LOSS_SLOT, PPOUpdater
from harness import dev, per_tensor_rel, rel, reproducible_states  # noqa: F401  (dev: fixture)
from oracle import sgnn_numpy as ON
from test_gpu_live_hyperparams import make_agent

pytestmark = pytest.mark.gpu

SPEC = synth.COMMUNITIES["small"]
N_CAP, E_CAP = SPEC.max_num_nodes, SPEC.max_num_edges
MODELS = ["sgnn", "mlp"]
GRAD_BAR, LOSS_RTOL, ADAM_BAR, V_BAR = 1e-4, 1e-4, 1e-5, 1.4e-5      # tests/test_gpu_update_scale.py's bars


def layout_of(model):
    return PL.MLP if model == "mlp" else PL.SGNN


def flat_init(model, seed):
    return PL.MLP.default_init(seed) if model == "mlp" else PL.default_init(seed)


def head(layout, p):
    p = np.asarray(p)
    w, b = layout.slots["val_w2"], layout.slots["val_b2"]
    return p[w.offset:w.offset + 32].copy(), np.float32(p[b.offset])


def engine(dev, model, **kw):
    from drl_urban_planning_b200.engine import Engine
    return Engine(dev, N_CAP, E_CAP, model=model, **kw)


# ---- a. the kernels against the oracle -------------------------------------------------------------------------------
def returns_sets(seed, T):
    rng = np.random.default_rng(seed)
    base = rng.normal(2.0, 3.0, T).astype(np.float32)
    nan = base.copy()
    nan[T // 3] = np.nan
    inf = base.copy()
    inf[-1] = np.inf
    return [("plain", base), ("x1e3", (base * 1e3 + 5e3).astype(np.float32)), ("nan", nan),
            ("small", (base * 1e-3).astype(np.float32)), ("inf", inf), ("constant", np.full(T, 7.0, np.float32))]


def kernel_update(eng, params, R, V):
    st0 = eng.get_value_norm_state()
    n0 = eng.launches
    r, v, ms = eng.value_norm_update(torch.as_tensor(R, device=eng.device), params, torch.as_tensor(V, device=eng.device))
    assert eng.launches == n0 + 1
    torch.cuda.synchronize()
    return st0, dict(state=eng.get_value_norm_state(), returns=r.cpu().numpy(), values=v.cpu().numpy(),
                     mean_std=tuple(ms.cpu().numpy().tolist()), params=params.cpu().numpy())


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("beta", [0.99999, 0.9])
def test_k_value_norm_against_the_oracle(dev, model, beta):
    layout = layout_of(model)
    T = 3001                                       # not a multiple of the block
    eng = engine(dev, model, value_norm=True, value_norm_beta=beta)
    twin = engine(dev, model, value_norm=True, value_norm_beta=beta)
    params = torch.as_tensor(flat_init(model, 3), device=dev).clone()
    rng = np.random.default_rng(5)
    for what, R in returns_sets(11, T):
        V = (R + rng.normal(0, 1, T)).astype(np.float32)
        p_before = params.cpu().numpy()
        w2, b2 = head(layout, p_before)
        twin_params = params.clone()
        twin.set_value_norm_state(eng.get_value_norm_state())
        st0, got = kernel_update(eng, params, R, V)
        want_state = VN.update(st0, R, beta)
        assert state_close(got["state"], want_state, R, beta), (what, got["state"], want_state)
        want = VN.step(st0, R, V, w2, b2, beta, new_state=got["state"])
        gw2, gb2 = head(layout, got["params"])
        assert np.array_equal(gw2, want["w2"]) and gb2 == want["b2"], (what, gb2, want["b2"])
        assert np.array_equal(got["returns"], want["returns"], equal_nan=True), what
        assert np.array_equal(got["values"], want["values"], equal_nan=True), what
        assert got["mean_std"] == want["stats"], what
        others = np.ones(layout.num_params, bool)
        others[layout.slots["val_w2"].offset:layout.slots["val_b2"].offset + 1] = False
        assert np.array_equal(got["params"][others], p_before[others]), what
        if not np.isfinite(R).all():
            assert got["state"] == st0 and np.array_equal(got["params"], p_before), what
        # deterministic: the same inputs on another context give the same bits
        _, again = kernel_update(twin, twin_params, R, V)
        assert again["state"] == got["state"] and again["mean_std"] == got["mean_std"], what
        for k in ("returns", "values", "params"):
            assert np.array_equal(again[k], got[k], equal_nan=True), (what, k)
        # k_value_denorm with the state just reached
        n = rng.normal(0, 2, T).astype(np.float32)
        n0 = eng.launches
        den = eng.denormalize_values(torch.as_tensor(n, device=dev)).cpu().numpy()
        assert eng.launches == n0 + 1
        assert np.array_equal(den, VN.denormalize(n, got["state"])), what
    assert eng.get_value_norm_state()[2] > 0


@pytest.mark.parametrize("model", MODELS)
def test_update_without_values_and_argument_errors(dev, model):
    eng = engine(dev, model, value_norm=True)
    params = torch.as_tensor(flat_init(model, 4), device=dev).clone()
    R = torch.linspace(-3, 9, 700, device=dev)
    r, v, ms = eng.value_norm_update(R, params)
    assert v is None
    torch.cuda.synchronize()
    want = VN.normalize(R.cpu().numpy(), VN.stats(*eng.get_value_norm_state()))
    assert np.array_equal(r.cpu().numpy(), want)
    off = engine(dev, model)
    with pytest.raises(ValueError, match="off"):
        off.value_norm_update(R, params)
    L = _lib.lib()
    rc = getattr(L, off._p + "value_norm_update")(off._ctx, R.data_ptr(), None, 700, params.data_ptr(),
                                                   r.data_ptr(), None, None, off._stream())
    assert rc != 0 and b"off" in L.upb_last_error()
    with pytest.raises(ValueError):
        eng.set_value_norm_state((0.0, -1.0, 0.5))
    with pytest.raises(ValueError):
        eng.set_value_norm_state((float("nan"), 0.0, 0.5))
    eng.set_value_norm_state((1.0, 5.0, 0.5))
    assert eng.get_value_norm_state() == (1.0, 5.0, 0.5)


# ---- a rollout of small graphs ---------------------------------------------------------------------------------------
def rollout(seed, T, reward_scale=1.0, reward_shift=0.0):
    states, actions = reproducible_states(seed, T)
    rng = np.random.default_rng(seed)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 40, replace=False)] = 0.0
    exps = np.where(rng.random(T) < 0.05, 0.0, 1.0).astype(np.float32)
    rewards = (rng.standard_normal(T) * reward_scale + reward_shift).astype(np.float32)
    return types.SimpleNamespace(T=T, states=states, actions=actions, rewards=rewards, masks=masks, exps=exps)


def updater(dev, model, flat, **kw):
    return PPOUpdater(flat, N_CAP, E_CAP, dev, gamma=0.99, tau=0.95, opt_num_epochs=2, mini_batch_size=64, model=model,
                      process_group=None, **{"clip_mode": _lib.CLIP_NEVER, **kw})


def run_update(up, ro, seed, iteration=0):
    logged = []
    np.random.seed(seed)
    out = up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps, iteration=iteration,
                           log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    torch.cuda.synchronize()
    return out, logged


# ---- b. identity on the first update ---------------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
def test_first_update_is_the_identity(dev, model):
    ro = rollout(7, 256, reward_scale=40.0, reward_shift=100.0)
    flat = flat_init(model, 7)
    on, off = updater(dev, model, flat, value_norm=True), updater(dev, model, flat)
    spied = {}
    inner = on.engine.value_norm_update

    def spy(returns, params, values=None):
        spied.update(returns=returns.cpu().numpy(), values=values.cpu().numpy())
        return inner(returns, params, values)
    on.engine.value_norm_update = spy
    out_on, logged = run_update(on, ro, 1)
    run_update(off, ro, 1)
    # the pre-pass is the same (the parameters are), so with d == 0 the values and GAE are bit for bit
    adv_off, ret_off = off.advantages.cpu().numpy(), off.returns.cpu().numpy()
    assert np.array_equal(on.advantages.cpu().numpy(), adv_off)
    assert np.array_equal(spied["returns"], ret_off)
    assert np.array_equal(spied["values"], off.old_values.cpu().numpy())
    beta = 0.99999
    st = on.engine.get_value_norm_state()
    assert st[2] == 1.0 - beta
    stats = VN.stats(*st)
    assert (out_on["value_norm_mean"], out_on["value_norm_std"]) == stats
    assert abs(stats[0] - ret_off.astype(np.float64).mean()) < 1e-9 * abs(stats[0])
    assert np.array_equal(on.returns.cpu().numpy(), VN.normalize(ret_off, stats))
    assert np.array_equal(on.old_values.cpu().numpy(), VN.normalize(spied["values"], stats))
    tags = {tag: (v, s) for tag, v, s in logged if tag.startswith("diag/value_norm")}
    assert tags == {"diag/value_norm_mean": (stats[0], 0), "diag/value_norm_std": (stats[1], 0)}


# ---- c. PopArt preserves the head's outputs on the device -----------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("start", [(0.0, 0.0, 0.0), (0.9, 60.0, 0.3)])
def test_rescale_preserves_the_denormalised_values(dev, model, start):
    states, actions = reproducible_states(9, 200)
    blob = pack_states(states).to(dev)
    eng = engine(dev, model, value_norm=True, value_norm_beta=0.9)
    eng.set_value_norm_state(start)
    params = torch.as_tensor(flat_init(model, 9), device=dev).clone()
    act = torch.as_tensor(actions, device=dev)
    before = eng.denormalize_values(eng.forward(blob, params, act)[0]).cpu().numpy()
    R = torch.as_tensor(np.random.default_rng(2).normal(30.0, 8.0, 200).astype(np.float32), device=dev)
    eng.value_norm_update(R, params)
    after = eng.denormalize_values(eng.forward(blob, params, act)[0]).cpu().numpy()
    new = VN.stats(*eng.get_value_norm_state())
    assert new[1] > 5.0 and abs(new[0]) > 5.0                 # the statistics moved a long way
    # relative to the values or to the new std, whichever is larger: every output now carries the fp32 rounding of
    # std-sized terms (the rescaled bias, fp32(mean), the head's normalised output times std)
    err = rel(after, before, floor=new[1])
    assert err <= 1e-5, err


# ---- d. three iterations, teacher forced -----------------------------------------------------------------------------
class Capture:
    """Records every upb_value_norm_update of an updater: its inputs, the state and head before it, its outputs."""

    def __init__(self, up):
        self.up, self.inner, self.calls = up, up.engine.value_norm_update, []
        up.engine.value_norm_update = self

    def __call__(self, returns, params, values=None):
        eng = self.up.engine
        rec = dict(returns=returns.cpu().numpy(), values=values.cpu().numpy(), state=eng.get_value_norm_state(),
                   params=params.cpu().numpy())
        out = self.inner(returns, params, values)
        torch.cuda.synchronize()
        rec.update(new_state=eng.get_value_norm_state(), new_params=params.cpu().numpy(),
                   norm_returns=out[0].cpu().numpy(), norm_values=out[1].cpu().numpy())
        self.calls.append(rec)
        return out


def state_close(got, want, R, beta):
    """Within 1e-12 of each value, or of the size of its batch term (a mean near 0 sums cancelling returns)."""
    r = np.asarray(R, np.float64)
    floors = (1.0 - beta) * np.array([np.abs(r).mean(), (r * r).mean(), 1.0]) if np.isfinite(r).all() else np.zeros(3)
    return all(abs(g - w) <= 1e-12 * max(abs(w), f) for g, w, f in zip(got, want, floors))


def check_update_call(c, layout, beta):
    want_state = VN.update(c["state"], c["returns"], beta)
    assert state_close(c["new_state"], want_state, c["returns"], beta), (c["new_state"], want_state)
    w2, b2 = head(layout, c["params"])
    want = VN.step(c["state"], c["returns"], c["values"], w2, b2, beta, new_state=c["new_state"])
    gw2, gb2 = head(layout, c["new_params"])
    assert np.array_equal(gw2, want["w2"]) and gb2 == want["b2"]
    assert np.array_equal(c["norm_returns"], want["returns"]) and np.array_equal(c["norm_values"], want["values"])


def check_step(layout, rec, k, stages, want_grad, want_losses, got_losses, grad_fn=None, wd=0.0):
    row = rec.bufs[k].cpu().numpy().astype(np.float64)
    bad = []
    e, where = per_tensor_rel(row[:layout.num_params], want_grad, layout)
    if not e < GRAD_BAR:
        bad.append(f"gradient {where} {e:.3g}")
    got_losses, want_losses = np.asarray(got_losses, np.float64), np.asarray(want_losses, np.float64)
    if not np.allclose(got_losses, want_losses, rtol=LOSS_RTOL, atol=1e-6):
        bad.append(f"losses {got_losses.tolist()} vs {want_losses.tolist()}")
    g = row[:layout.num_params] if grad_fn is None else grad_fn(row)
    p0, m0, v0, s0 = rec.before[k]
    p1, m1, v1, s1 = rec.after[k]
    want = DO.adam_step(p0, m0, v0, SC.entry_steps(s0, layout), g, SC.live_entries(stages, layout), wd)
    for name, got, w, bar in (("params", p1, want[0], ADAM_BAR), ("m", m1, want[1], ADAM_BAR), ("v", v1, want[2], V_BAR)):
        if not rel(got, w) < bar:
            bad.append(f"{name} {rel(got, w):.3g}")
    return bad


SAMPLE = [0, 3, 6]       # of the 2 x 4 steps of an iteration


@pytest.mark.parametrize("model", MODELS)
def test_three_iterations_teacher_forced(dev, model):
    layout = layout_of(model)
    beta = 0.9
    up = updater(dev, model, flat_init(model, 12), value_norm=True, value_norm_beta=beta)
    cap = Capture(up)
    failures = []
    for it, (scale, shift) in enumerate([(1.0, 0.0), (30.0, 200.0), (5.0, -50.0)]):
        ro = rollout(20 + it, 256, scale, shift)
        rec = SC.Recorder(up, SAMPLE, ro.T // 64)
        out, _ = run_update(up, ro, 40 + it, iteration=it)
        up.minibatch_step = rec.inner
        c = cap.calls[-1]
        check_update_call(c, layout, beta)
        assert (out["value_norm_mean"], out["value_norm_std"]) == VN.stats(*c["new_state"])
        if it:
            assert abs(out["value_norm_mean"]) > 1.0            # away from the identity
        stage = up.blob.info[:, 3].astype(np.int64)
        ret, adv = c["norm_returns"], up.advantages.cpu().numpy()
        fixed = up.fixed_log_probs.cpu().numpy()
        for k in SAMPLE:
            ids = rec.ids[k]
            flat = rec.before[k][0]
            if model == "sgnn":
                x = ON.ppo_minibatch(flat, [ro.states[i] for i in ids], ro.actions[ids], adv[ids], ret[ids], fixed[ids],
                                     ro.exps[ids])
            else:
                x = PPO.mlp_minibatch(flat, [ro.states[i] for i in ids], ro.actions[ids], adv[ids], ret[ids],
                                      fixed[ids], ro.exps[ids])
            bad = check_step(layout, rec, k, stage[ids], x["grad"],
                             [x["loss"], x["value_loss"], x["surr_loss"], x["entropy_loss"]],
                             up.engine.read_losses(rec.bufs[k]))
            if bad:
                failures.append(f"iteration {it} step {k}: " + "; ".join(bad))
    assert not failures, "\n".join(failures)


def test_sgnn_three_iterations_with_the_other_options(dev):
    layout = PL.SGNN
    beta, vclip = 0.9, float(np.float32(0.2))
    opts = dict(max_grad_norm=0.5, value_clip=0.2, normalize_advantage=True, kl_coef=0.1, diagnostics=True)
    up = updater(dev, "sgnn", flat_init("sgnn", 13), value_norm=True, value_norm_beta=beta, **opts)
    cap = Capture(up)
    so = up.engine.stat_offset
    failures = []
    for it, (scale, shift) in enumerate([(2.0, 10.0), (30.0, 200.0), (5.0, -50.0)]):
        ro = rollout(30 + it, 256, scale, shift)
        rec = SC.Recorder(up, SAMPLE, ro.T // 64)
        out, logged = run_update(up, ro, 50 + it, iteration=it)
        up.minibatch_step = rec.inner
        c = cap.calls[-1]
        check_update_call(c, layout, beta)
        assert np.array_equal(up.old_values.cpu().numpy(), c["norm_values"])
        assert "diag/total_explained_variance" in {tag for tag, _, _ in logged}
        stage = up.blob.info[:, 3].astype(np.int64)
        lp_old = [lp for lp, _ in KO.per_graph(up.old_cand_log_probs.cpu().numpy(), up.blob)]
        fixed = up.fixed_log_probs.cpu().numpy()
        for k in SAMPLE:
            ids = rec.ids[k]
            x = PPO.sgnn_minibatch(rec.before[k][0], [ro.states[i] for i in ids], ro.actions[ids],
                                   rec.norm_adv[k // 4][ids], c["norm_returns"][ids], fixed[ids], ro.exps[ids],
                                   old_values=c["norm_values"][ids], lp_old=[lp_old[i] for i in ids], value_clip=vclip,
                                   kl_coef=0.1)
            st = rec.bufs[k].cpu().numpy().astype(np.float64)[so:so + 20]
            n, ni = st[3], st[4]
            got = [st[1] / ni, st[VCLIP_LOSS_SLOT] / n, st[2] / ni, st[KLPEN_SLOT] / ni]
            want = [x["surr_sum"] / x["n_ind"], x["value_loss_sum"] / x["n"], x["ent_sum"] / x["n_ind"],
                    x["kl_sum"] / x["n_ind"]]
            bad = check_step(layout, rec, k, stage[ids], x["grad"], want, got,
                             grad_fn=lambda row: GO.clip64(row[:layout.num_params], 0.5)[0])
            norm = GO.clip64(rec.bufs[k].cpu().numpy().astype(np.float64)[:layout.num_params], 0.5)[1]
            if not abs(st[GCLIP_NORM_SLOT] - norm) < 1e-6 * norm:
                bad.append(f"slot 17 {st[GCLIP_NORM_SLOT]} vs {norm}")
            if bad:
                failures.append(f"iteration {it} step {k}: " + "; ".join(bad))
    assert not failures, "\n".join(failures)


# ---- e. checkpoints --------------------------------------------------------------------------------------------------
def checkpointing_agent(model, dev, flat, tmp, logged):
    ag = make_agent(model, dev, flat, logged, num_optim_epoch=2, mini_batch_size=16)
    ag.cfg.model_dir, ag.cfg.save_model_interval = str(tmp), 1

    def save_checkpoint(iteration):
        with open(os.path.join(str(tmp), "iteration_%04d.p" % (iteration + 1)), "wb") as f:
            pickle.dump({"actor_critic_dict": ag.actor_critic_net.state_dict(), "iteration": iteration}, f)

    def load_checkpoint(checkpoint, restore_best_rewards=True):
        with open(os.path.join(str(tmp), "iteration_%04d.p" % checkpoint), "rb") as f:
            cp = pickle.load(f)
        ag.actor_critic_net.load_state_dict(cp["actor_critic_dict"])
        return cp["iteration"] + 1
    ag.save_checkpoint, ag.load_checkpoint = save_checkpoint, load_checkpoint
    return ag


@pytest.mark.parametrize("model", MODELS)
def test_checkpoint_resume_is_bit_identical(dev, model, tmp_path):
    flat = flat_init(model, 14)
    kw = dict(clip_mode=_lib.CLIP_NEVER, process_group=None, value_norm=True, value_norm_beta=0.9)
    ros = [rollout(60 + i, 48, 20.0, 50.0 * i) for i in range(3)]
    a = checkpointing_agent(model, dev, flat, tmp_path, [])
    ctl_a = use_b200_update(a, **kw)
    for it in range(2):
        np.random.seed(70 + it)
        a.update_params(ros[it], it)
    a.save_checkpoint(1)
    assert "value_norm" in pickle.load(open(tmp_path / "iteration_0002.p", "rb"))[ctl_a.CHECKPOINT_KEY]
    b = checkpointing_agent(model, dev, flat_init(model, 99), tmp_path, [])
    ctl_b = use_b200_update(b, **kw)
    assert b.load_checkpoint(2) == 2
    assert ctl_b.value_stats() == ctl_a.value_stats() != (0.0, 1.0)
    for ag in (a, b):
        np.random.seed(72)
        ag.update_params(ros[2], 2)
    torch.cuda.synchronize()
    assert np.array_equal(ctl_a.updater.flat_params(), ctl_b.updater.flat_params())
    for x, y in zip(ctl_a.updater.engine.get_opt_state(), ctl_b.updater.engine.get_opt_state()):
        assert np.array_equal(x, y)
    assert ctl_a.updater.engine.get_value_norm_state() == ctl_b.updater.engine.get_value_norm_state()


# ---- f. off changes nothing ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
def test_off_is_unchanged_and_on_adds_two_launches(dev, model):
    ro = rollout(80, 256)
    flat = flat_init(model, 15)
    plain, off, on = (updater(dev, model, flat), updater(dev, model, flat, value_norm=False, value_norm_beta=0.5),
                      updater(dev, model, flat, value_norm=True))
    counts, res = [], []
    for up in (plain, off, on):
        n0 = up.engine.launches
        out, logged = run_update(up, ro, 3)
        counts.append(up.engine.launches - n0)
        res.append((up.flat_params(), out, logged))
    assert counts[0] == counts[1] and counts[2] == counts[0] + 2
    assert np.array_equal(res[0][0], res[1][0]) and res[0][2] == res[1][2]
    assert {k: np.asarray(v).tolist() for k, v in res[0][1].items()} == \
        {k: np.asarray(v).tolist() for k, v in res[1][1].items()}
    assert "value_norm_mean" not in res[0][1] and not any(t.startswith("diag/value_norm") for t, _, _ in res[0][2])
