"""GPU: one whole `update_params` iteration at the product's size -- 25,000 HLG-shaped states, minibatches of 256,
4 epochs, 388 optimiser steps -- which the other update tests (at most 1,024 states) never reach: chunked packing over
13 chunks, a 97-row statistics ring with a 168-state remainder, k_adv_norm on 97 blocks, k_gae over thousands of
episodes, hundreds of fused launches in a row, and buffers reused from one iteration to the next.

  a. the pre-pass: values and fixed log-probs of every state against the float64 oracle, GAE bit for bit;
  b. the schedule: each minibatch holds exactly its slice of the replayed np.random order, the remainder is never
     stepped, the logged losses are the ring rows, the totals their per-epoch means, the counters 388;
  c. sampled steps, teacher forced: the float64 oracle from the kernel's own parameters, moments and inputs just
     before the step (gradient, losses, the Adam step, the counters);
  d. the instrumentation changes nothing: an unwrapped run is bit-identical;
  e. three consecutive iterations (25,000, 6,561, 25,000 states) on one updater, each bit-identical to a fresh updater
     loaded with the previous parameters and Adam state;
  f. every PPO option at once (SGNN) against a float64 oracle composed from the per-option ones;
  g. rl-mlp: a-c against the rl-mlp port in float64 (its fused path is not run-to-run reproducible on arbitrary land-use
     graphs, harness.reproducible_states, so d and e do not apply).
A failing sampled step names the step, its epoch and the tensor.  The worst errors are printed (pytest -s)."""
import types

import numpy as np
import pytest
import torch

import decay_oracle as DO
import gclip_oracle as GO
import klpen_oracle as KO
import ppo_oracle as PPO
import scale_cases as SC
import vclip_oracle as VO
from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.engine import adapt_kl_coef
from drl_urban_planning_b200.ppo import (GCLIP_NORM_SLOT, KLPEN_SLOT, NONFINITE_SLOT, VCLIP_LOSS_SLOT, PPOUpdater)
from harness import dev, per_tensor_rel, rel, update_losses  # noqa: F401  (dev: fixture)
from oracle import sgnn_numpy as ON
from shape_cases import SPEC

pytestmark = pytest.mark.gpu

T, B, EPOCHS = SC.T_PRODUCT, SC.B, SC.EPOCHS
NB = T // B                                             # 97 minibatches per epoch
NP_SEED = 5
GRAD_BAR, LOSS_RTOL, ADAM_BAR = 1e-4, 1e-4, 1e-5
# The second moment's bar.  torch.optim.Adam adds (1 - beta2) g^2 with 1 - beta2 formed in double (fp32 0.001); the
# library forms the weight in fp32 as 1 - fp32(0.999) = 9.99987e-4, 1.29e-5 below it, and its bias correction
# 1 - fp32(0.999)^t carries the same factor, so v / (1 - beta2^t), and with it every parameter, agrees at fp32
# round-off (params 5e-8 here) while the stored v sits up to 1.29e-5 low after a step from zero moments (step 0).
V_BAR = 1.4e-5
ALL_OPTIONS = dict(clip_mode=_lib.CLIP_NEVER, max_grad_norm=0.5, weight_decay=1e-2, value_clip=0.2,
                   normalize_advantage=True, kl_coef=0.1, kl_target=0.01, skip_nonfinite=True, diagnostics=True)


def report(what, worst):
    print(f"\n[scale] {what}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.fixture(scope="module")
def pool():
    return SC.make_pool()


@pytest.fixture(scope="module")
def rollout(pool):
    states, _ = pool
    return SC.Rollout(states, T, seed=21)


def updater(dev, flat, model="sgnn", **kw):
    return PPOUpdater(flat, SPEC.max_num_nodes, SPEC.max_num_edges, dev, gamma=SC.GAMMA, tau=SC.TAU,
                      opt_num_epochs=EPOCHS, mini_batch_size=B, model=model, process_group=None,
                      **{"clip_mode": _lib.CLIP_REFERENCE, **kw})


def run(dev, ro, flat, sample=None, np_seed=NP_SEED, model="sgnn", **kw):
    """One update_params iteration of rollout `ro`, instrumented when `sample` is given."""
    up = updater(dev, flat, model, **kw)
    rec = SC.Recorder(up, sample, ro.T // B) if sample is not None else None
    logged = []
    np.random.seed(np_seed)
    out = up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps,
                           log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    torch.cuda.synchronize()
    m, v, steps = up.engine.get_opt_state()
    return types.SimpleNamespace(up=up, rec=rec, logged=logged, out=out, params=up.flat_params(), m=m, v=v,
                                 steps=steps, stage=up.blob.info[:, 3].astype(np.int64), ro=ro,
                                 adv=up.advantages.cpu().numpy(), ret=up.returns.cpu().numpy(),
                                 values=up.old_values.cpu().numpy(), fixed=up.fixed_log_probs.cpu().numpy())


def sampled(ro, seed=3):
    return SC.sample_steps(SC.epoch_orders(NP_SEED, ro.T), ro.big_pos, ro.T // B, seed)


@pytest.fixture(scope="module")
def sgnn(dev, rollout):
    return run(dev, rollout, PL.default_init(21), sampled(rollout))


@pytest.fixture(scope="module")
def mlp(dev, rollout):
    return run(dev, rollout, PL.MLP.default_init(21), sampled(rollout), model="mlp")


# ---- a. the pre-pass -------------------------------------------------------------------------------------------------
def check_prepass(r, per_pool, pool):
    ro = r.ro
    assert (ro.lengths == 1).any() and (ro.lengths > B).any() and ro.masks[-1] == 1
    assert (ro.exps == 0).any() and len(set(ro.src.tolist())) >= SC.POOL
    values, logp = SC.prepass_of_samples(per_pool, pool, ro.src, ro.actions)
    worst = dict(values=rel(r.values, values), fixed_log_probs=rel(r.fixed, logp))
    report(f"pre-pass ({r.up.engine.model})", worst)
    assert worst["values"] < 1e-4 and worst["fixed_log_probs"] < 1e-4, worst
    adv, ret = ON.estimate_advantages(ro.rewards, ro.masks, r.values, SC.GAMMA, SC.TAU)
    assert np.array_equal(r.adv, adv.ravel()) and np.array_equal(r.ret, ret.ravel())


def test_sgnn_prepass(sgnn, pool):
    states, _ = pool
    check_prepass(sgnn, SC.sgnn_prepass(states, PL.default_init(21)), states)


def test_mlp_prepass(mlp, pool):
    states, _ = pool
    check_prepass(mlp, SC.mlp_prepass(states, PL.MLP.default_init(21)), states)


# ---- b. the schedule -------------------------------------------------------------------------------------------------
def check_schedule(r):
    ro, rec, up = r.ro, r.rec, r.up
    nb = ro.T // B
    orders = SC.epoch_orders(NP_SEED, ro.T)
    assert len(rec.ids) == EPOCHS * nb
    for k, ids in enumerate(rec.ids):
        e, i = divmod(k, nb)
        want = orders[e][i * B:(i + 1) * B]
        assert np.array_equal(np.sort(ids), np.sort(want)), (k, e, i)
        assert rec.rows[k] == i, (k, rec.rows[k])
        assert rec.args[k] == (B, int((ro.exps[want] != 0).sum())), (k, rec.args[k])
    for e in range(EPOCHS):
        stepped = np.concatenate(rec.ids[e * nb:(e + 1) * nb])
        assert stepped.size == nb * B and not np.isin(orders[e][nb * B:], stepped).any(), e
    losses = update_losses(r.logged)
    assert losses.shape == (EPOCHS * nb, 4)
    ring = np.array([up.engine.read_losses(b) for b in rec.bufs])
    assert np.allclose(losses, ring, rtol=1e-6, atol=1e-7), np.abs(losses - ring).max()
    totals = losses.reshape(EPOCHS, nb, 4).sum(1).mean(0)
    got = [r.out[k] for k in ("total_loss", "total_value_loss", "total_surr_loss", "total_entropy_loss")]
    assert np.allclose(got, totals, rtol=1e-12, atol=0)
    has = [sum(bool((r.stage[ids] == s).any()) for ids in rec.ids) for s in (0, 1)]
    assert r.steps.tolist() == [EPOCHS * nb, EPOCHS * nb] + has, (r.steps.tolist(), has)
    assert ro.T != T or r.steps[0] == 388


def test_sgnn_schedule(sgnn):
    check_schedule(sgnn)


def test_mlp_schedule(mlp):
    check_schedule(mlp)


# ---- c. sampled steps, teacher forced --------------------------------------------------------------------------------
def check_adam(r, k, grad, worst, wd=0.0):
    """The step's parameters, moments and counters against one float64 Adam step from the snapshot before it, on the
    kernel's own (clipped) gradient; None, or what failed."""
    layout = PL.MLP if r.up.engine.model == "mlp" else PL.SGNN
    p0, m0, v0, s0 = r.rec.before[k]
    p1, m1, v1, s1 = r.rec.after[k]
    stages = r.stage[r.rec.ids[k]]
    live = SC.live_entries(stages, layout)
    want = DO.adam_step(p0, m0, v0, SC.entry_steps(s0, layout), grad, live, wd)
    errs = dict(params=rel(p1, want[0]), m=rel(m1, want[1]), v=rel(v1, want[2]))
    for name, e in errs.items():
        worst[name] = max(worst.get(name, 0.0), e)
    bad = [f"{name} {e:.3g}" for name, e in errs.items() if not e < (V_BAR if name == "v" else ADAM_BAR)]
    step = (s1 - s0).tolist()
    if step != [1, 1, int((stages == 0).any()), int((stages == 1).any())]:
        bad.append(f"counters {s0.tolist()} -> {s1.tolist()}")
    return bad


def check_grad(r, k, want, worst):
    layout = PL.MLP if r.up.engine.model == "mlp" else PL.SGNN
    row = r.rec.bufs[k].cpu().numpy().astype(np.float64)
    e, where = per_tensor_rel(row[:layout.num_params], want, layout)
    worst["grad"] = max(worst.get("grad", 0.0), e)
    return row, ([f"gradient {where} {e:.3g}"] if not e < GRAD_BAR else [])


def check_losses(got, want, worst):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    e = float((np.abs(got - want) / np.maximum(np.abs(want), 1e-30)).max())
    worst["losses"] = max(worst.get("losses", 0.0), e)
    return [] if np.allclose(got, want, rtol=LOSS_RTOL, atol=1e-6) else [f"losses {got.tolist()} vs {want.tolist()}"]


def check_sampled(r, oracle):
    """oracle(k) -> (want gradient, want losses) for the sampled step k; every sampled step is checked, the failures
    are reported together."""
    layout = PL.MLP if r.up.engine.model == "mlp" else PL.SGNN
    nb = r.ro.T // B
    worst, failures = {}, []
    for k, (want_grad, want_losses) in oracle.items():
        row, bad = check_grad(r, k, want_grad, worst)
        bad += check_losses(r.up.engine.read_losses(r.rec.bufs[k]), want_losses, worst)
        g = row[:layout.num_params]
        bad += check_adam(r, k, SC.clip_groups(g, layout) if k == 0 else g, worst)
        if bad:
            failures.append(f"step {k} (epoch {k // nb}, minibatch {k % nb}): " + "; ".join(bad))
    report(f"sampled steps {sorted(oracle)} ({r.up.engine.model})", worst)
    assert not failures, "\n".join(failures)


def test_sgnn_sampled_steps(sgnn):
    r = sgnn
    ks = sorted(r.rec.before)
    assert any(np.isin(r.rec.ids[k], r.ro.big_pos).any() for k in ks), "no sampled minibatch holds a large-path graph"
    res = SC.run_steps(SC._sgnn_step, [(r.rec.before[k][0], r.rec.ids[k]) for k in ks], states=r.ro.states,
                       actions=r.ro.actions, adv=r.adv, ret=r.ret, fixed=r.fixed, exps=r.ro.exps)
    check_sampled(r, {k: (x["grad"], [x["loss"], x["value_loss"], x["surr_loss"], x["entropy_loss"]])
                      for k, x in zip(ks, res)})


def test_mlp_sampled_steps(mlp):
    r = mlp
    ro = r.ro
    want = {}
    for k in sorted(r.rec.before):
        ids = r.rec.ids[k]
        x = PPO.mlp_minibatch(r.rec.before[k][0], [ro.states[i] for i in ids], ro.actions[ids], r.adv[ids],
                              r.ret[ids], r.fixed[ids], ro.exps[ids])
        want[k] = (x["grad"], [x["loss"], x["value_loss"], x["surr_loss"], x["entropy_loss"]])
    check_sampled(r, want)


# ---- d. the instrumentation changes nothing --------------------------------------------------------------------------
def assert_same_iteration(a, b, what, steps_too=True):
    assert np.array_equal(a.params, b.params), what
    assert np.array_equal(a.m, b.m) and np.array_equal(a.v, b.v), what
    assert a.steps.tolist() == b.steps.tolist(), (what, a.steps.tolist(), b.steps.tolist())
    key = (lambda x: x) if steps_too else (lambda x: x[:2])
    la, lb = [key(x) for x in a.logged], [key(x) for x in b.logged]
    assert len(la) == len(lb) and la == lb, (what, next((x, y) for x, y in zip(la, lb) if x != y) if la != lb else None)
    assert {k: np.asarray(v).tolist() for k, v in a.out.items()} == {k: np.asarray(v).tolist() for k, v in b.out.items()}


def test_sgnn_instrumentation_changes_nothing(dev, sgnn):
    plain = run(dev, sgnn.ro, PL.default_init(21))
    assert_same_iteration(sgnn, plain, "wrapped against plain")


# ---- e. consecutive iterations ---------------------------------------------------------------------------------------
def test_sgnn_consecutive_iterations_match_fresh_updaters(dev, pool):
    """25,000, then 6,561 (three 2,048-state chunks and a tail; 25 minibatches), then 25,000 states on one updater with
    diagnostics on, so the pinned and device blob buffers, the ring and the diagnostics read-back are reused after a
    larger and after a smaller iteration.  Each iteration is bit-identical to a fresh updater loaded with the
    previous parameters and Adam state (the first-step clip not re-armed); a fresh updater starts its own TensorBoard
    step count, so the step indices of the per-minibatch tags are left out."""
    states, _ = pool
    flat = PL.default_init(31)
    chained = updater(dev, flat, diagnostics=True)
    params, opt = flat, None
    for it, (n, seed) in enumerate([(T, 31), (6561, 32), (T, 33)]):
        ro = SC.Rollout(states, n, seed)
        fresh = updater(dev, params, diagnostics=True)
        if opt is not None:
            fresh.engine.set_opt_state(*opt, rearm_first_step_clip=False)
        res = []
        for up in (chained, fresh):
            logged = []
            np.random.seed(100 + it)
            out = up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps, iteration=it,
                                   log_fn=lambda tag, v, s: logged.append((tag, v, s)))
            torch.cuda.synchronize()
            m, v, steps = up.engine.get_opt_state()
            res.append(types.SimpleNamespace(params=up.flat_params(), m=m, v=v, steps=steps, out=out,
                                             logged=[x if x[0].startswith(("loss/epoch", "loss/total", "diag/total"))
                                                     else x[:2] for x in logged]))
        assert res[0].steps[0] == EPOCHS * sum(x // B for x in [T, 6561, T][:it + 1])
        assert_same_iteration(res[0], res[1], f"iteration {it} ({n} states)")
        params, opt = res[0].params, (res[0].m, res[0].v, res[0].steps)
        del fresh


# ---- f. every option on at once (SGNN) -------------------------------------------------------------------------------
def test_sgnn_every_option_at_scale(dev, rollout):
    ro = rollout
    so = PL.NUM_PARAMS + 3                                    # UPB_STAT_OFFSET
    r = run(dev, ro, PL.default_init(22), sampled(ro, seed=4), **ALL_OPTIONS)
    assert r.up.engine.stat_offset == so
    rec = r.rec
    orders = SC.epoch_orders(NP_SEED, T)
    stats = np.array([b[so:so + 20].cpu().numpy() for b in rec.bufs], np.float64)
    assert not stats[:, NONFINITE_SLOT].any() and r.out["nonfinite_skips"] == 0
    for e in range(EPOCHS):                                   # each epoch's normalised advantages
        # the stepped graphs only: the 168 remainder graphs of an epoch are never read, and after epoch 0 they keep
        # the values the epoch before normalised
        stepped = orders[e][:NB * B]
        want = VO.normalize64(r.adv, ro.exps, orders[e], B)[stepped]
        got = rec.norm_adv[e][stepped]
        assert np.array_equal(got, want) or np.abs(got - want).max() <= 2 * np.spacing(np.abs(want).max()), e
    beta = 0.1
    last = stats[(EPOCHS - 1) * NB:]
    assert r.out["kl_coef_next"] == adapt_kl_coef(beta, last[:, KLPEN_SLOT].sum(), last[:, 4].sum(), 0.01)
    assert r.steps.tolist()[:2] == [EPOCHS * NB] * 2
    lp_old = [lp for lp, _ in KO.per_graph(r.up.old_cand_log_probs.cpu().numpy(), r.up.blob)]
    ks = sorted(rec.before)
    res = SC.run_steps(SC._options_step, [(rec.before[k][0], rec.ids[k], rec.norm_adv[k // NB]) for k in ks],
                       states=ro.states, actions=ro.actions, ret=r.ret, fixed=r.fixed, exps=ro.exps,
                       old_values=r.values, lp_old=lp_old, opts=dict(value_clip=float(np.float32(0.2)), kl_coef=beta))
    worst, failures = {}, []
    for k, x in zip(ks, res):
        row, bad = check_grad(r, k, x["grad"], worst)
        st = row[so:so + 20]
        n, ni = st[3], st[4]
        got = [st[1] / ni, st[VCLIP_LOSS_SLOT] / n, st[2] / ni, st[KLPEN_SLOT] / ni]
        bad += check_losses(got, [x["surr_sum"] / x["n_ind"], x["value_loss_sum"] / x["n"], x["ent_sum"] / x["n_ind"],
                                  x["kl_sum"] / x["n_ind"]], worst)
        if (n, ni) != (x["n"], x["n_ind"]):
            bad.append(f"counts {(n, ni)}")
        g, norm = GO.clip64(row[:PL.NUM_PARAMS], 0.5)
        worst["norm"] = max(worst.get("norm", 0.0), abs(st[GCLIP_NORM_SLOT] - norm) / norm)
        if not abs(st[GCLIP_NORM_SLOT] - norm) < 1e-6 * norm:
            bad.append(f"slot 17 {st[GCLIP_NORM_SLOT]} vs {norm}")
        bad += check_adam(r, k, g, worst, wd=1e-2)
        if bad:
            failures.append(f"step {k} (epoch {k // NB}, minibatch {k % NB}): " + "; ".join(bad))
    report(f"every option, sampled steps {ks}", worst)
    assert not failures, "\n".join(failures)
