"""GPU: the training options together, both models, against float64 at the product's scale.  Builders and composed
oracles in tests/combined_cases.py; the worst errors are printed (pytest -s).

1. rl-mlp with every PPO option (test_gpu_update_scale.ALL_OPTIONS: the global clip, weight decay, clipped value loss,
   advantage normalisation, the adaptive KL penalty, the guard, diagnostics) on 25,000 HLG states: each epoch's
   normalised advantages, kl_coef_next, the counters, and 17 teacher-forced sampled steps against
   ppo_oracle.mlp_minibatch (gradient, the statistics sums of slots 1, 2, 15 and 18, slot 17, Adam).
   The rl-mlp fused rows are not run-to-run reproducible on land-use graphs, so nothing here is bit for bit.
2. Parameter groups, value normalisation (beta 0.9) and live schedules with every option, one PPOUpdater per model,
   three updates of 25,000, 6,561 and 25,000 states with rewards scaled and shifted per update.  Every tensor has its
   own group (lr, weight decay), three tensors that are not a prefix are frozen and one of them is trained again from
   the second update; each group's lr and clip_epsilon, value_pred_coef and entropy_coef change between updates; the
   third update carries one +inf reward.  The KL coefficient starts at 0.5 and a fifth of exps are 0, so that the
   penalty's gradient, and its 1 / |ind| against 1 / n, shows well above the gradient bar.  Per update:
     a. the value-norm call against vnorm_oracle (state, rescaled head, normalised returns and old values), and on the
        poisoned update state and head unchanged;
     b. every step on the host: frozen columns 0 in every ring row, each tensor's count against the host model, slot 19
        exactly on the minibatches that hold a non-finite sample (found by GAE per episode), nonfinite_skips and
        kl_coef_next;
     c. about 17 sampled steps plus the first steps after the unfreeze, teacher forced: gradient, losses, slot 17 over
        the trained columns, frozen tensors unchanged bit for bit, and each trained element's Adam step (parameter,
        first and second moment) against float64 with its own lr, weight decay and count (combined_cases.elem_excess,
        elem_excess_v).
3. The same three updates at 2,048 states through use_b200_update(param_groups=True, value_norm=True) with a per-group
   LambdaLR on agent.optimizer, requires_grad_ flags and agent coefficient assignments are bit for bit the PPOUpdater
   driven by explicit calls."""
import time
import types
import warnings

import numpy as np
import pytest
import torch

import combined_cases as CC
import gclip_oracle as GO
import klpen_oracle as KO
import ppo_oracle as PPO
import scale_cases as SC
import vclip_oracle as VO
import vnorm_oracle as VN
from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.agent import use_b200_update
from drl_urban_planning_b200.engine import adapt_kl_coef
from drl_urban_planning_b200.ppo import GCLIP_NORM_SLOT, KLPEN_SLOT, NONFINITE_SLOT, VCLIP_LOSS_SLOT, PPOUpdater
from harness import dev, rel, tensor_errors  # noqa: F401  (dev: fixture)
from shape_cases import SPEC
from test_gpu_live_hyperparams import E_CAP as SMALL_E, N_CAP as SMALL_N, make_agent
from test_gpu_update_scale import ALL_OPTIONS, GRAD_BAR, V_BAR, check_adam, check_grad, check_losses
from test_gpu_value_norm import Capture, check_update_call, head

pytestmark = pytest.mark.gpu

B, EPOCHS, NP_SEED = SC.B, SC.EPOCHS, 5
BETA_VN = 0.9
VCLIP = float(np.float32(ALL_OPTIONS["value_clip"]))
MAX_NORM = ALL_OPTIONS["max_grad_norm"]
OPTIONS = {k: v for k, v in ALL_OPTIONS.items() if k != "weight_decay"}      # the groups carry the weight decay
# the three updates: a larger KL coefficient and a fifth of exps 0, so that the penalty's gradient, and its 1 / |ind|
# against 1 / n, is well above the gradient bar
COMBINED = dict(OPTIONS, kl_coef=0.5)
EXPS_ZERO = 0.2


def report(what, worst):
    print(f"\n[combined] {what}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.fixture(scope="module")
def pool():
    return SC.make_pool()


@pytest.fixture(scope="module", autouse=True)
def timing():
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    yield
    free, total = torch.cuda.mem_get_info()
    print(f"\n[combined] module wall time {time.time() - t0:.0f} s, peak of torch's allocator "
          f"{torch.cuda.max_memory_allocated() / 2 ** 20:.0f} MiB, device memory in use at the end "
          f"{(total - free) / 2 ** 20:.0f} MiB")


def stats_of(rec, so):
    return np.array([b[so:so + 20].cpu().numpy() for b in rec.bufs], np.float64)


def lp_old_of(up):
    return [lp for lp, _ in KO.per_graph(up.old_cand_log_probs.cpu().numpy(), up.blob)]


def oracle_losses(st, x):
    """(got, want) of the four per-minibatch means: surrogate, clipped value loss, entropy, KL."""
    n, ni = st[3], st[4]
    return ([st[1] / ni, st[VCLIP_LOSS_SLOT] / n, st[2] / ni, st[KLPEN_SLOT] / ni],
            [x["surr_sum"] / x["n_ind"], x["value_loss_sum"] / x["n"], x["ent_sum"] / x["n_ind"],
             x["kl_sum"] / x["n_ind"]])


def check_norm(st, row, n_params, worst):
    norm = GO.clip64(row[:n_params], MAX_NORM)[1]
    e = abs(st[GCLIP_NORM_SLOT] - norm) / norm
    worst["slot17"] = max(worst.get("slot17", 0.0), e)
    return [] if e < 1e-6 else [f"slot 17 {st[GCLIP_NORM_SLOT]} vs {norm}"]


# ---- 1. rl-mlp with every PPO option at scale -------------------------------------------------------------------------
def test_mlp_every_option_at_scale(dev, pool):
    states, _ = pool
    ro = SC.Rollout(states, SC.T_PRODUCT, seed=21)
    nb = ro.T // B
    orders = SC.epoch_orders(NP_SEED, ro.T)
    up = PPOUpdater(PL.MLP.default_init(22), SPEC.max_num_nodes, SPEC.max_num_edges, dev, gamma=SC.GAMMA, tau=SC.TAU,
                    opt_num_epochs=EPOCHS, mini_batch_size=B, model="mlp", process_group=None, **ALL_OPTIONS)
    rec = SC.Recorder(up, SC.sample_steps(orders, ro.big_pos, nb, 4), nb)
    np.random.seed(NP_SEED)
    out = up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps)
    torch.cuda.synchronize()
    so = up.engine.stat_offset
    r = types.SimpleNamespace(up=up, rec=rec, ro=ro, stage=up.blob.info[:, 3].astype(np.int64))
    stats = stats_of(rec, so)
    assert not stats[:, NONFINITE_SLOT].any() and out["nonfinite_skips"] == 0
    adv = up.advantages.cpu().numpy()
    for e in range(EPOCHS):
        stepped = orders[e][:nb * B]
        want = VO.normalize64(adv, ro.exps, orders[e], B)[stepped]
        got = rec.norm_adv[e][stepped]
        assert np.array_equal(got, want) or np.abs(got - want).max() <= 2 * np.spacing(np.abs(want).max()), e
    last = stats[(EPOCHS - 1) * nb:]
    assert out["kl_coef_next"] == adapt_kl_coef(0.1, last[:, KLPEN_SLOT].sum(), last[:, 4].sum(), 0.01)
    assert up.engine.get_opt_state()[2].tolist()[:2] == [EPOCHS * nb] * 2
    lp_old = lp_old_of(up)
    ret, old_v, fixed = (x.cpu().numpy() for x in (up.returns, up.old_values, up.fixed_log_probs))
    worst, failures = {}, []
    for k in sorted(rec.before):
        ids = rec.ids[k]
        x = PPO.mlp_minibatch(rec.before[k][0], [ro.states[i] for i in ids], ro.actions[ids],
                              rec.norm_adv[k // nb][ids], ret[ids], fixed[ids], ro.exps[ids], old_values=old_v[ids],
                              lp_old=[lp_old[i] for i in ids], value_clip=VCLIP, kl_coef=0.1)
        row, bad = check_grad(r, k, x["grad"], worst)
        st = row[so:so + 20]
        bad += check_losses(*oracle_losses(st, x), worst)
        if (st[3], st[4]) != (x["n"], x["n_ind"]):
            bad.append(f"counts {(st[3], st[4])}")
        bad += check_norm(st, row, PL.MLP.num_params, worst)
        bad += check_adam(r, k, GO.clip64(row[:PL.MLP.num_params], MAX_NORM)[0], worst, wd=1e-2)
        if bad:
            failures.append(f"step {k} (epoch {k // nb}, minibatch {k % nb}): " + "; ".join(bad))
    report(f"rl-mlp every option, sampled steps {sorted(rec.before)}", worst)
    assert not failures, "\n".join(failures)


# ---- 2. groups, value normalisation and live schedules with every option, three updates -------------------------------
def combined_run(dev, states, model):
    """The three updates of combined_cases.UPDATES on one PPOUpdater; per update what the checks need."""
    layout = CC.layout_of(model)
    flat = PL.MLP.default_init(23) if model == "mlp" else PL.default_init(23)
    up = PPOUpdater(flat, SPEC.max_num_nodes, SPEC.max_num_edges, dev, gamma=SC.GAMMA, tau=SC.TAU,
                    opt_num_epochs=EPOCHS, mini_batch_size=B, model=model, process_group=None, param_groups=True,
                    value_norm=True, value_norm_beta=BETA_VN, **COMBINED)
    cap = Capture(up)
    runs = []
    for it, (n, seed, scale, shift) in enumerate(CC.UPDATES):
        ro = CC.thin_exps(CC.scaled(SC.Rollout(states, n, seed), scale, shift), EXPS_ZERO, seed)
        pos = CC.poison(ro) if it == 2 else None
        up.set_param_groups(CC.groups_at(model, it))
        if it:
            up.set_hyperparameters(**CC.COEFS[it])
        beta = up.kl_coef
        nb = n // B
        orders = SC.epoch_orders(NP_SEED + it, n)
        sample = set(SC.sample_steps(orders, ro.big_pos, nb, seed))
        if it == 1:
            sample |= {0, 1, 2}                    # the unfrozen tensor's first steps
        rec = CC.Recorder(up, sorted(sample), nb)
        np.random.seed(NP_SEED + it)
        out = up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps, iteration=it)
        torch.cuda.synchronize()
        up.minibatch_step = rec.inner
        call = cap.calls[-1]
        runs.append(types.SimpleNamespace(
            it=it, ro=ro, pos=pos, nb=nb, rec=rec, out=out, call=call, beta=beta, table=CC.table(model, it),
            coefs=CC.kernel_coefs(it), stage=up.blob.info[:, 3].astype(np.int64), lp_old=lp_old_of(up),
            adv=up.advantages.cpu().numpy(), fixed=up.fixed_log_probs.cpu().numpy(),
            stats=stats_of(rec, up.engine.stat_offset), so=up.engine.stat_offset))
        assert len(rec.ids) == EPOCHS * nb
    return types.SimpleNamespace(up=up, layout=layout, model=model, runs=runs)


_RUNS = {}


@pytest.fixture(scope="module", params=["sgnn", "mlp"])
def combined(request, dev, pool):
    if request.param not in _RUNS:
        _RUNS.clear()                                  # one model's records at a time
        _RUNS[request.param] = combined_run(dev, pool[0], request.param)
    return _RUNS[request.param]


def test_value_norm_call_of_every_update(combined):
    c = combined
    for r in c.runs:
        call = r.call
        check_update_call(call, c.layout, BETA_VN)
        if r.pos is None:
            assert call["new_state"] != call["state"], r.it
        else:                                          # the poisoned update: nothing moves
            assert call["new_state"] == call["state"], r.it
            w0, b0 = head(c.layout, call["params"])
            w1, b1 = head(c.layout, call["new_params"])
            assert np.array_equal(w0, w1) and b0 == b1, r.it
        assert (r.out["value_norm_mean"], r.out["value_norm_std"]) == VN.stats(*call["new_state"]), r.it
    assert abs(c.runs[1].out["value_norm_mean"]) > 1.0        # away from the identity


def test_every_step_on_the_host(combined):
    c = combined
    seg = CC.seg_of(c.layout)
    n_params = c.layout.num_params
    for r in c.runs:
        rec, ro = r.rec, r.ro
        lr, wd, trained = r.table
        frozen_cols = ~CC.entry_table(c.layout, trained)
        bad_pos = CC.nonfinite_positions(ro.rewards, ro.masks, r.call["values"], SC.GAMMA, SC.TAU)
        assert bad_pos.tolist() == ([] if r.pos is None else [r.pos]), (r.it, bad_pos[:8])
        # k_gae scans each episode on its own: the kernel's advantages are the per-episode scan's, bit for bit
        with np.errstate(invalid="ignore", over="ignore"):
            want_adv, _ = CC.gae_per_episode(ro.rewards, ro.masks, r.call["values"], SC.GAMMA, SC.TAU)
        assert np.array_equal(r.adv, want_adv, equal_nan=True), r.it
        counts = rec.tsteps[0]
        skipped_want = []
        for k, ids in enumerate(rec.ids):
            row = rec.bufs[k].cpu().numpy()
            assert not row[:n_params][frozen_cols].any(), (r.it, k)
            skipped = bool(np.isin(ids, bad_pos).any())
            skipped_want.append(skipped)
            assert (r.stats[k, NONFINITE_SLOT] == 1.0) == skipped, (r.it, k)
            counts = CC.next_counts(counts, trained, seg, r.stage[ids], skipped)
            assert rec.tsteps[k + 1].tolist() == counts.tolist(), (r.it, k, rec.tsteps[k + 1].tolist(), counts.tolist())
        assert r.out["nonfinite_skips"] == sum(skipped_want), r.it
        assert (r.pos is None) == (sum(skipped_want) == 0), r.it
        kept = r.stats[(EPOCHS - 1) * r.nb:][~np.array(skipped_want[(EPOCHS - 1) * r.nb:])]
        assert r.out["kl_coef_next"] == adapt_kl_coef(r.beta, kept[:, KLPEN_SLOT].sum(), kept[:, 4].sum(),
                                                      ALL_OPTIONS["kl_target"]), r.it
        assert np.isfinite(r.out["total_loss"]), r.it


# A bias sums its layer's per-node or per-candidate gradients with no feature weight, and late in these updates those
# sums can cancel (each graph's logit gradients sum to 0, and the KL seed p - p_old is a difference of nearly equal fp32
# numbers).  Where a bias misses the bar on its own scale and its gradient is smaller than its layer's weight gradient
# (the cancellation shown), its fp32 rounding is measured against the size of its terms, that weight gradient; how much
# looser this makes the bar (max |weight grad| / max |bias grad|) is recorded per bias and printed.
def terms_of(layout):
    """bias slot -> the weight slot of the same layer (x_b -> x_w, x_bN -> x_wN)."""
    out = {}
    for name in layout.slots:
        w = name.replace("_b", "_w", 1) if "_b" in name else None
        if w in layout.slots:
            out[name] = w
    return out


def check_grad_terms(layout, rec, k, want, worst, loosened):
    row = rec.bufs[k].cpu().numpy().astype(np.float64)
    got = row[:layout.num_params]
    errs = tensor_errors(got, want, layout)
    for b, w in terms_of(layout).items():
        if errs[b] < GRAD_BAR:
            continue
        sb, sw = layout.slots[b], layout.slots[w]
        wb = np.abs(want[sb.offset:sb.offset + sb.size]).max()
        ww = np.abs(want[sw.offset:sw.offset + sw.size]).max()
        if ww <= wb:
            continue
        d = np.abs(got[sb.offset:sb.offset + sb.size] - want[sb.offset:sb.offset + sb.size]).max()
        errs[b] = float(d / ww)
        loosened[b] = max(loosened.get(b, 0.0), float(ww / max(wb, 1e-30)))
    name = max(errs, key=errs.get)
    worst["grad"] = max(worst.get("grad", 0.0), errs[name])
    return row, ([f"gradient {name} {errs[name]:.3g}"] if not errs[name] < GRAD_BAR else [])


def sampled_oracles(c, r, ks):
    """The float64 minibatch of every sampled step k in ks (not skipped), from the kernel's own state and inputs."""
    rec, ro, call = r.rec, r.ro, r.call
    opts = dict(value_clip=VCLIP, kl_coef=float(np.float32(r.beta)), **r.coefs)
    if c.model == "sgnn":
        return SC.run_steps(SC._options_step, [(rec.before[k][0], rec.ids[k], rec.norm_adv[k // r.nb]) for k in ks],
                            states=ro.states, actions=ro.actions, ret=call["norm_returns"], fixed=r.fixed,
                            exps=ro.exps, old_values=call["norm_values"], lp_old=r.lp_old, opts=opts)
    out = []
    for k in ks:
        ids = rec.ids[k]
        out.append(PPO.mlp_minibatch(
            rec.before[k][0], [ro.states[i] for i in ids], ro.actions[ids], rec.norm_adv[k // r.nb][ids],
            call["norm_returns"][ids], r.fixed[ids], ro.exps[ids], old_values=call["norm_values"][ids],
            lp_old=[r.lp_old[i] for i in ids], **opts))
    return out


def test_sampled_steps_teacher_forced(combined):
    c = combined
    layout, n_params = c.layout, c.layout.num_params
    seg = CC.seg_of(layout)
    worst, failures, loosened = {}, [], {}
    for r in c.runs:
        rec = r.rec
        lr, wd, trained = r.table
        lr_e, wd_e, trained_e = (CC.entry_table(layout, x) for x in (lr, wd, trained))
        bad_pos = [] if r.pos is None else [r.pos]
        ks = sorted(rec.before)
        skipped = {k for k in ks if np.isin(rec.ids[k], bad_pos).any()}
        live_ks = [k for k in ks if k not in skipped]
        for k in skipped:                                  # a skipped step moves nothing
            p0, m0, v0, s0 = rec.before[k]
            p1, m1, v1, s1 = rec.after[k]
            assert np.array_equal(p0, p1) and np.array_equal(m0, m1) and np.array_equal(v0, v1), (r.it, k)
            assert s0.tolist() == s1.tolist() and rec.tsteps[k].tolist() == rec.tsteps[k + 1].tolist(), (r.it, k)
        for k, x in zip(live_ks, sampled_oracles(c, r, live_ks)):
            want_grad = np.where(trained_e, x["grad"], 0.0)
            row, bad = check_grad_terms(layout, rec, k, want_grad, worst, loosened)
            st = row[r.so:r.so + 20]
            bad += check_losses(*oracle_losses(st, x), worst)
            bad += check_norm(st, row, n_params, worst)
            p0, m0, v0, _ = rec.before[k]
            p1, m1, v1, _ = rec.after[k]
            t0, t1 = rec.tsteps[k], rec.tsteps[k + 1]
            if not (np.array_equal(p0[~trained_e], p1[~trained_e]) and np.array_equal(m0[~trained_e], m1[~trained_e])
                    and np.array_equal(v0[~trained_e], v1[~trained_e]) and (t0[~trained] == t1[~trained]).all()):
                bad.append("a frozen tensor moved")
            stages = r.stage[rec.ids[k]]
            live = SC.live_entries(stages, layout) & trained_e
            g = GO.clip64(row[:n_params], MAX_NORM)[0]
            want = CC.adam_want((p0, m0, v0), g, live, lr_e, wd_e, CC.entry_table(layout, t0).astype(np.float64))
            want_p = CC.param_step_want(p0, m1, v1, CC.entry_table(layout, t0), live, lr_e)
            for name, got1, got0, w in (("params", p1, p0, want_p), ("m", m1, m0, want[1])):
                ex = CC.elem_excess(got1[live], got0[live], w[live])
                worst[name + " (x bar)"] = max(worst.get(name + " (x bar)", 0.0), float(ex.max()))
                if ex.max() > 1:
                    j = np.flatnonzero(live)[int(ex.argmax())]
                    tensor = next(s.name for s in layout.slots.values() if s.offset <= j < s.offset + s.size)
                    bad.append(f"{name}[{j}] ({tensor}) {ex.max():.3g} x the bar")
            # v element by element: V_BAR of the element (the second moment's weight, see V_BAR) and 2 ulp
            ev = CC.elem_excess_v(v1[live], want[2][live], V_BAR)
            worst["v (x bar)"] = max(worst.get("v (x bar)", 0.0), float(ev.max()))
            if ev.max() > 1:
                bad.append(f"v[{np.flatnonzero(live)[int(ev.argmax())]}] {ev.max():.3g} x the bar")
            if t1.tolist() != CC.next_counts(t0, trained, seg, stages, False).tolist():
                bad.append(f"counts {t0.tolist()} -> {t1.tolist()}")
            if bad:
                failures.append(f"update {r.it} step {k} (epoch {k // r.nb}, minibatch {k % r.nb}): " + "; ".join(bad))
    report(f"{c.model} groups + value_norm + live values, sampled steps of 3 updates", worst)
    report(f"{c.model} bias bars loosened by (max |weight grad| / max |bias grad|)", loosened)
    assert not failures, "\n".join(failures)


# ---- 3. the agent path, bit for bit -----------------------------------------------------------------------------------
AGENT_T, AGENT_B, AGENT_EPOCHS = 2048, 256, 2


def agent_rollouts():
    out = []
    for it, (_, seed, scale, shift) in enumerate(CC.UPDATES):
        ro = CC.small_rollout(seed, AGENT_T, scale, shift)
        if it == 2:
            CC.poison(ro)
        out.append(ro)
    return out


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_agent_path_is_bit_identical(dev, model):
    layout = CC.layout_of(model)
    names = list(layout.slots)
    flat = PL.MLP.default_init(24) if model == "mlp" else PL.default_init(24)
    logs = [[], []]
    ag = make_agent(model, dev, flat, logs[0], num_optim_epoch=AGENT_EPOCHS, mini_batch_size=AGENT_B)
    by_slot = {}
    for key, p in ag.actor_critic_net.named_parameters():
        by_slot[next(sl.name for sl in layout.slots.values() if PL.state_dict_keys(sl)[0] == key)] = p
    ag.optimizer = torch.optim.Adam([dict(params=[by_slot[n]], lr=CC.base_lr(k), weight_decay=CC.base_wd(k))
                                     for k, n in enumerate(names)], eps=ag.cfg.eps)
    sched = torch.optim.lr_scheduler.LambdaLR(ag.optimizer, [CC.lr_lambda(k) for k in range(len(names))])
    ctl = use_b200_update(ag, param_groups=True, value_norm=True, value_norm_beta=BETA_VN, **OPTIONS)
    cfg = ag.cfg
    up = PPOUpdater(flat, SMALL_N, SMALL_E, dev, lr=cfg.lr, eps=cfg.eps, clip_epsilon=cfg.clip_epsilon,
                    value_pred_coef=cfg.value_pred_coef, entropy_coef=cfg.entropy_coef, gamma=cfg.gamma, tau=cfg.tau,
                    opt_num_epochs=AGENT_EPOCHS, mini_batch_size=AGENT_B, model=model, process_group=None,
                    param_groups=True, value_norm=True, value_norm_beta=BETA_VN, **OPTIONS)
    for it, ro in enumerate(agent_rollouts()):
        frozen = CC.frozen_at(model, it)
        for n, p in by_slot.items():
            p.requires_grad_(n not in frozen)
        if it:
            for k, v in CC.COEFS[it].items():
                setattr(ag, k, v)
            up.set_hyperparameters(**CC.COEFS[it])
        up.set_param_groups(CC.groups_at(model, it))
        np.random.seed(90 + it)
        ag.update_params(ro, it)
        np.random.seed(90 + it)
        up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps, iteration=it,
                         log_fn=lambda tag, v, s: logs[1].append((tag, v, s)))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")       # the agent's optimizer never steps: the H100 path trains
            sched.step()
        torch.cuda.synchronize()
        a, b = ctl.updater, up
        assert a.engine.param_groups == b.engine.param_groups, it
        assert np.array_equal(a.flat_params(), b.flat_params()), it
        for x, y in zip(a.engine.get_opt_state(), b.engine.get_opt_state()):
            assert np.array_equal(x, y), it
        assert a.engine.get_tensor_steps().tolist() == b.engine.get_tensor_steps().tolist(), it
        assert a.engine.get_value_norm_state() == b.engine.get_value_norm_state(), it
        assert logs[0] == logs[1], it
        assert np.array_equal(layout.from_state_dict(ag.actor_critic_net.state_dict()), b.flat_params()), it
    ts = up.engine.get_tensor_steps()
    unfrozen = names.index(CC.FROZEN[model][0])
    assert 0 < ts[unfrozen] < ts[unfrozen - 1]                  # trained again, behind its neighbour
    assert any(tag == "diag/nonfinite_skips" and v > 0 for tag, v, _ in logs[1])
