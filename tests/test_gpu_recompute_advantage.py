"""GPU (H100): advantages recomputed before every PPO epoch (`recompute_advantage`).

- The value-only sweep (Engine.values, upb_values / upb_mlp_values) equals Engine.forward(...)[0] bit for bit on both
  models: the HLG, DHM and mixed goldens, the concept caps (1,500 / 4,000: the global-scratch path), the saturated
  goldens (tier-2 pulls) and empty masks.  The value path has no atomics in either model (the rl-mlp atomics that make
  harness.reproducible_states necessary are in the backward), so the forward's run-to-run spread of the value is zero:
  asserted below by two forwards, and the comparison is exact.
- The targets launch (Engine.gae_targets): without value normalisation Engine.gae bit for bit; with it, the fp32
  denormalisation, k_gae and the fp32 normalisation composed (bit for bit) and tests/recompute_oracle.py (float64).
- Exact where it must be: the option off or one epoch changes nothing, launch count included; with the encoder and
  the value head frozen the targets cannot move, so an update with the option on is bit-identical to one without.
- At the kernel's own state: a 3-epoch update on combined_cases.small_rollout, the parameters snapshotted before every
  sweep, checked against the float64 values and GAE at those parameters, and sampled steps of epochs 1 and 2 against the
  float64 step on the targets they trained on."""
import numpy as np
import pytest
import torch

import cap_cases as CC
import combined_cases as CB
import ppo_oracle as PPO
import recompute_oracle as RO
import vnorm_oracle as VN
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from drl_urban_planning_b200.ppo import PPOUpdater
from fixtures_io import expand_states, synth_states
from harness import dev, load, per_tensor_rel, rel, t  # noqa: F401
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON

pytestmark = pytest.mark.gpu

GRAD_BAR = 1e-4                 # tests/test_gpu_update_scale.py's gradient bar
TARGET_BAR = 1e-5               # max|got - want| / max|want| of the values and targets against float64
SGNN_CASES = ["hlg", "hlg256", "dhm256", "small_mixed", "concept_mixed256", "edge_empty", "extreme_tanh",
              "extreme_clamp", "extreme_attention", "extreme_heads", "caps_concept", "concept"]
MLP_CASES = ["mlp_hlg", "mlp_small", "mlp_extreme_tanh", "mlp_extreme_heads", "mlp_caps_concept", "dhm256",
             "concept_mixed256", "edge_empty", "extreme_clamp"]
CASES = [("sgnn", n) for n in SGNN_CASES] + [("mlp", n) for n in MLP_CASES] + [("sgnn", "concept_caps"),
                                                                                ("mlp", "concept_caps")]


def layout(model):
    return PL.MLP if model == "mlp" else PL.SGNN


def case_inputs(golden_dir, model, name):
    """(states, actions, flat parameters) of a golden fixture, or of cap_cases' concept-cap batch; the fixture's own
    parameters when they belong to `model`, else the model's seeded initialisation."""
    if name == "concept_caps":
        states, actions, _ = CC.concept_batch()
        flat = None
    else:
        z = load(golden_dir, name)
        if "digest" in z.files:
            states, actions = synth_states(int(z["seed"]), str(z["community"]), int(z["count"]))
        else:
            states, actions = expand_states(z), np.asarray(z["actions"], np.float32)
        flat = np.asarray(z["params"], np.float32) if z["params"].size == layout(model).num_params else None
    if flat is None:
        flat = PL.MLP.default_init(5) if model == "mlp" else PL.default_init(5)
    return states, np.asarray(actions, np.float32), flat


@pytest.mark.parametrize("model,name", CASES)
def test_values_equal_the_forward_bit_for_bit(model, name, golden_dir, dev):
    states, actions, flat = case_inputs(golden_dir, model, name)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, model=model)
    p = t(flat, dev)
    want = eng.forward(blob, p, t(actions, dev))[0]
    again = eng.forward(blob, p, t(actions, dev))[0]
    assert torch.equal(want, again), "the forward's value is not reproducible run to run"
    n0 = eng.launches
    got = eng.values(blob, p)
    assert eng.launches == n0 + 1
    torch.cuda.synchronize()
    w, g = want.cpu().numpy(), got.cpu().numpy()
    assert np.isfinite(w).all()
    assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), f"{int((g != w).sum())} of {g.size} values differ"
    # a subset in another order: the listed graphs get their values, the others keep `out`
    sel = np.arange(blob.count)[::-3][: max(1, blob.count // 2)]
    out = torch.full((blob.count,), 7.0, device=dev)
    eng.values(blob, p, ids=t(sel.astype(np.int32), dev), out=out)
    o = out.cpu().numpy()
    assert np.array_equal(o[sel], w[sel])
    rest = np.setdiff1d(np.arange(blob.count), sel)
    assert (o[rest] == 7.0).all()


def episodes_rollout(seed, T):
    rng = np.random.default_rng(seed)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 40, replace=False)] = 0.0
    rewards = (rng.standard_normal(T) * 30.0 + 200.0).astype(np.float32)
    head = (rng.standard_normal(T) * 2.0).astype(np.float32)
    return rewards, masks, head


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
@pytest.mark.parametrize("gamma,tau", [(1.0, 0.0), (0.99, 0.95)])
def test_gae_targets(model, gamma, tau, dev):
    T = 25000
    rewards, masks, head = episodes_rollout(11, T)
    r, m, n = (t(x, dev) for x in (rewards, masks, head))
    eng = Engine(dev, 64, 64, model=model)
    adv, ret, anchor = eng.gae_targets(r, m, n, gamma, tau)
    a0, r0 = eng.gae(r, m, n, gamma, tau)
    assert torch.equal(adv, a0) and torch.equal(ret, r0) and torch.equal(anchor, n)
    want = RO.targets(rewards, masks, head, gamma, tau)
    assert rel(adv.cpu().numpy(), want[0]) < TARGET_BAR and rel(ret.cpu().numpy(), want[1]) < TARGET_BAR

    eng_v = Engine(dev, 64, 64, model=model, value_norm=True)
    moved = VN.update((0.0, 0.0, 0.0), rewards, 0.99)
    for state in [(0.0, 0.0, 0.0), moved]:
        eng_v.set_value_norm_state(state)
        adv, ret, anchor = eng_v.gae_targets(r, m, n, gamma, tau)
        values = VN.denormalize(head, state)
        a1, r1 = eng.gae(r, m, t(values, dev), gamma, tau)
        norm = VN.normalize(r1.cpu().numpy(), VN.stats(*state))
        assert torch.equal(adv, a1) and torch.equal(anchor, n)
        assert np.array_equal(ret.cpu().numpy().view(np.uint32), norm.view(np.uint32))
        want = RO.targets(rewards, masks, head, gamma, tau, state)
        assert rel(adv.cpu().numpy(), want[0]) < TARGET_BAR and rel(ret.cpu().numpy(), want[1]) < TARGET_BAR
        assert eng_v.get_value_norm_state() == tuple(state), "the targets launch moved the statistics"


# ---- whole updates -----------------------------------------------------------------------------------------------------
SPEC = synth.COMMUNITIES["small"]


def flat_init(model, seed=3):
    return PL.MLP.default_init(seed) if model == "mlp" else PL.default_init(seed)


def run_update(dev, model, ro, epochs, seed=21, B=128, groups=None, **kw):
    up = PPOUpdater(flat_init(model), SPEC.max_num_nodes, SPEC.max_num_edges, dev, gamma=0.99, tau=0.95,
                    opt_num_epochs=epochs, mini_batch_size=B, model=model, clip_mode=_lib.CLIP_NEVER,
                    param_groups=groups is not None, **kw)
    if groups is not None:
        up.set_param_groups(groups)
    logged = []
    np.random.seed(seed)
    n0 = up.engine.launches
    out = up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps,
                           log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    torch.cuda.synchronize()
    m, v, steps = up.engine.get_opt_state()
    return dict(params=up.flat_params(), m=m, v=v, steps=steps, ring=up._grad_ring.cpu().numpy(), logged=logged,
                launches=up.engine.launches - n0, out=out)


def assert_same(a, b, launches=True):
    for k in ("params", "m", "v", "steps", "ring"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k
    assert a["logged"] == b["logged"]
    if launches:
        assert a["launches"] == b["launches"]


OPTIONS = [dict(), dict(value_norm=True), dict(value_clip=0.2, normalize_advantage=True),
           dict(value_norm=True, value_clip=0.2, normalize_advantage=True, diagnostics=True)]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_off_and_one_epoch_change_nothing(model, dev):
    ro = CB.small_rollout(31, 640, 5.0, 1.0)
    for kw in OPTIONS[::3]:
        plain = run_update(dev, model, ro, 3, **kw)
        assert_same(run_update(dev, model, ro, 3, recompute_advantage=False, **kw), plain)
        one = run_update(dev, model, ro, 1, **kw)
        assert_same(run_update(dev, model, ro, 1, recompute_advantage=True, **kw), one)
        on = run_update(dev, model, ro, 3, recompute_advantage=True, **kw)
        assert on["launches"] == plain["launches"] + 2 * 2        # a sweep and a targets launch after epochs 0 and 1
        assert not np.array_equal(on["params"], plain["params"])


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_frozen_value_path_makes_the_option_exact(model, dev):
    """The encoder and the value head frozen, the policy heads trained: the values cannot move between epochs, so the
    recomputed targets are the pre-pass ones bit for bit, and so is the whole update."""
    ro = CB.small_rollout(32, 640, 5.0, 1.0)
    heads = [s for s in layout(model).slots if s.startswith(("lu_", "road_"))]
    groups = [dict(params=heads, lr=4e-4)]
    for kw in (dict(), dict(value_clip=0.2, normalize_advantage=True)):
        off = run_update(dev, model, ro, 3, groups=groups, **kw)
        on = run_update(dev, model, ro, 3, groups=groups, recompute_advantage=True, **kw)
        assert_same(on, off, launches=False)
        assert on["launches"] == off["launches"] + 4


def oracle_head(model, flat, states):
    """float64 value head outputs at `flat`."""
    if model == "sgnn":
        T = len(states)
        z = np.zeros(T, np.float32)
        r = ON.ppo_minibatch(flat, states, np.zeros((T, 2), np.float32), z, z, z, np.ones(T, np.float32),
                             want_grad=False)
        return np.asarray(r["value"], np.float64)
    P = MP.params_from_flat(flat, dtype=torch.float64)
    out = []
    for a in range(0, len(states), 64):
        with torch.no_grad():
            out.append(MP.value(P, MP.stack_states(states[a:a + 64])).numpy().ravel())
    return np.concatenate(out)


def oracle_step_grad(model, flat, states, actions, adv, ret, fixed, exps):
    if model == "sgnn":
        return ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)["grad"]
    return PPO.mlp_minibatch(flat, states, actions, adv, ret, fixed, exps)["grad"]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
@pytest.mark.parametrize("opts", range(len(OPTIONS)))
def test_targets_and_steps_against_float64_at_the_kernels_state(model, opts, dev):
    kw = OPTIONS[opts]
    T, B, epochs = 512, 128, 3
    ro = CB.small_rollout(33 + opts, T, 5.0, 40.0)
    up = PPOUpdater(flat_init(model), SPEC.max_num_nodes, SPEC.max_num_edges, dev, gamma=0.99, tau=0.95,
                    opt_num_epochs=epochs, mini_batch_size=B, model=model, clip_mode=_lib.CLIP_NEVER,
                    recompute_advantage=True, **kw)
    sweeps, steps = [], []
    recompute, step = up.recompute_targets, up.minibatch_step

    def spy_recompute():
        p = up.params.clone()
        recompute()
        sweeps.append((p, up.advantages.clone(), up.returns.clone(),
                       up.old_values.clone() if up.value_clip is not None else None))

    def spy_step(ids, global_batch, global_ind):
        # the first and the last step of every epoch after the first: teacher-forced against float64
        k = len(steps)
        if k // (T // B) >= 1 and k % (T // B) in (0, T // B - 1) and "value_clip" not in kw:
            adv = up.norm_advantages if up.normalize_advantage else up.advantages
            steps.append((ids.clone(), up.params.clone(), adv.clone(), up.returns.clone()))
        else:
            steps.append(None)
        step(ids, global_batch, global_ind)
        if steps[-1] is not None:
            steps[-1] = steps[-1] + (up.grad.clone(),)

    up.recompute_targets, up.minibatch_step = spy_recompute, spy_step
    np.random.seed(7)
    up.update_params(ro.states, ro.actions, ro.rewards, ro.masks, ro.exps)
    torch.cuda.synchronize()
    assert len(sweeps) == epochs - 1
    state = up.engine.get_value_norm_state() if up.value_norm else None
    for k, (p, adv, ret, anchor) in enumerate(sweeps):
        head = oracle_head(model, p.cpu().numpy(), ro.states)
        want = RO.targets(ro.rewards, ro.masks, head, 0.99, 0.95, state)
        errs = dict(adv=rel(adv.cpu().numpy(), want[0]), ret=rel(ret.cpu().numpy(), want[1]))
        if anchor is not None:
            errs["anchor"] = rel(anchor.cpu().numpy(), want[2])
        print(f"{model} {kw} sweep {k}: {errs}")
        assert all(e < TARGET_BAR for e in errs.values()), errs
    fixed = up.fixed_log_probs.cpu().numpy()
    checked = 0
    for rec in steps:
        if rec is None:
            continue
        ids, p, adv, ret, grad = (x.cpu().numpy() for x in rec)
        sel = np.sort(ids)
        want = oracle_step_grad(model, p, [ro.states[i] for i in sel], ro.actions[sel], adv[sel], ret[sel],
                                fixed[sel].reshape(-1, 1), ro.exps[sel])
        e, where = per_tensor_rel(grad[:layout(model).num_params], want, layout(model))
        print(f"{model} {kw} step: gradient {e:.3g} ({where})")
        assert e < GRAD_BAR, (e, where)
        checked += 1
    assert checked == (0 if "value_clip" in kw else 2 * (epochs - 1))
