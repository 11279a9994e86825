"""GPU (H100): the gradient-noise measurement (upb_ppo_grad_noise, grad_noise_every), both models.

1. {A, S, Q, N} of one measurement against independent references: A from one ppo_grad launch per CTA group with the
   minibatch's global 1/B and 1/|ind|, S from the reduced row, both squared in float64; one graph per CTA and two or
   three.  On one small SGNN case, against per-graph gradients of the torch port too.
2. Frozen tensors (parameter groups) are absent from A and S; the KL stop word gives N = 0; identical calls give
   identical bits.
3. Training with the option on is bit-identical to training without it (parameters, moments, counts, statistics rows,
   losses, logged tags, np.random's state); the estimate counts exactly the measured steps that applied Adam."""
import numpy as np
import pytest
import torch

import grad_noise_oracle as GO
from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.agent import use_b200_update
from drl_urban_planning_b200.engine import cta_group_sizes, grad_noise_estimate, grad_noise_terms
from drl_urban_planning_b200.ppo import PPOUpdater
from harness import Case, dev, reproducible_states, t
from test_gpu_live_hyperparams import E_CAP, N_CAP, batch, flat_init, make_agent

pytestmark = pytest.mark.gpu

NOISE_KEYS = ("grad_noise_scale", "grad_noise_g2", "grad_noise_trace", "grad_noise_samples")


def mixed_case(dev, model, count, seed=4):
    """`count` land-use and road graphs in random order (harness.reproducible_states), two with exps = 0."""
    states, actions = reproducible_states(seed, count)
    return Case(dev, model, states, actions, seed, zero_exps=(3, 7))


def global_args(case):
    n_ind = int((case.exps != 0).sum())
    return case.dev_args + (1.0 / case.count, 1.0 / n_ind)


def measure(case, eng, params, order):
    g, noise = eng.ppo_grad_noise(case.blob, params, *global_args(case), ids=t(np.asarray(order, np.int32), case.dev))
    torch.cuda.synchronize()
    return g.cpu().numpy(), noise.cpu().numpy()


def trained_columns(eng):
    """Boolean mask of the real parameter columns the engine trains (every one without parameter groups)."""
    mask = np.ones(eng.num_params, bool)
    if eng.param_groups is not None:
        for k, sl in enumerate(eng.layout.slots.values()):
            mask[sl.offset:sl.offset + sl.size] = eng.param_groups[2][k]
    return mask


def reference_A(case, eng, params, order, mask):
    """sum over the launch's CTAs of the squared norm of that CTA group's gradient, one ppo_grad launch per group"""
    grid = min(case.count, eng.grid)
    A = 0.0
    for c in range(grid):
        sel = t(np.asarray(order[c::grid], np.int32), case.dev)
        g = eng.ppo_grad(case.blob, params, *global_args(case), ids=sel)
        torch.cuda.synchronize()
        x = g.cpu().numpy()[:eng.num_params].astype(np.float64)
        A += float(np.square(x[mask]).sum())
    return A


@pytest.mark.parametrize("count", [100, 300])       # one graph per CTA; two or three on 132 CTAs
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_values_against_independent_references(model, count, dev):
    case = mixed_case(dev, model, count)
    eng = case.engine()
    params = t(case.flat, dev)
    order = np.random.default_rng(count).permutation(count)
    g, (A, S, Q, N) = measure(case, eng, params, order)
    mask = trained_columns(eng)
    S_ref = float(np.square(g[:eng.num_params].astype(np.float64)).sum())
    A_ref = reference_A(case, eng, params, order, mask)
    sizes = cta_group_sizes(count, eng.grid)
    assert (Q, N) == (float(np.square(sizes).sum()), float(count))
    if count > eng.grid:
        assert set(sizes.tolist()) == {2, 3}
    assert abs(S / S_ref - 1.0) < 1e-5, (S, S_ref)
    assert abs(A / A_ref - 1.0) < 1e-5, (A, A_ref)
    # the measurement's gradient buffer is the ppo_grad of the same graphs
    g2 = eng.ppo_grad(case.blob, params, *global_args(case), ids=t(np.asarray(order, np.int32), dev))
    assert np.array_equal(g, g2.cpu().numpy())


def test_sgnn_against_per_graph_port_gradients(dev):
    count, grid = 12, 5                                 # groups of 3, 3, 2, 2, 2
    case = mixed_case(dev, "sgnn", count, seed=9)
    eng = case.engine(grid_limit=grid)
    assert eng.grid == grid
    order = np.random.default_rng(1).permutation(count)
    _, noise = measure(case, eng, t(case.flat, dev), order)
    x = GO.sgnn_graph_terms(case.flat, case.states, case.actions, case.adv, case.ret, case.fixed, case.exps)
    want = GO.measure(x[order], grid)
    assert noise[2:].tolist() == want[2:].tolist()
    assert np.allclose(noise[:2], want[:2], rtol=1e-4, atol=0), (noise, want)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_frozen_tensors_are_absent(model, dev):
    case = mixed_case(dev, model, 300)
    params = t(case.flat, dev)
    order = np.random.default_rng(2).permutation(case.count)
    free = case.engine()
    frozen = case.engine()
    names = list(frozen.layout.slots)
    trained = [frozen.layout.slots[n].owner != "enc" for n in names]
    frozen.set_param_groups([1e-3] * len(names), [0.0] * len(names), trained)
    mask = trained_columns(frozen)
    assert not mask.all() and mask.any()
    _, (A0, S0, _, _) = measure(case, free, params, order)
    g, (A, S, _, _) = measure(case, frozen, params, order)
    assert not g[:frozen.num_params][~mask].any()
    S_ref = float(np.square(g[:frozen.num_params].astype(np.float64)[mask]).sum())
    A_ref = reference_A(case, free, params, order, mask)          # the free engine's groups, the trained columns
    assert abs(S / S_ref - 1.0) < 1e-5 and abs(A / A_ref - 1.0) < 1e-5, (A, A_ref, S, S_ref)
    assert A < A0 and S < S0


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_stop_word_gives_no_sample_and_calls_are_deterministic(model, dev):
    case = mixed_case(dev, model, 300)
    params = t(case.flat, dev)
    order = np.random.default_rng(3).permutation(case.count)
    eng = case.engine()
    first = measure(case, eng, params, order)
    again = measure(case, eng, params, order)
    assert np.array_equal(first[0], again[0]) and first[1].tobytes() == again[1].tobytes()
    assert first[1][3] == case.count and first[1][0] > 0
    stop = case.engine(target_kl=1e-12, clip_mode=_lib.CLIP_NEVER)
    g = stop.ppo_step(case.blob, params.clone(), *global_args(case))
    torch.cuda.synchronize()
    assert g.cpu().numpy()[stop.stat_offset + 13] == 1               # the step stopped and set the word
    g, noise = measure(case, stop, params, order)
    assert noise.tolist() == [0.0, 0.0, 0.0, 0.0]
    assert g[stop.stat_offset + 14] == 1


def run_update(model, dev, seed=7, b=None, log=None, **kw):
    flat = flat_init(model, 3)
    b = batch(4) if b is None else b
    up = PPOUpdater(flat, N_CAP, E_CAP, dev, lr=3e-3, gamma=0.99, tau=0.95, opt_num_epochs=3, mini_batch_size=16,
                    model=model, **kw)
    if kw.get("param_groups"):
        names = list(up.engine.layout.slots)
        up.set_param_groups([dict(params=[n for n in names if up.engine.layout.slots[n].owner != "enc"], lr=2e-3)])
    np.random.seed(seed)
    out = up.update_params(b.states, b.actions, b.rewards, b.masks, b.exps, iteration=2,
                           log_fn=None if log is None else (lambda tag, v, s: log.append((tag, v, s))))
    return up, out, np.random.get_state()


COMBOS = {
    "plain": dict(),
    "combined": dict(target_kl=0.02, normalize_advantage=True, value_clip=0.2, param_groups=True,
                     clip_mode=_lib.CLIP_NEVER),
}


@pytest.mark.parametrize("combo", list(COMBOS))
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_training_is_bit_identical_to_the_option_off(model, combo, dev):
    logs = ([], [])
    (u0, o0, r0), (u1, o1, r1) = (run_update(model, dev, log=logs[k], **COMBOS[combo],
                                             **(dict(grad_noise_every=1) if k else {})) for k in (0, 1))
    assert np.array_equal(u0.flat_params(), u1.flat_params())
    for a, c in zip(u0.engine.get_opt_state(), u1.engine.get_opt_state()):
        assert np.array_equal(a, c)
    if u0.engine.param_groups is not None:
        assert np.array_equal(u0.engine.get_tensor_steps(), u1.engine.get_tensor_steps())
    assert np.array_equal(u0._grad_ring.cpu().numpy(), u1._grad_ring.cpu().numpy())
    assert o1.keys() - o0.keys() == set(NOISE_KEYS) and o0.keys() <= o1.keys()
    assert all(np.array_equal(o0[k], o1[k]) for k in o0)
    assert r0[0] == r1[0] and np.array_equal(r0[1], r1[1]) and r0[2:] == r1[2:]
    assert logs[0] == [x for x in logs[1] if not x[0].startswith("diag/grad_noise")]
    noise_tags = [(tag, s) for tag, _, s in logs[1] if tag.startswith("diag/grad_noise")]
    assert sorted(noise_tags) == sorted(("diag/" + k, 2) for k in NOISE_KEYS)
    applied = o1.get("steps_applied", 3 * 3)
    assert o1["grad_noise_samples"] == applied
    # three launches per measured step: every step ran, the steps after a KL stop too
    assert u1.engine.launches - u0.engine.launches == 3 * 3 * (u1.opt_num_epochs if "kl_stop" not in o1 or
                                                               o1["kl_stop"] is None else o1["kl_stop"][0] + 1)


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_only_steps_that_applied_adam_count(model, dev):
    _, out, _ = run_update(model, dev, grad_noise_every=1, target_kl=1e-9, clip_mode=_lib.CLIP_NEVER)
    assert out["kl_stop"] is not None
    assert out["grad_noise_samples"] == out["steps_applied"] == 1       # the first step's KL is 0 and applies
    assert np.isfinite(out["grad_noise_scale"]) or np.isinf(out["grad_noise_scale"])
    b = batch(4)
    b.rewards = b.rewards.copy()
    b.rewards[0] = np.nan                               # graph 0 alone is not finite: its minibatch is skipped
    _, out, _ = run_update(model, dev, b=b, grad_noise_every=1, skip_nonfinite=True)
    assert out["nonfinite_skips"] == 3
    assert out["grad_noise_samples"] == 3 * 3 - 3


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_end_to_end_through_use_b200_update(model, dev):
    flat = flat_init(model, 3)
    b = batch(4)
    logs = {}
    for k in (None, 1, 5):                              # 48 graphs, 16 per minibatch: 3 steps per epoch
        logged = []
        ag = make_agent(model, dev, flat, logged, lr=3e-3, num_optim_epoch=2, mini_batch_size=16)
        ctl = use_b200_update(ag, **({} if k is None else dict(grad_noise_every=k)))
        np.random.seed(3)
        ag.update_params(b, 0)
        np.random.seed(4)
        ag.update_params(b, 1)
        logs[k] = logged
        if k is not None:
            assert ctl.updater.grad_noise_every == k
    for k, per_iter in ((1, 2 * 3), (5, 2)):            # k > 3: step 0 of each epoch only
        got = [(tag, v, s) for tag, v, s in logs[k] if tag.startswith("diag/grad_noise")]
        assert [s for tag, _, s in got if tag == "diag/grad_noise_samples"] == [0, 1]
        assert [v for tag, v, _ in got if tag == "diag/grad_noise_samples"] == [per_iter, per_iter]
        assert len(got) == 2 * 4
        assert [x for x in logs[k] if not x[0].startswith("diag/grad_noise")] == logs[None]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_update_estimate_is_the_combination_of_its_measurements(model, dev):
    """The update's report equals grad_noise_estimate over the rows it measured (captured around the engine call)."""
    flat = flat_init(model, 3)
    b = batch(4)
    up = PPOUpdater(flat, N_CAP, E_CAP, dev, lr=3e-3, opt_num_epochs=2, mini_batch_size=16, model=model,
                    grad_noise_every=2)
    rows, ids_seen = [], []
    inner = up.engine.ppo_grad_noise

    def spy(*a, **kw):
        out = inner(*a, **kw)
        torch.cuda.synchronize()
        rows.append(out[1].cpu().numpy().copy())
        ids_seen.append(kw["ids"].cpu().numpy().copy())
        return out
    up.engine.ppo_grad_noise = spy
    np.random.seed(5)
    out = up.update_params(b.states, b.actions, b.rewards, b.masks, b.exps)
    assert len(rows) == 2 * 2                           # steps 0 and 2 of both epochs
    assert all(r[3] == 16 for r in rows) and all(sorted(x.tolist()) != x.tolist() for x in ids_seen)
    want = grad_noise_estimate(*grad_noise_terms(rows), 16, 4)
    assert {k: out[k] for k in want} == want
