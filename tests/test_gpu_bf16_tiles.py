"""H100: the bf16-tile build (libupb200_bf16.so, BASELINE.json configs[2]) against the parity build and against float64
with the kernel's rounding (tests/bf16_oracle.py).

The library is chosen once per process (UPB_LIB, read when drl_urban_planning_b200._lib is imported), so the variant
runs in a child process -- this file run as a script, UPB_LIB set in the child's environment only -- and the parity
results come from this process, on the same inputs (`run`).  The child first checks that it loaded the variant.

  1. the tiles reach nothing else: forward / forward_cand, greedy and sampled select_action and policy_logits on the
     boundary batch, dhm256, concept_mixed256 and edge_empty, every rl-mlp entry point, gae, normalize_advantages and
     grad_norms are bit-identical to the parity build;
  2. where the tiles stop: in ppo_grad and a fused ppo_step, every gradient column outside bf16_oracle.TILE_TENSORS
     and statistics slots 0-16 (diagnostics on) are bit-identical, every tile tensor differs; slot 17 (the global
     norm) includes the tile tensors.  gcn1_b is the bias sum of the last layer's pull, formed before any tile, so it
     is among the equal columns;
  3. against the rounding oracle: each tensor within 1e-4 of bf16_oracle (the tile tensors within TILE_BAR, set from
     the measured effect of fp32 noise on bf16 rounding), each tile tensor at least TILE_APART times further from the
     exact float64 oracle (the variant really rounds);
  4. NaN: the poisoned steps of test_gpu_nonfinite_guard give the same non-finite gradient columns and the same guard
     decisions as the parity build (a NaN tile operand stays NaN);
  5. configs[2] as bench.py runs it: 256 DHM graphs per step in LPT order on the full grid, 8 fused steps from the
     first-step clip, steps 0, 1 and 7 teacher-forced against bf16_oracle and the float64 Adam; fused against two-call
     at every cross_path.SGNN_GRIDS size (the tile tensors at TILE_BAR).
Per-tensor errors against both oracles are printed (pytest -s)."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == "__main__":                          # the child process: the same imports as under pytest
    sys.path[:0] = [ROOT, HERE]

import torch  # noqa: E402

import bf16_oracle as BO  # noqa: E402
import cross_path as XP  # noqa: E402
import decay_oracle as DO  # noqa: E402
import scale_cases as SCL  # noqa: E402
import shape_cases as SC  # noqa: E402
from drl_urban_planning_b200 import _lib, params as PL, synth  # noqa: E402
from drl_urban_planning_b200.engine import Engine  # noqa: E402
from drl_urban_planning_b200.packing import pack_states  # noqa: E402
from drl_urban_planning_b200.ppo import GCLIP_NORM_SLOT, NONFINITE_SLOT  # noqa: E402
from fixtures_io import expand_states, synth_states  # noqa: E402
from harness import (Case, dev, fused_step, load, rel, reproducible_states, t, tensor_errors,  # noqa: E402,F401
                     two_call_step)
from oracle import sgnn_numpy as ON  # noqa: E402

pytestmark = pytest.mark.gpu

VARIANT = os.path.join(ROOT, "drl_urban_planning_b200", "libupb200_bf16.so")
GOLDEN = os.path.join(HERE, "golden")
NEVER = _lib.CLIP_NEVER
FORWARD_CASES = ["boundary", "dhm256", "concept_mixed256", "edge_empty"]
TRAIN_CASES = ["boundary", "small_mixed", "dhm256", "concept_mixed256"]
NON_TILE = [s for s in PL.SLOTS.values() if s.name not in BO.TILE_TENSORS]
STATS_EQUAL = 17                  # statistics slots 0-16; 17 is the pre-clip global norm, which sums the tile tensors
CAUSES = ["adv", "ret", "param"]
BENCH_SEED, BENCH_B, BENCH_STEPS, BENCH_CHECKED = 11, 256, 8, (0, 1, 7)
GRAD_BAR, ADAM_BAR, V_BAR = 1e-4, 1e-5, 1.4e-5          # test_gpu_update_scale's bars
# The tile tensors' bar against bf16_oracle, and how much further from exact float64 they must be.  A tile operand the
# kernel holds in fp32 and the oracle in float64 can sit on opposite sides of a bf16 rounding boundary; one such
# crossing moves its product by a bf16 ulp (2^-8 relative).  Measured on the CPU oracle: perturbing the A operands by 2^-22
# relative (fp32 noise) flips 3 of small_mixed's 90,288 roundings and moves gcn0_w by 3.2e-4, enc_b by 1.7e-4, gcn0_b by
# 6.5e-5 -- the H100's distances from bf16_oracle there (3.16e-4, 1.66e-4, 6.58e-5).  Rounding the B operands twice
# (TF32, then bf16) measured 1.3e-3 to 4.9e-3 from bf16_oracle, and exact float64 is 1.1e-3 to 5.2e-3 away.
TILE_BAR, TILE_APART = 5e-4, 5.0
FUSED_BAR = 1e-5                  # cross_path's fused-against-two-call bar, for the tensors the tiles do not reach


# ---- the cases -------------------------------------------------------------------------------------------------------
def case_inputs(name):
    """(states, actions, flat, adv, ret, fixed, exps); the PPO targets None for a forward-only fixture."""
    if name == "boundary":
        states, actions, _ = SC.boundary_batch(SC.BATCH_SEED)
        adv, ret, exps = synth.make_ppo_targets(SC.BATCH_SEED, len(states))
        exps[5] = 0.0
        fixed = np.random.default_rng(SC.BATCH_SEED).normal(-3.0, 0.3, size=(len(states), 1)).astype(np.float32)
        return states, actions, PL.default_init(SC.BATCH_SEED), adv, ret, fixed, exps
    z = load(GOLDEN, name)
    states = (synth_states(int(z["seed"]), str(z["community"]), int(z["count"]))[0] if "digest" in z.files
              else expand_states(z))
    if "advantages" not in z.files:
        return states, z["actions"], z["params"], None, None, None, None
    return states, z["actions"], z["params"], z["advantages"], z["returns"], z["fixed_log_probs"], z["exps"]


def train_args(dev, adv, ret, fixed, exps, actions):
    n_ind = max(int((np.asarray(exps) != 0).sum()), 1)
    return tuple(t(x, dev) for x in (actions, adv, ret, fixed, exps)) + (1.0 / len(exps), 1.0 / n_ind)


def np_(x):
    return np.zeros(0, np.float32) if x is None else x.detach().cpu().numpy().copy()


def opt_state(out, key, eng, p):
    torch.cuda.synchronize()
    m, v, s = eng.get_opt_state()
    out.update({key + "/params": np_(p), key + "/m": m, key + "/v": v, key + "/steps": s})


def run_sgnn_case(dev, name, out):
    states, actions, flat, adv, ret, fixed, exps = case_inputs(name)
    blob = pack_states(states).to(dev)
    kw = dict(clip_mode=NEVER, diagnostics=True)
    eng = Engine(dev, blob.n_cap, blob.e_cap, **kw)
    p = t(flat, dev)
    act = t(actions, dev)
    if name in FORWARD_CASES:
        res = eng.forward(blob, p, act, want_greedy=True, cand_log_probs=True)
        res += eng.forward(blob, p, act)
        uni = np.random.default_rng(7).random(blob.count).astype(np.float32)
        res += (eng.select_action(blob, p), eng.select_action(blob, p, t(uni, dev)))
        res += eng.policy_logits(blob, p)[:2]
        for i, x in enumerate(res):
            out[f"{name}/fwd{i}"] = np_(x)
    if name in TRAIN_CASES:
        args = train_args(dev, adv, ret, fixed, exps, actions)
        out[f"{name}/grad"] = np_(eng.ppo_grad(blob, p, *args))
        step = Engine(dev, blob.n_cap, blob.e_cap, **kw)
        p2 = p.clone()
        out[f"{name}/step"] = np_(step.ppo_step(blob, p2, *args))
        opt_state(out, f"{name}/step", step, p2)


def run_mlp(dev, out):
    """Every rl-mlp entry point on a minibatch whose rl-mlp gradients are run-to-run reproducible."""
    states, actions = reproducible_states(13, 16)
    c = Case(dev, "mlp", states, actions, 13)
    eng = c.engine()
    p = t(c.flat, dev)
    res = eng.forward(c.blob, p, c.dev_args[0], want_greedy=True, cand_log_probs=True)
    uni = np.random.default_rng(8).random(c.count).astype(np.float32)
    res += (eng.select_action(c.blob, p), eng.select_action(c.blob, p, t(uni, dev)))
    res += eng.policy_logits(c.blob, p)[:2]
    res += (eng.ppo_grad(c.blob, p, *c.step_args()),)
    e1, e2 = c.engine(), c.engine()
    p1, p2 = p.clone(), p.clone()
    for k in range(3):                       # the first step clips (two-call inside ppo_step), the others fuse
        res += (two_call_step(e1, c, p1), fused_step(e2, c, p2))
    for i, x in enumerate(res):
        out[f"mlp/{i}"] = np_(x)
    opt_state(out, "mlp/two", e1, p1)
    opt_state(out, "mlp/fused", e2, p2)


def run_misc(dev, out):
    """gae, normalize_advantages and grad_norms on seeded inputs."""
    rng = np.random.default_rng(9)
    eng = Engine(dev, 64, 128)
    T = 3000
    r, v = rng.standard_normal(T).astype(np.float32), rng.standard_normal(T).astype(np.float32)
    m = (rng.random(T) > 0.02).astype(np.float32)
    adv, ret = eng.gae(t(r, dev), t(m, dev), t(v, dev), 0.99, 0.95)
    exps = (rng.random(T) > 0.1).astype(np.float32)
    order = t(rng.permutation(T).astype(np.int32), dev)
    norm = eng.normalize_advantages(adv, t(exps, dev), order, 256)
    rows = t(rng.standard_normal((5, eng.grad_stride)).astype(np.float32), dev)
    out.update({"misc/adv": np_(adv), "misc/ret": np_(ret), "misc/norm": np_(norm),
                "misc/norms": np_(eng.grad_norms(rows))})


def nan_case(dev):
    states, actions = synth.make_states(5, "small", 12, stages=[i % 2 for i in range(12)])
    return Case(dev, "sgnn", states, actions, 5, zero_exps=(1,))


def run_nan(dev, out):
    """test_gpu_nonfinite_guard's poisoned steps on graph 0: an infinite advantage at a ratio inside the clip range, a
    NaN return, a NaN in the value head's output bias; guard on, both step paths."""
    c = nan_case(dev)
    logp0 = c.engine().forward(c.blob, t(c.flat, dev), c.dev_args[0])[1].cpu().numpy()
    for cause in CAUSES:
        adv, ret, fixed, flat = c.adv.copy(), c.ret.copy(), c.fixed.copy(), c.flat.copy()
        if cause == "adv":
            fixed[0], adv[0] = logp0[0], np.inf
        elif cause == "ret":
            ret[0] = np.nan
        else:
            flat[PL.SLOTS["val_b2"].offset] = np.nan
        c.dev_args = (c.dev_args[0], t(adv, dev), t(ret, dev), t(fixed, dev), c.dev_args[4])
        for path, run in (("fused", fused_step), ("two", two_call_step)):
            eng = c.engine(clip_mode=NEVER, skip_nonfinite=True, diagnostics=True)
            p = t(flat, dev)
            out[f"nan/{cause}/{path}/buf"] = np_(run(eng, c, p))
            opt_state(out, f"nan/{cause}/{path}", eng, p)


def bench_case():
    states, actions = synth.make_states(BENCH_SEED, "dhm", 2 * BENCH_B)
    rng = np.random.default_rng(BENCH_SEED)
    adv = rng.standard_normal(len(states)).astype(np.float32)
    ret = rng.standard_normal(len(states)).astype(np.float32)
    return states, actions, adv, ret, np.ones(len(states), np.float32), PL.default_init(BENCH_SEED)


def run_bench(dev, out):
    """configs[2] as bench.py runs it: two minibatches of 256 DHM graphs, each in the static LPT order, the full grid,
    the first-step clip, 8 fused steps; the device state before and after each step."""
    states, actions, adv, ret, exps, flat = bench_case()
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap)
    params = t(flat, dev)
    pert = t(flat * (1.0 + 0.05 * np.random.default_rng(3).standard_normal(flat.size)).astype(np.float32), dev)
    act = t(actions, dev)
    fixed = eng.forward(blob, pert, act)[1]
    cost = Engine.graph_cost(blob.info.astype(np.int64))
    ids = [eng.balance_ids(np.arange(m * BENCH_B, (m + 1) * BENCH_B), cost).astype(np.int32) for m in range(2)]
    out["bench/fixed"], out["bench/ids"] = np_(fixed), np.stack(ids)
    dargs = (act, t(adv, dev), t(ret, dev), fixed, t(exps, dev), 1.0 / BENCH_B, 1.0 / BENCH_B)
    for k in range(BENCH_STEPS):
        opt_state(out, f"bench/{k}/before", eng, params)
        out[f"bench/{k}/buf"] = np_(eng.ppo_step(blob, params, *dargs, ids=t(ids[k % 2], dev)))
        opt_state(out, f"bench/{k}/after", eng, params)
    c = Case(dev, "sgnn", states[:BENCH_B], actions[:BENCH_B], BENCH_SEED)
    for grid in XP.SGNN_GRIDS:
        e1, e2 = c.engine(grid_limit=grid), c.engine(grid_limit=grid)
        p1, p2 = t(c.flat, dev).clone(), t(c.flat, dev).clone()
        for step in range(4):                 # the first step clips (two-call inside ppo_step), the others fuse
            g1 = two_call_step(e1, c, p1)
            before = e2.launches
            g2 = fused_step(e2, c, p2)
            key = f"bench/grid{grid}/{step}"
            out.update({key + "/two": np_(g1), key + "/fused": np_(g2),
                        key + "/launches": np.array(e2.launches - before),
                        key + "/losses": np.array([e1.read_losses(g1), e2.read_losses(g2)])})
        opt_state(out, f"bench/grid{grid}/two", e1, p1)
        opt_state(out, f"bench/grid{grid}/fused", e2, p2)


def run(dev, variant):
    """Every workload of this module with the library this process loaded, as {key: numpy array}."""
    out = {}
    for name in dict.fromkeys(FORWARD_CASES + TRAIN_CASES):
        run_sgnn_case(dev, name, out)
    run_mlp(dev, out)
    run_misc(dev, out)
    run_nan(dev, out)
    if variant:
        run_bench(dev, out)
    torch.cuda.synchronize()
    return out


def loaded_libraries():
    with open("/proc/self/maps") as f:
        return {os.path.basename(line.split()[-1]) for line in f if line.rstrip().endswith(".so")}


# ---- the two builds --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def parity(dev):
    assert os.path.basename(_lib.LIB_PATH) == "libupb200.so", _lib.LIB_PATH
    return run(dev, variant=False)


@pytest.fixture(scope="module")
def variant(tmp_path_factory):
    assert os.path.exists(VARIANT), "libupb200_bf16.so is missing: build() makes it"
    out = tmp_path_factory.mktemp("bf16") / "variant.npz"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), str(out)]
    res = subprocess.run(cmd, env=dict(os.environ, UPB_LIB=VARIANT), capture_output=True, text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-6000:]
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


# ---- 1. the tiles reach nothing else ---------------------------------------------------------------------------------
@pytest.mark.parametrize("prefix", FORWARD_CASES + ["mlp", "misc"])
def test_untiled_entry_points_are_bit_identical(parity, variant, prefix):
    keys = [k for k in parity if k.startswith(prefix + "/") and (prefix not in TRAIN_CASES or "/fwd" in k)]
    assert len(keys) >= 4
    bad = [k for k in keys if not same_bits(variant[k], parity[k])]
    assert not bad, bad


# ---- 2. where the tiles stop -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("what", ["grad", "step"])
@pytest.mark.parametrize("name", TRAIN_CASES)
def test_only_the_tile_tensors_differ(parity, variant, name, what):
    a, b = variant[f"{name}/{what}"], parity[f"{name}/{what}"]
    for s in PL.SLOTS.values():
        same = same_bits(a[s.offset:s.offset + s.size], b[s.offset:s.offset + s.size])
        assert same == (s.name not in BO.TILE_TENSORS), (s.name, same)
    so = _lib.UPB_STAT_OFFSET
    assert same_bits(a[so:so + STATS_EQUAL], b[so:so + STATS_EQUAL]), np.flatnonzero(a[so:so + 17] != b[so:so + 17])
    if what == "step":                        # Adam is per entry: the untiled tensors' parameters and moments agree
        for part in ("params", "m", "v"):
            x, y = variant[f"{name}/step/{part}"], parity[f"{name}/step/{part}"]
            for s in NON_TILE:
                assert same_bits(x[s.offset:s.offset + s.size], y[s.offset:s.offset + s.size]), (part, s.name)
        assert same_bits(variant[f"{name}/step/steps"], parity[f"{name}/step/steps"])


# ---- 3. against the rounding oracle ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def oracles():
    """{case: (bf16 oracle gradient, exact float64 gradient)} at the cases' initial parameters."""
    res = {}
    for name in TRAIN_CASES:
        states, actions, flat, adv, ret, fixed, exps = case_inputs(name)
        args = (flat, states, actions, adv, ret, fixed, exps)
        res[name] = (BO.ppo_minibatch(*args)["grad"], ON.ppo_minibatch(*args)["grad"])
    return res


@pytest.mark.parametrize("what", ["grad", "step"])
@pytest.mark.parametrize("name", TRAIN_CASES)
def test_variant_against_the_rounding_oracle(variant, oracles, name, what):
    got = variant[f"{name}/{what}"][:PL.NUM_PARAMS].astype(np.float64)
    want_bf, want_exact = oracles[name]
    e_bf, e_exact = tensor_errors(got, want_bf), tensor_errors(got, want_exact)
    print(f"\n[bf16 tiles] {name} {what}: tensor, error vs bf16_oracle, vs exact float64")
    for s in PL.SLOTS.values():
        print(f"  {s.name:10s} {e_bf[s.name]:.3g} {e_exact[s.name]:.3g}")
    check_tile_split(e_bf, GRAD_BAR, name)
    for k in BO.TILE_TENSORS:
        assert e_exact[k] >= TILE_APART * e_bf[k] and e_exact[k] > 1e-3, (k, e_bf[k], e_exact[k])


def check_tile_split(errs, bar, what):
    """Every tensor the tiles do not reach within `bar`, the tile tensors within TILE_BAR."""
    bad = {k: e for k, e in errs.items() if not e < (TILE_BAR if k in BO.TILE_TENSORS else bar)}
    assert not bad, (what, bad)


# ---- 4. NaN ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["fused", "two"])
@pytest.mark.parametrize("cause", CAUSES)
def test_nonfinite_columns_and_guard_decisions_match(parity, variant, cause, path):
    key = f"nan/{cause}/{path}"
    a, b = variant[key + "/buf"], parity[key + "/buf"]
    fa, fb = np.isfinite(a[:PL.NUM_PARAMS]), np.isfinite(b[:PL.NUM_PARAMS])
    bad = [s.name for s in PL.SLOTS.values() if not np.array_equal(fa[s.offset:s.offset + s.size],
                                                                   fb[s.offset:s.offset + s.size])]
    assert not bad, (cause, path, bad)
    assert not fb.all()
    so = _lib.UPB_STAT_OFFSET
    for slot in (NONFINITE_SLOT, GCLIP_NORM_SLOT):
        assert same_bits(a[so + slot], b[so + slot]), (slot, a[so + slot], b[so + slot])
    assert a[so + NONFINITE_SLOT] == 1
    for part in ("params", "m", "v", "steps"):              # the guard skipped the step in both: nothing changed
        assert same_bits(variant[f"{key}/{part}"], parity[f"{key}/{part}"]), part


# ---- 5. configs[2] as bench.py runs it -------------------------------------------------------------------------------
@pytest.mark.parametrize("k", BENCH_CHECKED)
def test_bench_steps_teacher_forced(variant, k):
    states, actions, adv, ret, exps, _ = bench_case()
    sel = variant["bench/ids"][k % 2].astype(np.int64)
    assert sorted(sel.tolist()) == list(range((k % 2) * BENCH_B, (k % 2 + 1) * BENCH_B))
    p0, m0, v0, s0 = (variant[f"bench/{k}/before/{x}"] for x in ("params", "m", "v", "steps"))
    p1, m1, v1, s1 = (variant[f"bench/{k}/after/{x}"] for x in ("params", "m", "v", "steps"))
    fixed = variant["bench/fixed"]
    args = (p0, [states[i] for i in sel], actions[sel], adv[sel], ret[sel], fixed[sel], exps[sel])
    want = BO.ppo_minibatch(*args)["grad"]
    g = variant[f"bench/{k}/buf"][:PL.NUM_PARAMS].astype(np.float64)
    errs = tensor_errors(g, want)
    where = max(errs, key=errs.get)
    e_bf = errs[where]
    e_exact = tensor_errors(g, ON.ppo_minibatch(*args)["grad"]) if k == 0 else None
    print(f"\n[bf16 tiles] bench step {k}: gradient vs bf16_oracle {e_bf:.3g} ({where})"
          + ("" if e_exact is None else ", tile tensors vs exact " + ", ".join(f"{x} {e_exact[x]:.3g}"
                                                                              for x in BO.TILE_TENSORS)))
    check_tile_split(errs, GRAD_BAR, k)
    stages = np.array([int(np.argmax(states[i][8][:2])) for i in sel])
    live = SCL.live_entries(stages, PL.SGNN)
    want_p, want_m, want_v, _ = DO.adam_step(p0, m0, v0, SCL.entry_steps(s0, PL.SGNN),
                                             SCL.clip_groups(g, PL.SGNN) if k == 0 else g, live, 0.0)
    errs = dict(params=rel(p1, want_p), m=rel(m1, want_m), v=rel(v1, want_v))
    print(f"[bf16 tiles] bench step {k}: Adam " + ", ".join(f"{x} {e:.3g}" for x, e in errs.items()))
    assert errs["params"] < ADAM_BAR and errs["m"] < ADAM_BAR and errs["v"] < V_BAR, (k, errs)
    assert (s1 - s0).tolist() == [1, 1, int((stages == 0).any()), int((stages == 1).any())]


@pytest.mark.parametrize("grid", XP.SGNN_GRIDS)
def test_bench_fused_against_two_call(variant, grid):
    """cross_path.check_sgnn_fused_against_two_call on the variant: 4 steps, the first clipping.  From step 1 on the
    two paths' parameters differ by their reduction order, and that fp32 noise moves tile operands across bf16
    rounding boundaries, so the tile tensors are held to TILE_BAR, the others to the cross-path bar."""
    key = f"bench/grid{grid}"
    for step in range(4):
        g1, g2 = (variant[f"{key}/{step}/{x}"][:PL.NUM_PARAMS] for x in ("two", "fused"))
        check_tile_split(tensor_errors(g2, g1), FUSED_BAR, (grid, step))
        assert (int(variant[f"{key}/{step}/launches"]) == 1) == (step > 0), step
        l1, l2 = variant[f"{key}/{step}/losses"]
        assert np.allclose(l2, l1, rtol=1e-5, atol=1e-6), (step, l1, l2)
    for part, bar in (("m", FUSED_BAR), ("v", FUSED_BAR), ("params", 1e-6)):      # cross_path's bars
        check_tile_split(tensor_errors(variant[f"{key}/fused/{part}"], variant[f"{key}/two/{part}"]), bar, part)
    s1, s2 = variant[f"{key}/two/steps"].tolist(), variant[f"{key}/fused/steps"].tolist()
    assert s1 == s2 and s1[:2] == [4, 4], (s1, s2)


# ---- the child process -----------------------------------------------------------------------------------------------
if __name__ == "__main__":
    assert os.path.basename(_lib.LIB_PATH) == "libupb200_bf16.so", _lib.LIB_PATH
    _lib.lib()
    libs = loaded_libraries()
    assert "libupb200_bf16.so" in libs and "libupb200.so" not in libs, sorted(x for x in libs if "upb" in x)
    results = run(torch.device("cuda", 0), variant=True)
    np.savez(sys.argv[1], **results)
