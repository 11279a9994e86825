"""GPU (H100): both models on graphs above the hlg caps (tests/cap_cases.py) against float64 -- oracle/sgnn_numpy.py for
the SGNN, oracle/mlp_port.py run in float64 for the rl-mlp -- at the bars of the other parity tests: per-tensor 1e-4 for
gradients, 1e-4 for values and entropies, lp_tol for log-probs.

The cases are the shipped concept configs' caps (1500 nodes, 4000 edges: every edge or every node a candidate, one
past each hlg cap, a hub row) and the blob format's 16-bit limits (65535 nodes / 32767 edges: node ids, row pointers,
slot tags and candidate ids with bit 15 set, a hub row of degree 32767, 32767 land-use and 65535 road candidates).
Each graph runs in a launch of its own and in one mixed launch with ordinary concept-sized graphs, walked by one CTA
in order (big -> small -> big); the forward outputs must be bit-identical in both.

Memory: at 65535 / 32767 the SGNN's per-CTA global scratch is scratch_floats = 65535 x 146 + 65535 x 18 + 64 floats,
about 43 MB (the rl-mlp's 9 MB), so the engines on these caps run on grid_limit CTAs, and each test closes its engines
before the next builds its own.  Measured on an H100 80GB HBM3 (cudaMemGetInfo just before each engine is closed,
less the use at the module's start; engines allocate outside torch's caching allocator): at most 958 MiB."""
import math

import numpy as np
import pytest
import torch

import cap_cases as CC
from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.model import MASK_FILL
from drl_urban_planning_b200.packing import pack_states
from harness import dev, heads, lp_tol, per_tensor_rel, rel, t
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from test_gpu_select import BELOW_ONE, band, boundary_uniforms, check_sweep, grid_uniforms

pytestmark = pytest.mark.gpu

TOL = 1e-4
GRID = 4                    # CTAs of an engine on the 65535 / 32767 caps
CASES = [r[0] for r in CC.CONCEPT_CASES] + [r[0] for r in CC.ABI_CASES]
ROWS = {r[0]: r for r in CC.CONCEPT_CASES + CC.ABI_CASES}


def layout(model):
    return PL.MLP if model == "mlp" else PL.SGNN


def flat_params(model, seed=5):
    return PL.MLP.default_init(seed) if model == "mlp" else PL.default_init(seed)


# ------------------------------------------------------------------------------------------------------ minibatches
class Batch:
    """States with PPO targets: old log-probs at the float64 log-prob + N(0, 0.1), so ratios straddle the clip range
    whatever the candidate count; the last graph has exps = 0 when there are several."""

    def __init__(self, states, actions, labels, seed=7):
        self.states, self.actions, self.labels = states, actions, labels
        self.count = len(states)
        rng = np.random.default_rng(seed)
        self.adv = rng.standard_normal((self.count, 1)).astype(np.float32)
        self.ret = rng.standard_normal((self.count, 1)).astype(np.float32)
        self.exps = np.ones(self.count, np.float32)
        if self.count > 1:
            self.exps[-1] = 0.0
        self.noise = rng.normal(0.0, 0.1, (self.count, 1))
        self.n_cap, self.e_cap = states[0][1].shape[0], states[0][2].shape[0]
        self.stage = np.array([int(np.argmax(st[8][:2])) for st in states])
        self._ref = {}

    def fixed(self, model, flat):
        return (self.ref(model, flat)["log_prob"].reshape(-1, 1) + self.noise).astype(np.float32)

    def ref(self, model, flat):
        """float64: per graph value, log-prob, entropy and (candidate index, logit) rows; with the old log-probs,
        the gradient and the four losses.  Cached per model."""
        if model not in self._ref:
            self._ref[model] = (sgnn_ref if model == "sgnn" else mlp_ref)(flat, self)
        return self._ref[model]

    def dev_args(self, model, flat, dev):
        return tuple(t(x, dev) for x in (self.actions, self.adv, self.ret, self.fixed(model, flat), self.exps))


def sgnn_ref(flat, b):
    P = ON._p64(flat)
    out = dict(value=[], log_prob=[], entropy=[], cands=[])
    for i, st in enumerate(b.states):
        fw = ON.forward(P, ON.unpad(st), action=int(b.actions[i, b.stage[i]]), keep=True)
        c = fw["cache"]
        w1 = P["lu_w1" if b.stage[i] == 0 else "road_w1"].reshape(-1)
        out["cands"].append((c["idx"], c["th"] @ w1))
        for k in ("value", "log_prob", "entropy"):
            out[k].append(fw[k])
    out = {k: (np.array(v) if k != "cands" else v) for k, v in out.items()}
    fixed = (out["log_prob"].reshape(-1, 1) + b.noise).astype(np.float32)
    mb = ON.ppo_minibatch(flat, b.states, b.actions, b.adv, b.ret, fixed, b.exps)
    out.update(grad=mb["grad"], losses=[mb["loss"], mb["value_loss"], mb["surr_loss"], mb["entropy_loss"]])
    return out


def mlp_ref(flat, b):
    """The port's losses graph by graph in float64 (one padded 65535-node state at a time), each term scaled by the
    minibatch's 1/B or 1/|ind| exactly as the port's means, so the summed autograd gradient is the port's."""
    P = MP.params_from_flat(flat, torch.float64, requires_grad=True)
    B, n_ind = b.count, max(int((b.exps != 0).sum()), 1)
    out = dict(value=[], log_prob=[], entropy=[], cands=[])
    terms = []
    for i, st in enumerate(b.states):
        pb = MP.stack_states([st])
        v = MP.value(P, pb)[0, 0]
        lp, en = MP.log_prob_entropy(P, pb, torch.tensor(b.actions[i:i + 1]))
        with torch.no_grad():
            zl, zr = MP.masked_logits(P, pb)
        idx = np.flatnonzero(st[6] if b.stage[i] == 0 else st[7])
        out["cands"].append((idx, (zl if b.stage[i] == 0 else zr)[0].numpy()[idx]))
        for k, x in (("value", v), ("log_prob", lp[0, 0]), ("entropy", en[0, 0])):
            out[k].append(float(x.detach()))
        terms.append((v, lp[0, 0], en[0, 0]))
    out = {k: (np.array(v) if k != "cands" else v) for k, v in out.items()}
    fixed = out["log_prob"] + b.noise.reshape(-1)
    fixed = fixed.astype(np.float32).astype(np.float64)
    vl = surr = el = 0.0
    for i, (v, lp, en) in enumerate(terms):
        vl = vl + (v - float(b.ret[i, 0])) ** 2 / B
        if b.exps[i] != 0:
            r = torch.exp(lp - fixed[i])
            a = float(b.adv[i, 0])
            surr = surr - torch.min(r * a, torch.clamp(r, 0.8, 1.2) * a) / n_ind
            el = el - en / n_ind
    loss = surr + 0.5 * vl + 0.01 * el
    loss.backward()
    out["grad"] = PL.MLP.flatten({k: (p.grad.numpy() if p.grad is not None else np.zeros(tuple(p.shape)))
                                  for k, p in P.items()})
    out["losses"] = [float(x) for x in (loss, vl, surr, el)]
    return out


_batches = {}


def batch(name):
    """'concept' / 'abi' (the mixed batches) or a case label (that graph alone, as built in its mixed batch)."""
    if name not in _batches:
        if name == "concept":
            _batches[name] = Batch(*CC.concept_batch())
        elif name == "abi":
            _batches[name] = Batch(*CC.abi_batch())
        else:
            mixed = batch("abi" if name in {r[0] for r in CC.ABI_CASES} else "concept")
            i = mixed.labels.index(name)
            _batches[name] = Batch([mixed.states[i]], mixed.actions[i:i + 1], [name])
    return _batches[name]


# ------------------------------------------------------------------------------------------------------ checks
def lp_err_ratio(lp, lp64, zabs):
    return float((np.abs(np.asarray(lp, np.float64) - lp64) / lp_tol(lp64, zabs)).max())


def check_forward(eng, model, b, flat, dev, ids=None, worst=None):
    """forward_cand, greedy and policy_logits of the batch against float64; returns the forward outputs (numpy)."""
    ref = b.ref(model, flat)
    blob = pack_states(b.states).to(dev)
    params = t(flat, dev)
    ids_d = None if ids is None else t(np.asarray(ids, np.int32), dev)
    value, logp, ent, greedy, cand = (x.cpu().numpy() for x in eng.forward(
        blob, params, t(b.actions, dev), ids=ids_d, want_greedy=True, cand_log_probs=True))
    worst = {} if worst is None else worst

    def note(key, v):
        worst[key] = max(worst.get(key, 0.0), v)

    note("value", rel(value, ref["value"]))
    note("entropy", rel(ent, ref["entropy"]))
    assert worst["value"] < TOL and worst["entropy"] < TOL, (b.labels, worst)
    offs = np.concatenate([[0], np.cumsum((blob.info[:, 2] + 3) // 4 * 4)])
    for i, (idx, z) in enumerate(ref["cands"]):
        label, zabs = b.labels[i], float(np.abs(z).max()) if z.size else 0.0
        zs = z - z.max()
        lp64 = zs - math.log(np.exp(zs).sum())
        note("log_prob", lp_err_ratio(logp[i], ref["log_prob"][i], zabs))
        lpk = cand[offs[i]:offs[i] + idx.size]
        note("cand_log_prob", lp_err_ratio(lpk, lp64, zabs))
        assert worst["log_prob"] <= 1.0 and worst["cand_log_prob"] <= 1.0, (label, worst)
        # greedy: the float64 arg-max wherever its margin over the runner-up exceeds both log-probs' tolerances
        top = np.argsort(-lp64, kind="stable")
        margin = lp64[top[0]] - lp64[top[1]] if idx.size > 1 else np.inf
        if margin > 2 * lp_tol(lp64[top[0]], zabs):
            assert greedy[i] == idx[top[0]], (label, greedy[i], idx[top[0]], margin)
        else:
            near = idx[lp64 >= lp64[top[0]] - 2 * lp_tol(lp64[top[0]], zabs)]
            assert greedy[i] in near, (label, greedy[i], near)
    # masked logit rows: the fill value bit for bit, the candidates against float64
    lu, rd, stage = eng.policy_logits(blob, params, ids=ids_d)
    rows = {0: lu.cpu().numpy() if lu is not None else None, 1: rd.cpu().numpy() if rd is not None else None}
    order = np.arange(b.count) if ids is None else np.asarray(ids)
    for s in (0, 1):
        mine = order[stage[order] == s]
        for r, i in enumerate(mine):
            idx, z = ref["cands"][i]
            row = rows[s][r]
            assert row.size == (b.e_cap if s == 0 else b.n_cap)
            fill = np.ones(row.size, bool)
            fill[idx] = False
            assert (row[fill].view(np.uint32) == np.float32(MASK_FILL).view(np.uint32)).all(), b.labels[i]
            if idx.size:
                note("logits", float(np.abs(row[idx] - z).max() / max(np.abs(z).max(), 1e-9)))
                assert worst["logits"] < TOL, (b.labels[i], worst)
    return dict(value=value, logp=logp, ent=ent, greedy=greedy, cand=cand, offs=offs, info=blob.info)


def check_grad(eng, model, b, flat, dev, ids=None, worst=None):
    """ppo_grad (every tensor, the statistics' losses) against float64; returns the kernel's gradient buffer."""
    ref = b.ref(model, flat)
    blob = pack_states(b.states).to(dev)
    ids_d = None if ids is None else t(np.asarray(ids, np.int32), dev)
    n_ind = max(int((b.exps != 0).sum()), 1)
    g = eng.ppo_grad(blob, t(flat, dev), *b.dev_args(model, flat, dev), 1.0 / b.count, 1.0 / n_ind, ids=ids_d)
    L = layout(model)
    gk = g.cpu().numpy()
    err, where = per_tensor_rel(gk[:L.num_params], ref["grad"], L)
    if worst is not None:
        worst["grad"] = max(worst.get("grad", 0.0), err)
    assert err < TOL, (b.labels, err, where)
    assert np.allclose(eng.read_losses(g), ref["losses"], rtol=1e-4, atol=1e-5), (eng.read_losses(g), ref["losses"])
    return g, gk


WORST = {}
PEAK = {"base": None, "peak": 0}


def in_use():
    free, total = torch.cuda.mem_get_info()
    return total - free


@pytest.fixture(scope="module", autouse=True)
def device_memory(dev):
    """The most device memory the module held above its start, printed with -s."""
    torch.cuda.synchronize()
    PEAK["base"] = in_use()
    yield
    print(f"\n[caps] device memory above the module's start: at most {PEAK['peak'] / 2**20:.0f} MiB")


def close(*engines):
    torch.cuda.synchronize()
    PEAK["peak"] = max(PEAK["peak"], in_use() - PEAK["base"])
    for e in engines:
        e.close()


def report(key, worst):
    """Worst errors per check, printed with -s (value / entropy / logits / grad / params: relative; log-probs: share
    of lp_tol)."""
    WORST.setdefault(key, {})
    for k, v in worst.items():
        WORST[key][k] = max(WORST[key].get(k, 0.0), v)
    print(f"\n[caps] {key}: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST[key].items())))


# ------------------------------------------------------------------------------------------------------ tests
def test_caps_past_the_format_are_refused(dev):
    for n_cap, e_cap in ((65536, 100), (100, 32768), (0, 10)):
        with pytest.raises(_lib.UpbError, match="caps must satisfy"):
            Engine(dev, n_cap, e_cap)
    for model in ("sgnn", "mlp"):
        eng = Engine(dev, CC.MAX_N, CC.MAX_E, model=model, grid_limit=1)
        close(eng)


def sample_sweep(eng, model, b, flat, fw, dev, grid):
    """select_action with one uniform per copy of the graph against the float64 inverse CDF, by
    test_gpu_select.py's rule (kernel CDF within band(k), float64 CDF within band(k) plus the log-prob error)."""
    idx, z = b.ref(model, flat)["cands"][0]
    if idx.size == 0:
        return
    zs = z - z.max()
    lp64 = zs - math.log(np.exp(zs).sum())
    lpk = fw["cand"][:idx.size].astype(np.float64)
    pk = np.exp(lpk - lpk.max())
    cdfk = np.cumsum(pk) / pk.sum()
    cdf64 = np.cumsum(np.exp(lp64))
    err64 = float(2 * (np.exp(lp64) * np.abs(lpk - lp64)).sum())
    pick = np.random.default_rng(3).choice(idx.size - 1, size=min(4, idx.size - 1), replace=False) \
        if idx.size > 1 else np.zeros(0, int)
    u = np.concatenate([grid_uniforms(grid), boundary_uniforms(cdfk[pick]), [0.0, BELOW_ONE]]).astype(np.float32)
    blob = pack_states([b.states[0]] * u.size).to(dev)
    picks = eng.select_action(blob, t(flat, dev), uniforms=t(u, dev)).cpu().numpy()
    check_sweep(b.labels[0], u, picks, idx, lp64, [("kernel", cdfk, band(idx.size)),
                                                    ("float64", cdf64, band(idx.size) + err64)], grid)
    assert np.array_equal(eng.select_action(pack_states([b.states[0]]).to(dev), t(flat, dev)).cpu().numpy(),
                          fw["greedy"][:1])


def adam_check(eng, model, b, flat, gk, params, worst):
    """One Adam step (no clip) from zero moments with the kernel's own gradient, against float64 Adam; the absent
    head (a one-stage minibatch) untouched."""
    L = layout(model)
    live = np.ones(L.num_params, bool)
    for s, sl in heads(L).items():
        if not (b.stage == s).any():
            live[sl] = False
    want, m, v, _ = ON.adam_step(flat, 0.0, 0.0, 0.0, gk[:L.num_params].astype(np.float64), live)
    got = params.cpu().numpy()
    for s, sl in heads(L).items():
        if not live[sl].any():
            assert np.array_equal(got[sl], flat[sl])
    err = rel(got, want)
    worst["params"] = max(worst.get("params", 0.0), err)
    assert err < 1e-6, err
    mk, vk, steps = eng.get_opt_state()
    assert rel(mk, m) < 1e-5 and rel(vk, v) < 1.4e-5


@pytest.mark.parametrize("label", CASES)
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_graph_alone_matches_float64(model, label, dev):
    """One cap-sized graph in a launch of its own: forward outputs, every candidate's log-prob, greedy, the sampler's
    inverse CDF, the masked logit row, ppo_grad and one Adam step from the kernel's own state."""
    b = batch(label)
    flat = flat_params(model)
    eng = Engine(dev, b.n_cap, b.e_cap, model=model, grid_limit=GRID, clip_mode=_lib.CLIP_NEVER)
    try:
        worst = {}
        fw = check_forward(eng, model, b, flat, dev, worst=worst)
        sample_sweep(eng, model, b, flat, fw, dev, 64 if b.n_cap <= 1500 else 8)
        g, gk = check_grad(eng, model, b, flat, dev, worst=worst)
        params = t(flat, dev).clone()
        eng.apply(params, g)
        torch.cuda.synchronize()
        adam_check(eng, model, b, flat, gk, params, worst)
        report(f"{model} {'concept' if b.n_cap <= 1500 else 'abi'} alone", worst)
    finally:
        close(eng)


@pytest.mark.parametrize("name", ["concept", "abi"])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_mixed_launch_matches_float64_and_each_graph_alone(model, name, dev):
    """The cap-sized graphs and ordinary concept graphs in one launch, walked in order by one CTA (big -> small ->
    big) and then spread over GRID CTAs: float64 as above, and every forward output bit-identical to the graph's launch
    of its own."""
    b = batch(name)
    flat = flat_params(model)
    worst = {}
    alone = {}
    for label in b.labels:
        if label in ROWS:
            one = batch(label)
            e1 = Engine(dev, one.n_cap, one.e_cap, model=model, grid_limit=1)
            try:
                blob = pack_states(one.states).to(dev)
                alone[label] = [x.cpu().numpy() for x in e1.forward(blob, t(flat, dev), t(one.actions, dev),
                                                                  want_greedy=True, cand_log_probs=True)]
            finally:
                close(e1)
    for grid in (1, GRID):
        eng = Engine(dev, b.n_cap, b.e_cap, model=model, grid_limit=grid)
        try:
            assert eng.grid == grid
            fw = check_forward(eng, model, b, flat, dev, worst=worst)
            check_grad(eng, model, b, flat, dev, worst=worst)
        finally:
            close(eng)
        for i, label in enumerate(b.labels):
            if label not in alone:
                continue
            v, lp, en, gr, cand = alone[label]
            got = (fw["value"][i], fw["logp"][i], fw["ent"][i], fw["greedy"][i],
                   fw["cand"][fw["offs"][i]:fw["offs"][i] + cand.size])
            want = (v[0], lp[0], en[0], gr[0], cand)
            for what, x, y in zip(("value", "log_prob", "entropy", "greedy", "cand"), got, want):
                assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (label, grid, what)
    report(f"{model} {name} mixed", worst)


@pytest.mark.parametrize("name,grid", [("concept", 1), ("concept", 3), ("concept", 0), ("abi", 1), ("abi", 3)])
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_fused_step_matches_two_call_path(model, name, grid, dev):
    """upb_ppo_step against upb_ppo_grad + upb_apply over three steps (the first clips and runs the two-call path
    inside the library) at the tolerances of test_gpu_shapes.test_fused_tail_at_every_grid_size."""
    b = batch(name)
    flat = flat_params(model)
    L = layout(model)
    a = b.dev_args(model, flat, dev)
    n_ind = max(int((b.exps != 0).sum()), 1)
    blob = pack_states(b.states).to(dev)
    e1 = Engine(dev, b.n_cap, b.e_cap, model=model, grid_limit=grid)
    e2 = Engine(dev, b.n_cap, b.e_cap, model=model, grid_limit=grid)
    try:
        p1, p2 = t(flat, dev).clone(), t(flat, dev).clone()
        for step in range(3):
            before = e2.launches
            g1 = e1.ppo_grad(blob, p1, *a, 1.0 / b.count, 1.0 / n_ind)
            e1.apply(p1, g1)
            g2 = e2.ppo_step(blob, p2, *a, 1.0 / b.count, 1.0 / n_ind)
            torch.cuda.synchronize()
            assert (e2.launches - before == 1) == (step > 0)
            err, where = per_tensor_rel(g2.cpu().numpy()[:L.num_params], g1.cpu().numpy()[:L.num_params], L)
            assert err < 1e-5, (step, err, where)
            assert np.allclose(e2.read_losses(g2), e1.read_losses(g1), rtol=1e-5, atol=1e-6)
            assert rel(p2.cpu().numpy(), p1.cpu().numpy()) < 1e-6, step
        m1, v1, s1 = e1.get_opt_state()
        m2, v2, s2 = e2.get_opt_state()
        assert s1.tolist() == s2.tolist() == [3, 3, 3, 3]
        assert rel(m2, m1) < 1e-5 and rel(v2, v1) < 1e-5
    finally:
        close(e1, e2)
