"""Parameter transforms and minibatches for the magnitude regimes of tests/test_gpu_extremes.py, shared with the
golden-vector generator tests/golden/make_golden_extremes.py (which records the unmodified reference on them).

Each `*_case` has make_golden.run_fixture's hook signature f(flat, states, actions, adv, ret, exps) -> overrides: it
transforms the given initial parameters and builds its own states, actions and PPO targets from fixed seeds."""
import math

import numpy as np
import torch

from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.packing import pack_states
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from shape_cases import big_states

CLAMP = 40.0                # exp2a clamps 2a to +-80 (sgnn_kernel.cuh)
OFF_COL = PL.NODE_DIM - 1   # a uniform(-1, 1) feature column, turned into a per-graph common embedding offset
# node-factor targets per graph, cycled: below the clamp's neighbourhood, in [38, 40), beyond it
TARGETS = [None, 39.0, 70.0, 38.4, 160.0, 45.0]
LOG_TINY = math.log(2.0 ** -149)          # below this a probability is under the smallest fp32 denormal


def slot(flat, name, layout=PL.SGNN):
    s = layout.slots[name]
    return flat[s.offset:s.offset + s.size].reshape(s.shape)      # a view: writes go to `flat`


def targets(seed, count):
    adv, ret, exps = synth.make_ppo_targets(seed, count)
    exps[::7] = 0.0
    return adv, ret, exps


# ---------------------------------------------------------------------------------------------------- GCN factors
def graph_reciprocal_tiers(P, state):
    """Per GCN layer, which form of the pull's tanh terms the kernel picks for one graph (sgnn_kernel.cuh fwd_term /
    bwd_term), from the oracle's float64 activations under the parameters `P` (ON._p64): 0 = one shared reciprocal per
    entry (|pre-activation| <= 10.9), 1 = the exact two."""
    hs = ON.forward(P, ON.unpad(state), keep=True)["cache"]["hs"]
    tiers = []
    for l in range(2):
        W, b = P[f"gcn{l}_w"], P[f"gcn{l}_b"]
        amax = max(np.abs(hs[l] @ W[:, :16].T + b).max(), np.abs(hs[l] @ W[:, 16:].T).max())
        assert amax < 38.0, "beyond the exp-form's clamp (|pre-activation| <= 40): not a case these tests are for"
        tiers.append(0 if amax <= 10.9 else 1)
    return tiers


def edge_amax(P, state):
    """Per GCN layer, from the oracle's float64 activations: (max |node factor| over P_i = W_a h_i + b and
    Q_i = W_b h_i, max |P_u + Q_v| over the directed edge entries)."""
    g = ON.unpad(state)
    hs = ON.forward(P, g, keep=True)["cache"]["hs"]
    u, v = g.edges[:, 0], g.edges[:, 1]
    out = []
    for l in range(2):
        W, b = P[f"gcn{l}_w"], P[f"gcn{l}_b"]
        Pn, Qn = hs[l] @ W[:, :16].T + b, hs[l] @ W[:, 16:].T
        edge = max(np.abs(Pn[u] + Qn[v]).max(), np.abs(Pn[v] + Qn[u]).max()) if len(u) else 0.0
        out.append((max(np.abs(Pn).max(), np.abs(Qn).max()), edge))
    return out


def difference_detector(flat, layers, s, sign=-1.0):
    """GCN layers in `layers` become [s A | -s A] (A = the given W_a), so P_u + Q_v = s A (h_u - h_v) + b stays
    moderate while P and Q grow with a common offset of the embeddings (sign = +1: [s A | s A], the edge pre-activation
    grows with them); the other layer is made blind to that offset (zero row sums).  enc_w's column OFF_COL becomes all
    ones: a node's feature OFF_COL is added to every channel of its embedding."""
    out = np.array(flat, np.float32)
    for l in range(2):
        W = slot(out, f"gcn{l}_w")
        if l in layers:
            A = W[:, :16].copy()
            W[:, :16], W[:, 16:] = s * A, sign * s * A
        else:
            W[:, :16] -= W[:, :16].mean(1, keepdims=True)
            W[:, 16:] -= W[:, 16:].mean(1, keepdims=True)
    slot(out, "enc_w")[:, OFF_COL] = 1.0
    return out


def with_offset(state, c):
    st = [a.copy() for a in state]
    st[1][st[4], OFF_COL] = c
    return st


def place_offsets(flat, states, layers, want):
    """Per graph, the offset c (bisection) that brings the largest node factor of `layers` to want[i] (None: c = 0)."""
    P = ON._p64(flat)
    amax = lambda st: max(edge_amax(P, st)[l][0] for l in layers)
    out = []
    for st, w in zip(states, want):
        if w is None:
            out.append(with_offset(st, 0.0))
            continue
        lo, hi = 0.0, 256.0
        assert amax(with_offset(st, lo)) < w < amax(with_offset(st, hi))
        for _ in range(40):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if amax(with_offset(st, mid)) < w else (lo, mid)
        out.append(with_offset(st, np.float32(0.5 * (lo + hi))))
    return out


def small_clamp_batch(flat, layers, seed=5):
    """24 `small` graphs of both stages, difference-detector weights on `layers`, offsets straddling the clamp."""
    states, actions = synth.make_states(seed, "small", 24)
    flat = difference_detector(flat, layers, 4.0)
    states = place_offsets(flat, states, layers, [TARGETS[i % len(TARGETS)] for i in range(len(states))])
    return flat, states, actions


def clamp_case(flat, *_):
    """Both layers beyond the clamp on four graphs past the shared-memory path (1000 / 3000 caps) and four fast ones
    in the same launch."""
    states, actions = big_states(9, 4)
    spec = synth.CommunitySpec("big", 1000, 3000, 470, 1000, 3.0, 0.3)
    rng = np.random.default_rng(10)
    for i, n in enumerate((40, 60, 90, 120)):
        st, a = synth.make_state(rng, spec, n=n, stage=i % 2)
        states.append(st)
        row = np.zeros((1, 2), np.float32)
        row[0, i % 2] = a
        actions = np.vstack([actions, row])
    flat = difference_detector(flat, [0, 1], 4.0)
    states = place_offsets(flat, states, [0, 1], [TARGETS[i % len(TARGETS)] for i in range(len(states))])
    adv, ret, exps = targets(9, len(states))
    return dict(params=flat, states=states, actions=actions, advantages=adv, returns=ret, exps=exps)


# ---------------------------------------------------------------------------------------------------- attention
def attention_logits(P, state):
    c = ON.forward(P, ON.unpad(state), keep=True)["cache"]
    return c["k1"] @ c["q1"] / 4.0


def attention_case(flat, *_):
    """12 `small` graphs plus one with two isolated nodes of identical features lifted above every other node's
    attention logit (a tie at the maximum); the key projection scaled until every graph's logits span 1.5 x 104."""
    seed = 8
    flat = np.array(flat, np.float32)
    states, actions = synth.make_states(seed, "small", 12)
    P = ON._p64(flat)
    st, a = synth.make_exact_state(np.random.default_rng(seed), synth.COMMUNITIES["small"], 40, 50, 5, 0, isolated=2)
    g = ON.unpad(st)
    lone = np.setdiff1d(np.arange(g.x.shape[0]), g.edges.ravel())
    c = ON.forward(P, g, keep=True)["cache"]
    w = P["enc_w"].T @ (P["att_k_w"].T @ (P["mha_in_w"][16:32].T @ c["q1"])) / 4.0   # d s_i / d x_i, isolated node
    s = c["k1"] @ c["q1"] / 4.0
    lift = (np.delete(s, lone).max() + 3.0 - s[lone[0]]) / (w @ w)
    st[1][lone] = (st[1][lone[0]].astype(np.float64) + max(lift, 0.0) * w).astype(np.float32)
    states.append(st)
    actions = np.vstack([actions, np.array([[a, 0]], np.float32)])
    f = 1.5 * 104.0 / min(np.ptp(attention_logits(P, s)) for s in states)
    slot(flat, "mha_in_w")[16:32] *= np.float32(f)
    adv, ret, exps = targets(seed, len(states))
    return dict(params=flat, states=states, actions=actions, advantages=adv, returns=ret, exps=exps)


# ---------------------------------------------------------------------------------------------------- policy heads
RATIOS = [1.0, 0.5, 2.0, 0.0]        # inside [1 - eps, 1 + eps], below, above, underflowing to 0
ADVS = [1.0, -1.0, 0.0]


def scaled_head(model, flat, stage, scale):
    """`flat` with the output layer of the stage's policy head (lu_w1 / road_w1, no bias) times `scale`: every logit of
    that head is scaled by the same factor, up to the fp32 rounding of the scaled weights."""
    out = flat.copy()
    sl = (PL.SLOTS if model == "sgnn" else PL.MLP.slots)["lu_w1" if stage == 0 else "road_w1"]
    out[sl.offset:sl.offset + sl.size] *= np.float32(scale)
    return out


def head_logits(model, flat, states):
    """Per graph: the candidate indices and their float64 logits."""
    out = []
    if model == "sgnn":
        P = ON._p64(flat)
        for st in states:
            fw = ON.forward(P, ON.unpad(st), keep=True)
            c = fw["cache"]
            out.append((c["idx"], c["th"] @ P["lu_w1" if fw["stage_id"] == 0 else "road_w1"].reshape(-1)))
        return out
    P = MP.params_from_flat(flat, torch.float64)
    with torch.no_grad():
        zl, zr = MP.masked_logits(P, MP.stack_states(states))
    for i, st in enumerate(states):
        stage = int(np.argmax(st[8][:2]))
        idx = np.flatnonzero(st[6] if stage == 0 else st[7])
        out.append((idx, (zl if stage == 0 else zr)[i].numpy()[idx]))
    return out


def log_softmax(z):
    zs = z - z.max()
    return zs - np.log(np.exp(zs).sum())


def heads_case(model):
    """Both heads' output layers scaled (scaled_head) until the median logit span passes 150; actions cycle through
    the arg-max, a candidate of fp32 probability 0 (float64 log-prob below log 2^-149) and a masked one; old log-probs
    put the ratio inside, below and above the clip range and underflow it, each with A > 0, A < 0 and A = 0.  A masked
    action's log-prob is the fill value (ulp 512 in fp32), so its ratio only ever underflows; a zero-probability
    action's ratio sits inside the range only with A = 0, so its fp32 log-prob error does not enter the gradient."""
    def case(flat, *_):
        seed = 12
        states, actions = synth.make_states(seed, "small", 36)
        flat = np.array(flat, np.float32)
        span = np.median([np.ptp(z) for idx, z in head_logits(model, flat, states) if idx.size > 1])
        for stage in (0, 1):
            flat = scaled_head(model, flat, stage, 150.0 / span)
        heads = head_logits(model, flat, states)
        adv, ret, exps = synth.make_ppo_targets(seed, len(states))
        fixed = np.zeros((len(states), 1), np.float32)
        count = [0, 0, 0]
        for i, st in enumerate(states):
            stage = int(np.argmax(st[8][:2]))
            idx, lp = heads[i][0], log_softmax(heads[i][1])
            kind = i % 3
            if kind == 1 and not (lp < LOG_TINY).any():
                kind = 0
            c, count[kind] = count[kind], count[kind] + 1
            if kind == 0:
                pos = int(np.argmax(lp))
                r, A = RATIOS[c % 4], ADVS[(c // 4) % 3]
                fixed[i] = lp[pos] + 200.0 if r == 0.0 else lp[pos] - np.log(r)
            elif kind == 1:
                pos = int(np.flatnonzero(lp < LOG_TINY)[0])
                A = ADVS[c % 3]
                fixed[i] = lp[pos] if A == 0.0 else lp[pos] + 200.0
            if kind < 2:
                j = int(idx[pos])
            else:
                cap = len(st[6]) if stage == 0 else len(st[7])
                j = int(np.setdiff1d(np.arange(cap), idx)[0])
                A = ADVS[c % 3]
                fixed[i] = -3.0
            actions[i, stage] = j
            adv[i] = A
        return dict(params=flat, states=states, actions=actions, advantages=adv, returns=ret, exps=exps,
                    fixed_log_probs=fixed)
    return case


# ---------------------------------------------------------------------------------------------------- saturated tanh
def tanh_case(model):
    """Numeric-encoder and value-head weights x40, policy-head hidden layers x100: most pre-activations pass |9|."""
    layout = PL.SGNN if model == "sgnn" else PL.MLP

    def case(flat, *_):
        seed = 14
        states, actions = synth.make_states(seed, "small", 16)
        flat = np.array(flat, np.float32)
        for name in ("num_w0", "num_w1", "val_w0", "val_w1"):
            slot(flat, name, layout)[:] *= 40.0
        for name in ("lu_w0", "road_w0"):
            slot(flat, name, layout)[:] *= 100.0
        adv, ret, exps = targets(seed, len(states))
        return dict(params=flat, states=states, actions=actions, advantages=adv, returns=ret, exps=exps)
    return case


# ---------------------------------------------------------------------------------------------------- float64 results
def sgnn_reference(flat, states, actions, adv, ret, fixed, exps):
    """Oracle results plus per-graph greedy, largest |logit| and near-tie flag, and the float64 parameters after the
    engine's first (clipped) Adam step."""
    ref = ON.ppo_minibatch(flat, states, actions, adv, ret, fixed, exps)
    P = ON._p64(flat)
    ref["greedy"], ref["zabs"], ref["tie"] = [], [], []
    for st in states:
        fw = ON.forward(P, ON.unpad(st), keep=True)
        c = fw["cache"]
        z = c["th"] @ P["lu_w1" if fw["stage_id"] == 0 else "road_w1"].reshape(-1) if c["idx"].size else np.zeros(1)
        top = np.sort(z)[::-1]
        ref["greedy"].append(fw["greedy"])
        ref["zabs"].append(np.abs(z).max())
        ref["tie"].append(len(top) > 1 and top[0] - top[1] < 1e-4 * (1.0 + np.abs(z).max()))
    ref["after"] = ON.adam_step(flat, 0.0, 0.0, 0.0, ON.clip_groups(ref["grad"]), ON.live_mask(states))[0]
    return ref


def mlp_reference(flat, states, actions, adv, ret, fixed, exps):
    """The same for the rl-mlp: the port in float64, autograd, torch's Adam after the reference's first-step clip."""
    b, act = MP.stack_states(states), torch.tensor(actions)
    ind = torch.tensor(exps).nonzero(as_tuple=False).squeeze(1)
    agent = MP.MLPPortAgent(flat, dtype=torch.float64)
    with torch.no_grad():
        v = MP.value(agent.P, b).numpy().ravel()
        lp, en = MP.log_prob_entropy(agent.P, b, act)
        zl, zr = MP.masked_logits(agent.P, b)
    losses = agent.backward(b, act, torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    ref = dict(value=v, log_prob=lp.numpy().ravel(), entropy=en.numpy().ravel(), grad=agent.flat_grad())
    ref.update(loss=losses[0], value_loss=losses[1], surr_loss=losses[2], entropy_loss=losses[3])
    ref["greedy"], ref["zabs"], ref["tie"] = [], [], []
    for i, st in enumerate(states):
        stage = int(np.argmax(st[8][:2]))
        idx = np.flatnonzero(st[6] if stage == 0 else st[7])
        z = (zl if stage == 0 else zr)[i].numpy()[idx] if idx.size else np.zeros(1)
        top = np.sort(z)[::-1]
        ref["greedy"].append(int(idx[np.argmax(z)]) if idx.size else 0)
        ref["zabs"].append(np.abs(z).max())
        ref["tie"].append(len(top) > 1 and top[0] - top[1] < 1e-4 * (1.0 + np.abs(z).max()))
    for names in agent.groups:
        torch.nn.utils.clip_grad_norm_([agent.P[n] for n in names], 1.0)
    agent.opt.step()
    ref["after"] = agent.flat()
    return ref


def reference_deviation(model, z, ref):
    """Per tensor, max|delta| / max|float64| of the reference's recorded first-step gradient (fixture z) from the
    float64 oracle's: how far the reference's own fp32 arithmetic lands from exact in this regime."""
    slots = PL.SLOTS if model == "sgnn" else PL.MLP.slots
    out = {}
    for s in slots.values():
        a, b = z["grads"][0][s.offset:s.offset + s.size], ref["grad"][s.offset:s.offset + s.size]
        out[s.name] = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
    return out


# ---------------------------------------------------------------------------------------------------- regimes
def tier(amax):
    """The form of the pull's tanh terms the kernel picks for a layer (sgnn_kernel.cuh epq_phase): 0 = one shared
    reciprocal (<= 10.9, as graph_reciprocal_tiers), 1 = two, 2 = raw pre-activations (beyond the
    clamp)."""
    return 0 if amax <= 10.9 else 1 if amax <= CLAMP else 2


def assert_beyond_clamp(flat, states, layers):
    """From the float64 activations: every form occurs, some graph lies in [38, 40) and some beyond the clamp on each
    layer in `layers` (both stages), while edge pre-activations stay below it."""
    P = ON._p64(flat)
    am = [edge_amax(P, st) for st in states]
    amax, emax = np.array([[a for a, _ in x] for x in am]), np.array([[e for _, e in x] for x in am])
    stage = np.array([int(np.argmax(st[8][:2])) for st in states])
    top = amax[:, layers].max(1)
    assert {tier(a) for a in amax.ravel()} == {0, 1, 2}, amax
    assert ((top >= 38.0) & (top < CLAMP)).any(), top
    for l in layers:
        for s in (0, 1):
            assert (amax[stage == s, l] > CLAMP).any(), (l, s, amax[:, l])
    assert emax.max() < 20.0, emax


def pre_activations(model, flat, states):
    """Float64 pre-activations of the numeric encoder, value head and policy-head hidden layers over the batch."""
    if model == "sgnn":
        P = ON._p64(flat)
        pre = {k: [] for k in ("num", "val", "head")}
        for st in states:
            fw = ON.forward(P, ON.unpad(st), keep=True)
            c = fw["cache"]
            pre["num"] += [P["num_w0"] @ ON.unpad(st).numerical + P["num_b0"], P["num_w1"] @ c["a0"] + P["num_b1"]]
            pre["val"] += [P["val_w0"] @ c["sv"] + P["val_b0"], P["val_w1"] @ c["y0"] + P["val_b1"]]
            if c["idx"].size:
                w0, b0 = ("lu_w0", "lu_b0") if fw["stage_id"] == 0 else ("road_w0", "road_b0")
                pre["head"].append((c["xin"] @ P[w0].T + P[b0]).ravel())
        return {k: np.concatenate(v) for k, v in pre.items()}
    P = MP.params_from_flat(flat, torch.float64)
    b = MP.stack_states(states)
    with torch.no_grad():
        lu, hn, sv = MP.encode(P, b)
        a0 = b["numerical"].double() @ P["num_w0"].T + P["num_b0"]
        a1 = torch.tanh(a0) @ P["num_w1"].T + P["num_b1"]
        y0 = sv @ P["val_w0"].T + P["val_b0"]
        y1 = torch.tanh(y0) @ P["val_w1"].T + P["val_b1"]
        hl = (lu @ P["lu_w0"].T + P["lu_b0"])[b["land_use_mask"]]
        hr = (hn @ P["road_w0"].T + P["road_b0"])[b["road_mask"]]
    cat = lambda *x: np.concatenate([np.asarray(v).ravel() for v in x])
    return {"num": cat(a0, a1), "val": cat(y0, y1), "head": cat(hl, hr)}


def assert_regime(name, model, flat, states, actions, fixed, adv):
    """The golden batch `name` is in its regime, from the oracle's float64 activations."""
    if name == "extreme_clamp":
        info = pack_states(states).info
        assert (info[:, 0] > 464).any() and (info[:, 0] <= 464).any()
        assert_beyond_clamp(flat, states, [0, 1])
    elif name == "extreme_attention":
        P = ON._p64(flat)
        spans = [np.ptp(attention_logits(P, st)) for st in states]
        assert min(spans) > 104.0, spans
        s = attention_logits(P, states[-1])
        top = np.sort(s)
        assert np.isclose(top[-1], top[-2], rtol=1e-12, atol=0) and top[-3] < top[-1] - 1.0
    elif name.endswith("heads"):
        heads = head_logits(model, flat, states)
        assert np.median([np.ptp(z) for idx, z in heads if idx.size > 1]) > 104.0
        seen = set()
        for i, st in enumerate(states):
            stage = int(np.argmax(st[8][:2]))
            idx, lp = heads[i][0], log_softmax(heads[i][1])
            j = int(actions[i, stage])
            if j not in idx:
                seen.add(("masked", None, float(adv[i])))
                continue
            lpa = lp[int(np.flatnonzero(idx == j)[0])]
            kind = "argmax" if lpa == lp.max() else "zero" if lpa < LOG_TINY else "other"
            r = np.exp(lpa - float(fixed[i]))
            seen.add((kind, 0 if r < 1e-30 else -1 if r < 0.8 else 1 if r > 1.2 else 0.5, float(adv[i])))
        assert {k for k, _, _ in seen} >= {"argmax", "zero", "masked"}, seen
        assert {(r, a) for k, r, a in seen if k == "argmax"} == {(r, a) for r in (0.5, -1, 1, 0) for a in ADVS}
    else:
        for k, v in pre_activations(model, flat, states).items():
            assert (np.abs(v) > 9.0).mean() > 0.3, (k, (np.abs(v) > 9.0).mean())


# name, community (model caps), rl-mlp, case
FIXTURES = [
    ("extreme_clamp", "hlg", False, clamp_case),
    ("extreme_attention", "small", False, attention_case),
    ("extreme_heads", "small", False, heads_case("sgnn")),
    ("extreme_tanh", "small", False, tanh_case("sgnn")),
    ("mlp_extreme_heads", "small", True, heads_case("mlp")),
    ("mlp_extreme_tanh", "small", True, tanh_case("mlp")),
]
