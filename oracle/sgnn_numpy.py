"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Unpadded float64 numpy restatement of the reference's SGNN policy/value forward pass and a hand-derived
backward pass (SURVEY.md appendix A.2 / A.4 / A.7), one graph at a time.  It is the high-precision arbiter
for the CUDA kernels: the fp32 padded port (`oracle/torch_port.py`, itself pinned to the unmodified
reference by the golden fixtures) and this file must agree to fp32 round-off, and the CUDA path is then
compared with this file at tolerances far below the 1e-4 the task allows.

Reference sites restated (padded rows contribute exactly nothing, so unpadded evaluation is exact):
  urban_planning/models/state_encoder.py:184-214 (+ helpers :84-182)   encoder
  urban_planning/models/policy.py:45-104                               masked categorical heads
  urban_planning/models/value.py:36-39                                 value head
  khrylib/rl/agents/agent_pg.py:19-23, urban_planning/agents/urban_planning_agent.py:363-371   losses
  khrylib/rl/core/common.py:5-26                                       GAE
  torch.optim.Adam / clip_grad_norm_ as called from urban_planning_agent.py:145-149,336-337, agent_ppo.py:43-46
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from drl_urban_planning_b200 import params as PL

EPS_DEG = 1e-6
D = PL.GCN_DIM


@dataclass
class Graph:
    """One unpadded rollout state."""
    numerical: np.ndarray      # (52,)
    x: np.ndarray              # (n,23)
    edges: np.ndarray          # (e,2) int
    x_cur: np.ndarray          # (23,)
    lu_mask: np.ndarray        # (e,) bool
    road_mask: np.ndarray      # (n,) bool
    stage: np.ndarray          # (3,)
    n_cap: int                 # padded N (only used for the all-masked degenerate distribution)
    e_cap: int


def unpad(state: Sequence[np.ndarray]) -> Graph:
    """Reference 9-array state -> Graph.  Masks must be prefix masks (observation_extractor.py:60-66 pads
    an all-True vector with False), edges must join real nodes."""
    numerical, nf, ei, cur, nmask, emask, lum, rm, stage = state
    n, e = int(nmask.sum()), int(emask.sum())
    assert nmask[:n].all() and emask[:e].all(), "node/edge masks must be prefix masks"
    edges = np.asarray(ei[:e], dtype=np.int64)
    assert e == 0 or (edges.min() >= 0 and edges.max() < n), "real edges must join real nodes"
    assert not lum[e:].any() and not rm[n:].any(), "action masks must lie on real edges / nodes"
    return Graph(np.asarray(numerical, np.float64).reshape(-1), np.asarray(nf[:n], np.float64), edges,
                 np.asarray(cur, np.float64), np.asarray(lum[:e], bool), np.asarray(rm[:n], bool),
                 np.asarray(stage, np.float64), int(nf.shape[0]), int(ei.shape[0]))


def _p64(flat: np.ndarray) -> Dict[str, np.ndarray]:
    return {k: np.asarray(v, np.float64) for k, v in PL.unflatten(np.asarray(flat)).items()}


# ----------------------------------------------------------------------------- forward
def forward(P: Dict[str, np.ndarray], g: Graph, action: Optional[int] = None, keep: bool = False):
    """Returns dict with value, log_prob (of `action`, if given), entropy, greedy action, and (keep=True)
    every intermediate the backward needs."""
    n, e = g.x.shape[0], g.edges.shape[0]
    u, v = g.edges[:, 0], g.edges[:, 1]
    c = {}
    a0 = np.tanh(P["num_w0"] @ g.numerical + P["num_b0"])
    h_num = np.tanh(P["num_w1"] @ a0 + P["num_b1"])
    h = g.x @ P["enc_w"].T + P["enc_b"]
    hc = P["enc_w"] @ g.x_cur + P["enc_b"]
    deg = np.bincount(u, minlength=n) + np.bincount(v, minlength=n)
    inv = 1.0 / (deg + EPS_DEG)
    hs, t1s, t2s = [h], [], []
    he = np.zeros((e, D))
    for l in range(PL.NUM_GCN_LAYERS):
        W, b = P[f"gcn{l}_w"], P[f"gcn{l}_b"]
        Pn = h @ W[:, :D].T + b
        Qn = h @ W[:, D:].T
        t1 = np.tanh(Pn[u] + Qn[v])
        t2 = np.tanh(Pn[v] + Qn[u])
        he = 0.5 * (t1 + t2)
        S = np.zeros((n, D))
        np.add.at(S, u, he)
        np.add.at(S, v, he)
        h = h + S * inv[:, None]
        hs.append(h); t1s.append(t1); t2s.append(t2)
    m_e = he.mean(0) if e > 0 else np.full(D, np.nan)
    m_n = h.mean(0)
    # attention (state_encoder.py:150-161; nn.MultiheadAttention with 1 head, scale 1/sqrt(16))
    Wi, bi = P["mha_in_w"], P["mha_in_b"]
    q0 = P["att_q_w"] @ hc + P["att_q_b"]
    k0 = h @ P["att_k_w"].T + P["att_k_b"]
    v0 = h @ P["att_v_w"].T + P["att_v_b"]
    q1 = Wi[:D] @ q0 + bi[:D]
    k1 = k0 @ Wi[D:2 * D].T + bi[D:2 * D]
    v1 = v0 @ Wi[2 * D:].T + bi[2 * D:]
    s = k1 @ q1 / 4.0
    s = s - s.max()
    alpha = np.exp(s); alpha /= alpha.sum()
    ctx = alpha @ v1
    att = P["mha_out_w"] @ ctx + P["mha_out_b"]
    sv = np.concatenate([h_num, m_n, m_e, att, g.stage])
    y0 = np.tanh(P["val_w0"] @ sv + P["val_b0"])
    y1 = np.tanh(P["val_w1"] @ y0 + P["val_b1"])
    value = float(P["val_w2"].reshape(-1) @ y1 + P["val_b2"].reshape(-1)[0])

    stage_id = int(np.argmax(g.stage[:2])) if g.stage[:2].sum() > 0 else -1
    out = dict(value=value, log_prob=0.0, entropy=0.0, greedy=0, stage_id=stage_id)
    if stage_id == 0:
        idx = np.flatnonzero(g.lu_mask)
        xin = np.concatenate([he[idx], np.tile(hc, (idx.size, 1)), he[idx] * hc, he[idx] - hc], axis=1)
        th = np.tanh(xin @ P["lu_w0"].T + P["lu_b0"])
        z = th @ P["lu_w1"].reshape(-1)
        cap = g.e_cap
    elif stage_id == 1:
        idx = np.flatnonzero(g.road_mask)
        xin = h[idx]
        th = np.tanh(xin @ P["road_w0"].T + P["road_b0"])
        z = th @ P["road_w1"].reshape(-1)
        cap = g.n_cap
    if stage_id >= 0:
        if idx.size == 0:
            # every logit equals the fill value -> uniform over the padded width (policy.py:50-52)
            # every logit equals the fill value -2^32+1: in the reference's fp32 arithmetic logsumexp(logits) = fill
            # + log(cap) rounds back to fill (ulp 512), so the normalised logits are exactly 0: log_prob = 0, entropy = 0
            # (measured on the unmodified reference, tests/golden/edge_empty.npz), arg-max = first index
            out.update(log_prob=0.0, entropy=0.0, greedy=0)
            p = logp = np.zeros(0)
        else:
            zs = z - z.max()
            logp = zs - np.log(np.exp(zs).sum())
            p = np.exp(logp)
            out["entropy"] = float(-(p * logp).sum())
            out["greedy"] = int(idx[np.argmax(p)])         # argmax of probs, first max on ties
            if action is not None:
                pos = np.flatnonzero(idx == int(action))
                # an action outside the mask has logit == fill: log-prob = fill - logsumexp (finite, huge)
                out["log_prob"] = float(logp[pos[0]]) if pos.size else float(-2.0 ** 32 + 1 - z.max()
                                                                             - np.log(np.exp(zs).sum()))
                out["action_pos"] = int(pos[0]) if pos.size else -1
    if keep:
        c.update(a0=a0, h_num=h_num, hc=hc, hs=hs, t1s=t1s, t2s=t2s, he=he, inv=inv, m_e=m_e, m_n=m_n,
                 q0=q0, k0=k0, v0=v0, q1=q1, k1=k1, v1=v1, alpha=alpha, ctx=ctx, att=att, sv=sv, y0=y0,
                 y1=y1, u=u, v=v)
        if stage_id >= 0:
            c.update(idx=idx, xin=xin, th=th, p=p, logp=logp)
        out["cache"] = c
    return out


# ----------------------------------------------------------------------------- backward
def backward(P: Dict[str, np.ndarray], g: Graph, fw: dict, g_value: float, g_logp: float, g_ent: float,
             tile=np.matmul) -> Dict[str, np.ndarray]:
    """Gradient of  g_value*V + g_logp*log_prob + g_ent*entropy  w.r.t. all 32 tensors (A.7).  `tile(A, B)` forms the
    three products the CUDA backward runs as tensor-core tiles (GPQ^T h^l, GPQ Wpq, g_h0^T X); the default is A @ B
    (tests/bf16_oracle.py passes one that rounds the operands as the bf16-tile build does)."""
    c = fw["cache"]
    n, e = g.x.shape[0], g.edges.shape[0]
    u, v = c["u"], c["v"]
    G = {k: np.zeros_like(val) for k, val in P.items()}
    hL = c["hs"][-1]
    g_hL = np.zeros((n, D))
    g_he = np.zeros((e, D))
    g_hc = np.zeros(D)
    sid = fw["stage_id"]

    # ---- policy head (policy.py:49-61, 92-102)
    if sid >= 0 and c["idx"].size > 0:
        p, logp, idx, th, xin = c["p"], c["logp"], c["idx"], c["th"], c["xin"]
        H = fw["entropy"]
        g_z = -g_logp * p - g_ent * p * (logp + H)
        if fw.get("action_pos", -1) >= 0:
            g_z[fw["action_pos"]] += g_logp
        w0, w1 = ("lu_w0", "lu_w1") if sid == 0 else ("road_w0", "road_w1")
        b0 = "lu_b0" if sid == 0 else "road_b0"
        G[w1] += (g_z @ th).reshape(P[w1].shape)
        g_u = np.outer(g_z, P[w1].reshape(-1)) * (1 - th ** 2)
        G[w0] += g_u.T @ xin
        G[b0] += g_u.sum(0)
        g_x = g_u @ P[w0]
        if sid == 0:
            ga, gb, gc, gd = g_x[:, :D], g_x[:, D:2 * D], g_x[:, 2 * D:3 * D], g_x[:, 3 * D:]
            hc = c["hc"]
            g_he[idx] += ga + gc * hc + gd
            g_hc += (gb + gc * c["he"][idx] - gd).sum(0)
        else:
            g_hL[idx] += g_x

    # ---- value head (value.py:36-39)
    y0, y1, sv = c["y0"], c["y1"], c["sv"]
    G["val_b2"] += g_value
    G["val_w2"] += g_value * y1.reshape(1, -1)
    d1 = g_value * P["val_w2"].reshape(-1) * (1 - y1 ** 2)
    G["val_w1"] += np.outer(d1, y0); G["val_b1"] += d1
    d0 = (P["val_w1"].T @ d1) * (1 - y0 ** 2)
    G["val_w0"] += np.outer(d0, sv); G["val_b0"] += d0
    g_sv = P["val_w0"].T @ d0
    g_hnum, g_mn, g_me, g_att = g_sv[:16], g_sv[16:32], g_sv[32:48], g_sv[48:64]
    g_hL += g_mn / n
    if e > 0:
        g_he += g_me / e

    # ---- numeric encoder (state_encoder.py:35-57)
    dn1 = g_hnum * (1 - c["h_num"] ** 2)
    G["num_w1"] += np.outer(dn1, c["a0"]); G["num_b1"] += dn1
    dn0 = (P["num_w1"].T @ dn1) * (1 - c["a0"] ** 2)
    G["num_w0"] += np.outer(dn0, g.numerical); G["num_b0"] += dn0

    # ---- attention (state_encoder.py:150-161)
    Wi = P["mha_in_w"]
    G["mha_out_w"] += np.outer(g_att, c["ctx"]); G["mha_out_b"] += g_att
    g_ctx = P["mha_out_w"].T @ g_att
    g_v1 = np.outer(c["alpha"], g_ctx)
    g_alpha = c["v1"] @ g_ctx
    g_s = c["alpha"] * (g_alpha - (c["alpha"] * g_alpha).sum())
    g_q1 = (g_s @ c["k1"]) / 4.0
    g_k1 = np.outer(g_s, c["q1"]) / 4.0
    G["mha_in_w"][:D] += np.outer(g_q1, c["q0"]);      G["mha_in_b"][:D] += g_q1
    G["mha_in_w"][D:2 * D] += g_k1.T @ c["k0"];        G["mha_in_b"][D:2 * D] += g_k1.sum(0)
    G["mha_in_w"][2 * D:] += g_v1.T @ c["v0"];         G["mha_in_b"][2 * D:] += g_v1.sum(0)
    g_q0 = Wi[:D].T @ g_q1
    g_k0 = g_k1 @ Wi[D:2 * D]
    g_v0 = g_v1 @ Wi[2 * D:]
    G["att_q_w"] += np.outer(g_q0, c["hc"]); G["att_q_b"] += g_q0
    G["att_k_w"] += g_k0.T @ hL;             G["att_k_b"] += g_k0.sum(0)
    G["att_v_w"] += g_v0.T @ hL;             G["att_v_b"] += g_v0.sum(0)
    g_hc += P["att_q_w"].T @ g_q0
    g_hL += g_k0 @ P["att_k_w"] + g_v0 @ P["att_v_w"]

    # ---- GCN layers, last to first (state_encoder.py:110-148,194-197)
    g_h = g_hL
    for l in reversed(range(PL.NUM_GCN_LAYERS)):
        W = P[f"gcn{l}_w"]
        h_in = c["hs"][l]
        gs = g_h * c["inv"][:, None]
        ge = gs[u] + gs[v]
        if l == PL.NUM_GCN_LAYERS - 1:
            ge = ge + g_he
        g1 = 0.5 * ge * (1 - c["t1s"][l] ** 2)
        g2 = 0.5 * ge * (1 - c["t2s"][l] ** 2)
        gP = np.zeros((n, D)); gQ = np.zeros((n, D))
        np.add.at(gP, u, g1); np.add.at(gP, v, g2)
        np.add.at(gQ, v, g1); np.add.at(gQ, u, g2)
        G[f"gcn{l}_b"] += gP.sum(0)
        G[f"gcn{l}_w"][:, :D] += tile(gP.T, h_in)
        G[f"gcn{l}_w"][:, D:] += tile(gQ.T, h_in)
        g_h = g_h + tile(gP, W[:, :D]) + tile(gQ, W[:, D:])

    # ---- node encoder (state_encoder.py:189-191)
    G["enc_w"] += tile(g_h.T, g.x) + np.outer(g_hc, g.x_cur)
    G["enc_b"] += g_h.sum(0) + g_hc
    return G


# ----------------------------------------------------------------------------- minibatch loss
def ppo_minibatch(flat: np.ndarray, states: Sequence, actions: np.ndarray, advantages: np.ndarray,
                  returns: np.ndarray, fixed_log_probs: np.ndarray, exps: np.ndarray,
                  clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01, want_grad=True, tile=np.matmul):
    """Losses (loss, value_loss, surr_loss, entropy_loss), per-graph (value, log_prob, entropy) and the
    flat float64 gradient of the total loss for one minibatch (urban_planning_agent.py:322-333).  tile: see backward."""
    P = _p64(flat)
    B = len(states)
    adv = np.asarray(advantages, np.float64).reshape(-1)
    ret = np.asarray(returns, np.float64).reshape(-1)
    flp = np.asarray(fixed_log_probs, np.float64).reshape(-1)
    ind = np.flatnonzero(np.asarray(exps).reshape(-1) != 0)
    n_ind = max(len(ind), 1)
    in_ind = np.zeros(B, bool); in_ind[ind] = True
    vals, lps, ents = np.zeros(B), np.zeros(B), np.zeros(B)
    Gtot = {k: np.zeros_like(v) for k, v in P.items()}
    surr = vloss = eloss = 0.0
    for i, st in enumerate(states):
        g = unpad(st)
        sid = int(np.argmax(g.stage[:2]))
        a = int(actions[i, sid])
        fw = forward(P, g, action=a, keep=want_grad)
        vals[i], lps[i], ents[i] = fw["value"], fw["log_prob"], fw["entropy"]
        vloss += (fw["value"] - ret[i]) ** 2 / B
        g_lp = g_en = 0.0
        if in_ind[i]:
            r = np.exp(lps[i] - flp[i])
            s1, s2 = r * adv[i], np.clip(r, 1 - clip_epsilon, 1 + clip_epsilon) * adv[i]
            surr += -min(s1, s2) / n_ind
            eloss += -ents[i] / n_ind
            inside = (1 - clip_epsilon) <= r <= (1 + clip_epsilon)
            if inside or s1 < s2:
                g_lp = -adv[i] * r / n_ind
            if inside and s1 == s2:
                pass  # torch.min ties send the whole gradient through both equal branches -> same value
            g_en = -entropy_coef / n_ind
        if want_grad:
            g_v = 2.0 * value_pred_coef * (fw["value"] - ret[i]) / B
            Gi = backward(P, g, fw, g_v, g_lp, g_en, tile)
            for k in Gtot:
                Gtot[k] += Gi[k]
    loss = surr + value_pred_coef * vloss + entropy_coef * eloss
    grad = None
    if want_grad:
        grad = np.zeros(PL.NUM_PARAMS)
        for s in PL.SLOTS.values():
            grad[s.offset:s.offset + s.size] = Gtot[s.name].reshape(-1)
    return dict(loss=loss, value_loss=vloss, surr_loss=surr, entropy_loss=eloss, value=vals, log_prob=lps,
                entropy=ents, grad=grad)


# ----------------------------------------------------------------------------- clip + Adam
def clip_groups(grad: np.ndarray, max_norm: float = 1.0) -> np.ndarray:
    """The reference's first-step clipping: policy group then value group (agent_ppo.py:43-46,
    urban_planning_agent.py:46), torch.nn.utils.clip_grad_norm_ semantics (coef = min(1, max/(norm+1e-6)))."""
    g = np.array(grad, dtype=np.float64)
    pol = np.r_[0:PL.POLICY_END]
    val = np.r_[0:PL.ENCODER_END, PL.POLICY_END:PL.NUM_PARAMS]
    for sel in (pol, val):
        norm = np.sqrt((g[sel] ** 2).sum())
        g[sel] *= min(1.0, max_norm / (norm + 1e-6))
    return g


def adam_step(flat, m, v, t, grad, live, lr=4e-4, b1=0.9, b2=0.999, eps=1e-5):
    """torch.optim.Adam (no weight decay, no amsgrad) on the `live` entries; t is a per-entry step count."""
    flat, m, v, t = (np.array(a, dtype=np.float64) for a in (flat, m, v, t))
    t = t + live
    m = np.where(live, b1 * m + (1 - b1) * grad, m)
    v = np.where(live, b2 * v + (1 - b2) * grad * grad, v)
    tt = np.maximum(t, 1)
    step = lr / (1 - b1 ** tt)
    denom = np.sqrt(v) / np.sqrt(1 - b2 ** tt) + eps
    flat = np.where(live, flat - step * m / denom, flat)
    return flat, m, v, t


def live_mask(states: Sequence) -> np.ndarray:
    """Entries that receive a (non-None) gradient for this minibatch: everything except a policy head whose
    stage does not occur (policy.py:48,57; SURVEY A.6-7)."""
    live = np.ones(PL.NUM_PARAMS, bool)
    stages = np.array([int(np.argmax(np.asarray(st[8])[:2])) for st in states])
    if not (stages == 0).any():
        live[PL.SLOTS["lu_w0"].offset:PL.SLOTS["road_w0"].offset] = False
    if not (stages == 1).any():
        live[PL.SLOTS["road_w0"].offset:PL.POLICY_END] = False
    return live


# ----------------------------------------------------------------------------- GAE
def estimate_advantages(rewards, masks, values, gamma, tau):
    """khrylib/rl/core/common.py:5-26 in float32 with the reference's operation order."""
    r = np.asarray(rewards, np.float32).reshape(-1)
    mk = np.asarray(masks, np.float32).reshape(-1)
    val = np.asarray(values, np.float32).reshape(-1)
    T = r.shape[0]
    adv = np.zeros(T, np.float32)
    g32, gt32 = np.float32(gamma), np.float32(gamma * tau)
    prev_v = np.float32(0); prev_a = np.float32(0)
    for i in range(T - 1, -1, -1):
        delta = np.float32(np.float32(r[i] + np.float32(np.float32(g32 * prev_v) * mk[i])) - val[i])
        adv[i] = np.float32(delta + np.float32(np.float32(gt32 * prev_a) * mk[i]))
        prev_v, prev_a = val[i], adv[i]
    return adv.reshape(-1, 1), (val + adv).reshape(-1, 1)
