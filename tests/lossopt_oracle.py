"""Dual-clip PPO (Ye et al. 2020, Tianshou's PPOPolicy(dual_clip=c)) and the Huber value loss (MAPPO's use_huber_loss)
for the oracles, which implement neither.

Per graph with exps != 0, ratio r and advantage A (Tianshou's form):
    clip1 = min(r A, clamp(r, lo, hi) A),  surr = -(A < 0 ? max(clip1, c A) : clip1)
with c A constant: its gradient is clip1's where clip1 > c A, zero where c A > clip1 and half on a tie.
Per graph, the value term h(e) = 2 huber_loss(V, R, delta), e = V - R: e^2 inside delta, 2 delta (|e| - delta / 2)
beyond, with gradient 2 clamp(e, -delta, delta); with value clipping max(h(V - R), h(Vc - R)) under vclip_oracle's
tie and inclusive-clamp rules."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from drl_urban_planning_b200 import params as PL
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP


# ---- float64 per-graph terms ------------------------------------------------------------------------------------------
def surr64(r, A, lo, hi, dual_clip=None):
    """float64 per-graph (surrogate term -clip, d term / d r, dual bound strictly active)."""
    r, A = (np.asarray(x, np.float64).reshape(-1) for x in (r, A))
    s1, s2 = r * A, np.clip(r, lo, hi) * A
    clip1 = np.minimum(s1, s2)
    gr = np.where(((r >= lo) & (r <= hi)) | (s1 < s2), -A, 0.0)
    active = np.zeros(r.shape, bool)
    surr = -clip1
    if dual_clip is not None:
        cA = dual_clip * A
        neg = A < 0
        active = neg & (cA > clip1)
        tie = neg & (cA == clip1)
        surr = np.where(active, -cA, surr)
        gr = np.where(active, 0.0, np.where(tie, 0.5 * gr, gr))
    return surr, gr, active


def huber64(e, delta):
    """float64 (h(e), dh/de, linear branch) of h = 2 huber_loss; delta None: (e^2, 2 e, False)."""
    e = np.asarray(e, np.float64)
    if delta is None:
        return e * e, 2.0 * e, np.zeros(e.shape, bool)
    z = np.abs(e)
    return np.where(z < delta, z * z, 2.0 * delta * (z - 0.5 * delta)), 2.0 * np.clip(e, -delta, delta), z > delta


def value64(V, R, delta, V_old=None, value_clip=None):
    """float64 per-graph (d loss / dV, loss term, linear branch of the chosen term)."""
    V, R = (np.asarray(x, np.float64).reshape(-1) for x in (V, R))
    la, ga, lin_a = huber64(V - R, delta)
    if value_clip is None:
        return ga, la, lin_a
    V_old = np.asarray(V_old, np.float64).reshape(-1)
    d = V - V_old
    Vc = V_old + np.clip(d, -value_clip, value_clip)
    lb, gb, lin_b = huber64(Vc - R, delta)
    gb = np.where((d >= -value_clip) & (d <= value_clip), gb, 0.0)
    g = np.where(la > lb, ga, np.where(lb > la, gb, 0.5 * ga + 0.5 * gb))
    return g, np.maximum(la, lb), np.where(lb > la, lin_b, lin_a)


# ---- the kernels' fp32 seeds ------------------------------------------------------------------------------------------
def dual_seed32(r, A, lo, hi, c, inv_ind=1.0):
    """The step kernels' fp32 log-prob seed g_lp, surrogate term and dual-active flag from the kernel's own ratio r
    (softmax_seeds): g_lp = -A r (1/|ind|) where clip1 takes the ratio, 0 where c A > clip1, half on a tie."""
    f = np.float32
    r, A = (np.asarray(x, np.float32).reshape(-1) for x in (r, A))
    lo, hi = f(lo), f(hi)
    with np.errstate(over="ignore", invalid="ignore"):
        s1, s2 = f(r * A), f(np.minimum(np.maximum(r, lo), hi) * A)
        inside = (r >= lo) & (r <= hi)
        clip1 = np.minimum(s1, s2)
        glp = np.where(inside | (s1 < s2), f(f(-A * r) * f(inv_ind)), f(0))
        surr = -clip1
        active = np.zeros(r.shape, bool)
        if c is not None:
            cA = f(f(c) * A)
            neg = A < 0
            active = neg & (cA > clip1)
            tie = neg & (cA == clip1)
            surr = np.where(active, -cA, surr)
            glp = np.where(active, f(0), np.where(tie, f(f(0.5) * glp), glp))
    return glp.astype(np.float32), surr.astype(np.float32), active


def _h32(e, delta):
    f = np.float32
    z = np.abs(e)
    return np.where(z < delta, f(z * z), f(f(2) * f(delta * f(z - f(f(0.5) * delta)))))


def _clamp32(e, delta):
    return np.where(e < -delta, -delta, np.where(e > delta, delta, e)).astype(np.float32)


def value_seed32(V, R, delta, c_value=0.5, inv_batch=1.0, V_old=None, value_clip=None):
    """The step kernels' fp32 value seed g_V = 2 c_v clamp(e, -delta, delta) (1/B), the loss term and the linear-branch
    flag (value_seed): what one graph contributes to the value-head bias gradient and to slots 15 / 21.  delta None:
    the square."""
    f = np.float32
    V, R = (np.asarray(x, np.float32).reshape(-1) for x in (V, R))
    d32 = None if delta is None else f(delta)
    with np.errstate(over="ignore", invalid="ignore"):
        dv = f(V - R)
        sq = lambda e: f(e * e) if d32 is None else _h32(e, d32)                          # noqa: E731
        cl = lambda e: e if d32 is None else _clamp32(e, d32)                             # noqa: E731
        lin = lambda e: np.zeros(e.shape, bool) if d32 is None else np.abs(e) > d32        # noqa: E731
        if value_clip is None:
            gv = f(f(f(f(2) * f(c_value)) * cl(dv)) * f(inv_batch))
            return gv, sq(dv), lin(dv)
        c = f(value_clip)
        V_old = np.asarray(V_old, np.float32).reshape(-1)
        d = f(V - V_old)
        Vc = f(V_old + np.minimum(np.maximum(d, -c), c))
        dvc = f(Vc - R)
        la, lb = sq(dv), sq(dvc)
        ga, gb = f(f(2) * cl(dv)), np.where((d >= -c) & (d <= c), f(f(2) * cl(dvc)), f(0))
        g = np.where(la > lb, ga, np.where(lb > la, gb, f(f(f(0.5) * ga) + f(f(0.5) * gb))))
        gv = f(f(f(c_value) * g) * f(inv_batch))
        return gv, np.where(lb > la, lb, la), np.where(lb > la, lin(dvc), lin(dv))


# ---- torch forms (Tianshou / MAPPO) -----------------------------------------------------------------------------------
def surrogate(ratio, adv, clip_epsilon, dual_clip=None, reduce=True):
    """Tianshou's dual-clip surrogate: -where(A < 0, max(clip1, c A), clip1), averaged when reduce."""
    s1 = ratio * adv
    s2 = torch.clamp(ratio, 1.0 - clip_epsilon, 1.0 + clip_epsilon) * adv
    clip1 = torch.min(s1, s2)
    term = clip1 if dual_clip is None else torch.where(adv < 0, torch.max(clip1, dual_clip * adv), clip1)
    return -term.mean() if reduce else -term


def value_terms(v, ret, huber_delta=None, old_values=None, value_clip=None):
    """Per-graph value terms: (v - ret)^2 or 2 huber_loss(v, ret, delta), and with value_clip the max of the unclipped
    and clipped terms (MAPPO)."""
    def term(x):
        if huber_delta is None:
            return (x - ret).pow(2)
        return 2 * F.huber_loss(x, ret, reduction="none", delta=huber_delta)
    a = term(v)
    if value_clip is None:
        return a
    vc = old_values + torch.clamp(v - old_values, -value_clip, value_clip)
    return torch.max(a, term(vc))


# ---- the float64 minibatch oracle -------------------------------------------------------------------------------------
def ppo_minibatch(flat, states, actions, advantages, returns, fixed_log_probs, exps, dual_clip=None, huber_delta=None,
                  old_values=None, value_clip=None, clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01):
    """oracle/sgnn_numpy.ppo_minibatch with dual clip, the Huber value loss and (optionally) value clipping: float64
    losses, values, the flat gradient and the statistics sums of slots 15, 20 and 21."""
    P = ON._p64(flat)
    B = len(states)
    adv, ret, flp = (np.asarray(x, np.float64).reshape(-1) for x in (advantages, returns, fixed_log_probs))
    ind = np.flatnonzero(np.asarray(exps).reshape(-1) != 0)
    n_ind = max(len(ind), 1)
    fws, vals, lps = [], np.zeros(B), np.zeros(B)
    for i, st in enumerate(states):
        g = ON.unpad(st)
        sid = int(np.argmax(g.stage[:2]))
        fw = ON.forward(P, g, action=int(actions[i, sid]), keep=True)
        fws.append((g, fw))
        vals[i], lps[i] = fw["value"], fw["log_prob"]
    gv, vl_terms, linear = value64(vals, ret, huber_delta, old_values, value_clip)
    r = np.exp(lps - flp)
    s_terms, gr, active = surr64(r, adv, 1 - clip_epsilon, 1 + clip_epsilon, dual_clip)
    Gtot = {k: np.zeros_like(v) for k, v in P.items()}
    surr = eloss = 0.0
    dual = 0
    for i, (g, fw) in enumerate(fws):
        g_lp = g_en = 0.0
        if i in ind:
            surr += s_terms[i] / n_ind
            eloss += -fw["entropy"] / n_ind
            g_lp = gr[i] * r[i] / n_ind
            g_en = -entropy_coef / n_ind
            dual += int(active[i])
        Gi = ON.backward(P, g, fw, value_pred_coef * gv[i] / B, g_lp, g_en)
        for k in Gtot:
            Gtot[k] += Gi[k]
    vloss = vl_terms.sum() / B
    grad = np.zeros(PL.NUM_PARAMS)
    for s in PL.SLOTS.values():
        grad[s.offset:s.offset + s.size] = Gtot[s.name].reshape(-1)
    return dict(loss=surr + value_pred_coef * vloss + entropy_coef * eloss, value_loss=vloss, surr_loss=surr,
                entropy_loss=eloss, value=vals, grad=grad, value_loss_sum=vl_terms.sum(), dual=dual,
                linear=int(linear.sum()))


# ---- torch-port agents ------------------------------------------------------------------------------------------------
class PortAgent(TP.PortAgent):
    """oracle/torch_port.PortAgent with dual clip, the Huber value loss and value clipping against `old_values` (set
    per step when value_clip is on)."""

    def __init__(self, flat, dual_clip=None, huber_delta=None, value_clip=None, **kw):
        super().__init__(flat, **kw)
        self.dual_clip, self.huber_delta, self.value_clip, self.old_values = dual_clip, huber_delta, value_clip, None

    def backward(self, b, actions, advantages, returns, fixed_log_probs, ind):
        v = TP.value(self.P, b)
        lp, ent = TP.log_prob_entropy(self.P, b, actions)
        ratio = torch.exp(lp[ind] - fixed_log_probs[ind])
        surr = surrogate(ratio, advantages[ind], self.clip_epsilon, self.dual_clip)
        vl = value_terms(v, returns, self.huber_delta, self.old_values, self.value_clip).mean()
        el = -ent[ind].mean()
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el
        self.opt.zero_grad()
        loss.backward()
        return loss.item(), vl.item(), surr.item(), el.item()


class MLPPortAgent(MP.MLPPortAgent):
    """oracle/mlp_port.MLPPortAgent with the same options."""

    def __init__(self, flat, dual_clip=None, huber_delta=None, value_clip=None, **kw):
        super().__init__(flat, **kw)
        self.dual_clip, self.huber_delta, self.value_clip, self.old_values = dual_clip, huber_delta, value_clip, None

    def backward(self, b, actions, adv, ret, fixed, ind):
        v = MP.value(self.P, b)
        lp, ent = MP.log_prob_entropy(self.P, b, actions)
        ratio = torch.exp(lp[ind] - fixed.to(lp.dtype)[ind])
        surr = surrogate(ratio, adv.to(lp.dtype)[ind], self.clip_epsilon, self.dual_clip)
        ov = None if self.old_values is None else self.old_values.to(v.dtype)
        vl = value_terms(v, ret.to(v.dtype), self.huber_delta, ov, self.value_clip).mean()
        el = -ent[ind].mean()
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el
        self.opt.zero_grad()
        loss.backward()
        return loss.item(), vl.item(), surr.item(), el.item()
