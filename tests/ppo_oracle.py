"""The PPO minibatch with every loss option, in float64 for both models, and the torch-port agents that train with the
options.  The oracles (oracle/) implement the reference's loss only; the options are:

  * value_clip (OpenAI baselines' ppo2, CleanRL's clip_vloss): d = V - V_old, Vc = V_old + clamp(d, -c, c), the term
    max(h(V - R), h(Vc - R)).  Its gradient is autograd's for torch.maximum (a tie sends half to each input) and the
    inclusive clamp.
  * huber_delta (MAPPO's use_huber_loss): h(e) = 2 huber_loss = e^2 inside delta, 2 delta (|e| - delta / 2) beyond,
    with gradient 2 clamp(e, -delta, delta).  Without it h(e) = e^2.
  * dual_clip (Ye et al. 2020, Tianshou's PPOPolicy(dual_clip=c)): clip1 = min(r A, clamp(r, lo, hi) A),
    surr = -(A < 0 ? max(clip1, c A) : clip1).  c A is constant: the gradient is clip1's where clip1 > c A, zero where
    c A > clip1 and half on a tie.
  * kl_coef (upb_set_kl_penalty), on the exact categorical KL against the update's pre-pass policy: for a graph with
    candidates c, KL_g = sum_c p_old(c) (lp_old(c) - lp(c)) and d KL_g / d z(c) = p(c) - p_old(c).  The sum is taken
    in log space, so a new probability that underflows gives a large finite term and a p_old that underflows adds 0.
    The penalty is kl_coef (1/|ind|) sum over ind of KL_g.
  * prox_flat, the EWMA proximal policy (PPO-EWMA, upb_set_prox_ewma): r = exp(lp - lp_p), the constant weight
    w = exp(lp_p - lp_b) and surr = -w min(r A, clamp(r) A).  Since w > 0 this is the surrogate at the anchor lp_p with
    A' = w A (the dual clip's bound likewise).  The value loss, the entropy and the KL penalty do not see w.

The statistics sums carry the step kernels' slot numbers: 1 surr_sum, 2 ent_sum, 3 n, 4 n_ind, 15 value_loss_sum,
16 clipped, 18 kl_sum, 20 dual, 21 linear, 23 prox_weight and 24 prox_kl."""
from __future__ import annotations

import types

import numpy as np
import torch
import torch.nn.functional as F

import klpen_oracle as KO
from drl_urban_planning_b200 import params as PL
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP


def _col(x):
    return np.asarray(x, np.float64).reshape(-1)


# ---- float64 per-graph terms ------------------------------------------------------------------------------------------
def surr64(r, A, lo, hi, dual_clip=None):
    """float64 per-graph (surrogate term, d term / d r, dual bound strictly active)."""
    r, A = _col(r), _col(A)
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
    """float64 (h(e), dh/de, linear branch).  Without delta the square is pow's, as sgnn_numpy.ppo_minibatch's scalar
    (V - R) ** 2 rounds (numpy squares an array as e * e)."""
    e = np.asarray(e, np.float64)
    if delta is None:
        return np.float_power(e, 2), 2.0 * e, np.zeros(e.shape, bool)
    z = np.abs(e)
    return np.where(z < delta, z * z, 2.0 * delta * (z - 0.5 * delta)), 2.0 * np.clip(e, -delta, delta), z > delta


def value64(V, R, delta=None, V_old=None, value_clip=None):
    """float64 per-graph (d term / dV, value term, clipped branch taken, linear branch of the chosen term)."""
    V, R = _col(V), _col(R)
    la, ga, lin_a = huber64(V - R, delta)
    if value_clip is None:
        return ga, la, np.zeros(V.shape, bool), lin_a
    V_old = _col(V_old)
    d = V - V_old
    Vc = V_old + np.clip(d, -value_clip, value_clip)
    lb, gb, lin_b = huber64(Vc - R, delta)
    gb = np.where((d >= -value_clip) & (d <= value_clip), gb, 0.0)
    g = np.where(la > lb, ga, np.where(lb > la, gb, 0.5 * ga + 0.5 * gb))
    return g, np.maximum(la, lb), lb > la, np.where(lb > la, lin_b, lin_a)


def kl64(lp_old, lp):
    """float64 (KL_g, d KL_g / d z) of one graph from its candidates' old and new log-probs (any order, same for both)."""
    lo, ln = np.asarray(lp_old, np.float64), np.asarray(lp, np.float64)
    po, p = np.exp(lo), np.exp(ln)
    return float(np.where(po > 0, po * (lo - ln), 0.0).sum()), p - po


def weights64(lp_p, lp_b):
    """float64 per-graph behaviour weight w = exp(lp_p - lp_b) and the KL estimate expm1(d) - d (slots 23, 24)."""
    d = _col(lp_p) - _col(lp_b)
    return np.exp(d), np.expm1(d) - d


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


def value_seed32(V, R, delta=None, c_value=0.5, inv_batch=1.0, V_old=None, value_clip=None):
    """The step kernels' fp32 value seed g_V = 2 c_v clamp(e, -delta, delta) (1/B), the value term, and the clipped and
    linear-branch flags (value_seed), with their rounding: what one graph contributes to the value-head bias gradient
    and to slots 15, 16 and 21.  delta None: the square."""
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
            return gv, sq(dv), np.zeros(V.shape, bool), lin(dv)
        c = f(value_clip)
        V_old = np.asarray(V_old, np.float32).reshape(-1)
        d = f(V - V_old)
        Vc = f(V_old + np.minimum(np.maximum(d, -c), c))
        dvc = f(Vc - R)
        la, lb = sq(dv), sq(dvc)
        ga, gb = f(f(2) * cl(dv)), np.where((d >= -c) & (d <= c), f(f(2) * cl(dvc)), f(0))
        g = np.where(la > lb, ga, np.where(lb > la, gb, f(f(f(0.5) * ga) + f(f(0.5) * gb))))
        gv = f(f(f(c_value) * g) * f(inv_batch))
        return gv, np.where(lb > la, lb, la), lb > la, np.where(lb > la, lin(dvc), lin(dv))


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


# ---- the float64 minibatch --------------------------------------------------------------------------------------------
def _anchor(adv, fixed, lp_p):
    """The surrogate's advantages and anchor, and the per-graph prox weight and KL estimate (zero without lp_p)."""
    A, lp_b = _col(adv), _col(fixed)
    if lp_p is None:
        return A, lp_b, np.zeros(A.size), np.zeros(A.size)
    w, kl = weights64(lp_p, lp_b)
    return w * A, _col(lp_p), w, kl


def _terms(V, lp, adv, ret, fixed, exps, lp_p, *, clip_epsilon, old_values, value_clip, huber_delta, dual_clip):
    """Every per-graph float64 term of a minibatch from its values and log-probs."""
    t = types.SimpleNamespace(V=V, lp=lp, ind=np.asarray(exps).reshape(-1) != 0)
    t.A, t.anchor, t.w, t.pkl = _anchor(adv, fixed, lp_p)
    t.r = np.exp(lp - t.anchor)
    t.surr, t.g_r, t.dual = surr64(t.r, t.A, 1 - clip_epsilon, 1 + clip_epsilon, dual_clip)
    t.g_v, t.vterm, t.clipped, t.linear = value64(V, ret, huber_delta, old_values, value_clip)
    return t


def _result(t, ents, kl_g, lp_p, grad, **losses):
    ind = t.ind
    return dict(losses, value=t.V, log_prob=t.lp, prox_log_prob=lp_p, grad=grad,
                surr_sum=t.surr[ind].sum(), ent_sum=-ents[ind].sum(), value_loss_sum=t.vterm.sum(),
                clipped=int(t.clipped.sum()), kl_sum=kl_g.sum(), dual=int(t.dual[ind].sum()),
                linear=int(t.linear.sum()), prox_weight=t.w[ind].sum(), prox_kl=t.pkl[ind].sum(), n=ind.size,
                n_ind=int(ind.sum()))


def _action(g, actions, i):
    return int(actions[i, int(np.argmax(g.stage[:2]))])


def sgnn_minibatch(flat, states, actions, adv, ret, fixed, exps, *, clip_epsilon=0.2, value_pred_coef=0.5,
                   entropy_coef=0.01, old_values=None, value_clip=None, huber_delta=None, dual_clip=None, lp_old=None,
                   kl_coef=0.0, prox_flat=None):
    """One SGNN minibatch in float64 through oracle/sgnn_numpy: the losses (loss, value_loss, surr_loss, entropy_loss,
    kl_loss), per-graph value and log_prob, prox_log_prob (the log-probs at prox_flat, or None), the flat gradient and
    the statistics sums.  With every option off the losses and the gradient are ON.ppo_minibatch's bit for bit: the
    same operations in the same order.

    lp_old: per graph, its candidates' old log-probs in mask-index order; given, kl_sum is formed, and with kl_coef the
    penalty.  Its logit seed enters ON.backward as a second call whose g_z is exactly that seed (the backward is linear
    in g_z: with g_logp = -1, g_ent = 0 and no action, g_z is the cached p, replaced by the seed)."""
    P = ON._p64(flat)
    B = len(states)
    runs = []
    for i, st in enumerate(states):
        g = ON.unpad(st)
        runs.append((g, ON.forward(P, g, action=_action(g, actions, i), keep=True)))
    lp_p = None
    if prox_flat is not None:
        Pp = ON._p64(prox_flat)
        lp_p = np.array([ON.forward(Pp, g, action=_action(g, actions, i))["log_prob"] for i, (g, _) in enumerate(runs)])
    vals, lps, ents = (np.array([fw[k] for _, fw in runs]) for k in ("value", "log_prob", "entropy"))
    t = _terms(vals, lps, adv, ret, fixed, exps, lp_p, clip_epsilon=clip_epsilon, old_values=old_values,
               value_clip=value_clip, huber_delta=huber_delta, dual_clip=dual_clip)
    n_ind = max(int(t.ind.sum()), 1)
    G = {k: np.zeros_like(v) for k, v in P.items()}
    surr = vloss = eloss = 0.0
    kl_g = np.zeros(B)
    for i, (g, fw) in enumerate(runs):
        vloss += t.vterm[i] / B
        g_lp = g_en = 0.0
        if t.ind[i]:
            surr += t.surr[i] / n_ind
            eloss += -ents[i] / n_ind
            g_lp = t.g_r[i] * t.r[i] / n_ind
            g_en = -entropy_coef / n_ind
        Gi = ON.backward(P, g, fw, value_pred_coef * t.g_v[i] / B, g_lp, g_en)
        c = fw["cache"]
        if lp_old is not None and t.ind[i] and c.get("logp") is not None and c["logp"].size:
            kl_g[i], seed = kl64(lp_old[i], c["logp"])
            if kl_coef:
                G2 = ON.backward(P, g, dict(fw, cache=dict(c, p=kl_coef / n_ind * seed), action_pos=-1), 0.0, -1.0, 0.0)
                Gi = {k: Gi[k] + G2[k] for k in Gi}
        for k in G:
            G[k] += Gi[k]
    kl = kl_g.sum() / n_ind
    grad = np.zeros(PL.NUM_PARAMS)
    for s in PL.SLOTS.values():
        grad[s.offset:s.offset + s.size] = G[s.name].reshape(-1)
    return _result(t, ents, kl_g, lp_p, grad, loss=surr + value_pred_coef * vloss + entropy_coef * eloss + kl_coef * kl,
                   value_loss=vloss, surr_loss=surr, entropy_loss=eloss, kl_loss=kl)


def _mlp_log_probs(P, states, act, chunk):
    with torch.no_grad():
        return np.concatenate([MP.log_prob_entropy(P, MP.stack_states(states[a:a + chunk]), act[a:a + chunk])[0]
                               .reshape(-1).numpy() for a in range(0, len(states), chunk)])


def _mlp_kl(P, b, lp_old, ind):
    """Per graph of a sub-batch, its exact KL against lp_old through the port's masked logits; 0 for a graph outside
    ind or without candidates."""
    zl, zr = MP.masked_logits(P, b)
    out = []
    for j in range(len(ind)):
        lu = bool(b["stage"][j, 0] > 0)
        z = (zl if lu else zr)[j][(b["land_use_mask"] if lu else b["road_mask"])[j]]
        if not ind[j] or z.numel() == 0:
            out.append(torch.zeros((), dtype=torch.float64))
            continue
        lo = torch.tensor(np.asarray(lp_old[j], np.float64))
        po = lo.exp()
        out.append(torch.where(po > 0, po * (torch.where(po > 0, lo, 0.0) - torch.log_softmax(z, -1)), 0.0).sum())
    return torch.stack(out)


def mlp_minibatch(flat, states, actions, adv, ret, fixed, exps, *, clip_epsilon=0.2, value_pred_coef=0.5,
                  entropy_coef=0.01, old_values=None, value_clip=None, huber_delta=None, dual_clip=None, lp_old=None,
                  kl_coef=0.0, prox_flat=None, chunk=32):
    """sgnn_minibatch's arguments and keys for the rl-mlp, through oracle/mlp_port's autograd in float64 (the
    parameters taken from `flat` in float64, not rounded to fp32), in sub-batches of `chunk` graphs: the padded
    land-use features of 256 graphs take 400 MB in float64.  The flat gradient is stored in fp32 by PL.MLP.flatten, as
    the port's flat_grad stores it."""
    P = KO.mlp_params64(flat, requires_grad=True)
    n = len(states)
    act = torch.tensor(np.asarray(actions))
    ind = np.asarray(exps).reshape(-1) != 0
    n_ind = max(int(ind.sum()), 1)
    lp_p = None if prox_flat is None else _mlp_log_probs(KO.mlp_params64(prox_flat), states, act, chunk)
    A, anchor, _, _ = _anchor(adv, fixed, lp_p)
    R = _col(ret)
    V_old = None if old_values is None else _col(old_values)
    vals, lps, ents, kl_g = (np.zeros(n) for _ in range(4))
    for a in range(0, n, chunk):
        sl = slice(a, min(a + chunk, n))
        b = MP.stack_states(states[sl])
        v = MP.value(P, b).reshape(-1)
        lp, ent = (x.reshape(-1) for x in MP.log_prob_entropy(P, b, act[sl]))
        on = torch.tensor(ind[sl])
        r = torch.exp(lp - torch.tensor(anchor[sl]))
        surr = surrogate(r, torch.tensor(A[sl]), clip_epsilon, dual_clip, reduce=False)[on].sum()
        vl = value_terms(v, torch.tensor(R[sl]), huber_delta, None if V_old is None else torch.tensor(V_old[sl]),
                         value_clip).sum()
        loss = surr / n_ind + value_pred_coef * vl / n - entropy_coef * ent[on].sum() / n_ind
        if lp_old is not None:
            kl = _mlp_kl(P, b, lp_old[sl], ind[sl])
            kl_g[sl] = kl.detach().numpy()
            loss = loss + kl_coef * kl.sum() / n_ind
        loss.backward()
        vals[sl], lps[sl], ents[sl] = (x.detach().numpy() for x in (v, lp, ent))
    t = _terms(vals, lps, adv, ret, fixed, exps, lp_p, clip_epsilon=clip_epsilon, old_values=old_values,
               value_clip=value_clip, huber_delta=huber_delta, dual_clip=dual_clip)
    grad = PL.MLP.flatten({k: (x.grad.numpy() if x.grad is not None else np.zeros(tuple(x.shape)))
                           for k, x in P.items()})
    out = _result(t, ents, kl_g, lp_p, np.asarray(grad, np.float64))
    sl, vl, el, kl = out["surr_sum"] / n_ind, out["value_loss_sum"] / n, out["ent_sum"] / n_ind, out["kl_sum"] / n_ind
    out.update(loss=sl + value_pred_coef * vl + entropy_coef * el + kl_coef * kl, value_loss=vl, surr_loss=sl,
               entropy_loss=el, kl_loss=kl)
    return out


# ---- torch-port agents ------------------------------------------------------------------------------------------------
class _Options:
    """The loss and optimiser options of the port agents.  value_clip clips against `old_values`, set per step; kl_coef
    penalises the KL against the policy of `P_old`, set with snapshot(), and may change between steps (last_kl is the
    last step's mean KL); max_grad_norm clips all parameters with clip_grad_norm_ on every step in place of the
    reference's clip; weight_decay is torch.optim.Adam's (coupled L2)."""

    def __init__(self, flat, *, value_clip=None, huber_delta=None, dual_clip=None, kl_coef=None, max_grad_norm=None,
                 weight_decay=0.0, **kw):
        super().__init__(flat, **kw)
        self.value_clip, self.huber_delta, self.dual_clip = value_clip, huber_delta, dual_clip
        self.kl_coef, self.max_grad_norm = kl_coef, max_grad_norm
        self.old_values = self.P_old = self.last_kl = None
        for group in self.opt.param_groups:
            group["weight_decay"] = weight_decay

    def snapshot(self):
        self.P_old = {k: v.detach().clone() for k, v in self.P.items()}

    def _backward(self, kl_fn, b, v, lp, ent, adv, ret, fixed, ind):
        ratio = torch.exp(lp[ind] - fixed.to(lp.dtype)[ind])
        surr = surrogate(ratio, adv.to(lp.dtype)[ind], self.clip_epsilon, self.dual_clip)
        ov = None if self.old_values is None else self.old_values.to(v.dtype)
        vl = value_terms(v, ret.to(v.dtype), self.huber_delta, ov, self.value_clip).mean()
        el = -ent[ind].mean()
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el
        if self.kl_coef is not None:
            kl = kl_fn(self.P, self.P_old, b)[ind].mean()
            loss = loss + self.kl_coef * kl
            self.last_kl = kl.item()
        self.opt.zero_grad()
        loss.backward()
        return loss.item(), vl.item(), surr.item(), el.item()


class PortAgent(_Options, TP.PortAgent):
    """oracle/torch_port.PortAgent with the options."""

    def backward(self, b, actions, advantages, returns, fixed_log_probs, ind):
        v = TP.value(self.P, b)
        lp, ent = TP.log_prob_entropy(self.P, b, actions)
        return self._backward(KO.sgnn_kl, b, v, lp, ent, advantages, returns, fixed_log_probs, ind)

    def clip(self):
        if self.max_grad_norm is None:
            return super().clip()
        torch.nn.utils.clip_grad_norm_(list(self.P.values()), self.max_grad_norm)


class MLPPortAgent(_Options, MP.MLPPortAgent):
    """oracle/mlp_port.MLPPortAgent with the options."""

    def backward(self, b, actions, adv, ret, fixed, ind):
        v = MP.value(self.P, b)
        lp, ent = MP.log_prob_entropy(self.P, b, actions)
        return self._backward(KO.mlp_kl, b, v, lp, ent, adv, ret, fixed, ind)

    def step(self, *args):
        if self.max_grad_norm is None:
            return super().step(*args)
        out = self.backward(*args)
        torch.nn.utils.clip_grad_norm_(list(self.P.values()), self.max_grad_norm)
        self.opt.step()
        self.steps_done += 1
        return out
