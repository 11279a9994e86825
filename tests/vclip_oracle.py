"""Clipped value loss (OpenAI baselines' ppo2, CleanRL's clip_vloss) and per-minibatch advantage normalisation
(Stable-Baselines3's normalize_advantage) for the oracles, which themselves implement neither.

The clipped value loss of one graph, in torch's operations:
    d = V - V_old,  Vc = V_old + clamp(d, -c, c),  a = (V - R)^2,  b = (Vc - R)^2,  loss = max(a, b)
averaged over the minibatch's B graphs.  Its gradient is autograd's for torch.maximum (a tie sends half to each input)
and the inclusive clamp: 2 (V - R) where a > b, 2 (Vc - R) [-c <= d <= c] where b > a, the half-sum on a tie."""
from __future__ import annotations

import numpy as np
import torch

from drl_urban_planning_b200 import params as PL
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP


def seed64(V, R, V_old, c):
    """float64 per-graph (d loss / dV, loss, clipped) of the clipped value loss, arrays of the graphs."""
    V, R, V_old = (np.asarray(x, np.float64).reshape(-1) for x in (V, R, V_old))
    d = V - V_old
    Vc = V_old + np.clip(d, -c, c)
    a, b = (V - R) ** 2, (Vc - R) ** 2
    ga, gb = 2.0 * (V - R), np.where((d >= -c) & (d <= c), 2.0 * (Vc - R), 0.0)
    g = np.where(a > b, ga, np.where(b > a, gb, 0.5 * ga + 0.5 * gb))
    return g, np.maximum(a, b), (b > a).astype(np.float64)


def seed32(V, R, V_old, c, c_value=0.5, inv_batch=1.0):
    """The step kernels' fp32 seed g_V = (c_v * dloss/dV) * (1/B), loss and branch, with their rounding: what one graph
    contributes to the value-head bias gradient and to statistics slots 15 / 16."""
    f = np.float32
    V, R, V_old = (np.asarray(x, np.float32).reshape(-1) for x in (V, R, V_old))
    c = f(c)
    with np.errstate(over="ignore", invalid="ignore"):
        dv = f(V - R)
        d = f(V - V_old)
        Vc = f(V_old + np.minimum(np.maximum(d, -c), c))
        dvc = f(Vc - R)
        la, lb = f(dv * dv), f(dvc * dvc)
        ga, gb = f(f(2) * dv), np.where((d >= -c) & (d <= c), f(f(2) * dvc), f(0))
        g = np.where(la > lb, ga, np.where(lb > la, gb, f(f(f(0.5) * ga) + f(f(0.5) * gb))))
        gv = f(f(f(c_value) * g) * f(inv_batch))
    return gv, np.where(lb > la, lb, la), (lb > la).astype(np.float32)


def clipped_value_loss(v, ret, old_values, c):
    """The torch form: mean of torch.max(a, b), all tensors of one shape."""
    d = v - old_values
    vc = old_values + torch.clamp(d, -c, c)
    return torch.max((v - ret).pow(2), (vc - ret).pow(2)).mean()


def normalize64(adv, exps, order, B):
    """float64 normalisation of every minibatch order[i B, (i + 1) B), i < len(order) // B, rounded as the kernel does:
    mean and unbiased std to fp32 once each, then (A - mean) / (std + 1e-8) in fp32.  Other entries keep their values."""
    adv = np.asarray(adv, np.float32).reshape(-1)
    exps = np.asarray(exps).reshape(-1)
    out = adv.copy()
    for i in range(len(order) // B):
        idx = np.asarray(order[i * B:(i + 1) * B])
        sel = adv[idx[exps[idx] != 0]].astype(np.float64)
        if sel.size < 2:
            continue
        mean = np.float32(sel.mean())
        std = np.float32(np.sqrt(((sel - sel.mean()) ** 2).sum() / (sel.size - 1)))
        out[idx] = (adv[idx] - mean) / np.float32(std + np.float32(1e-8))
    return out


def normalize_torch(adv, exps, order, B):
    """The Stable-Baselines3 formula in torch fp32 on each minibatch's exps != 0 advantages, written to all its graphs."""
    adv = torch.as_tensor(np.asarray(adv, np.float32).reshape(-1))
    exps = torch.as_tensor(np.asarray(exps).reshape(-1))
    out = adv.clone()
    for i in range(len(order) // B):
        idx = torch.as_tensor(np.asarray(order[i * B:(i + 1) * B]), dtype=torch.long)
        sel = adv[idx][exps[idx] != 0]
        if sel.numel() < 2:
            continue
        out[idx] = (adv[idx] - sel.mean()) / (sel.std() + 1e-8)
    return out.numpy()


def ppo_minibatch(flat, states, actions, advantages, returns, fixed_log_probs, exps, old_values, value_clip,
                  clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01):
    """oracle/sgnn_numpy.ppo_minibatch with the clipped value loss: float64 losses, per-graph values and the flat
    gradient, plus the slot 15 / 16 sums (value_loss_sum, clipped)."""
    P = ON._p64(flat)
    B = len(states)
    adv, ret, flp = (np.asarray(x, np.float64).reshape(-1) for x in (advantages, returns, fixed_log_probs))
    ind = np.flatnonzero(np.asarray(exps).reshape(-1) != 0)
    n_ind = max(len(ind), 1)
    fws, vals = [], np.zeros(B)
    for i, st in enumerate(states):
        g = ON.unpad(st)
        sid = int(np.argmax(g.stage[:2]))
        fw = ON.forward(P, g, action=int(actions[i, sid]), keep=True)
        fws.append((g, fw))
        vals[i] = fw["value"]
    gv, vl_terms, clipped = seed64(vals, ret, old_values, value_clip)
    Gtot = {k: np.zeros_like(v) for k, v in P.items()}
    surr = eloss = 0.0
    for i, (g, fw) in enumerate(fws):
        g_lp = g_en = 0.0
        if i in ind:
            r = np.exp(fw["log_prob"] - flp[i])
            s1, s2 = r * adv[i], np.clip(r, 1 - clip_epsilon, 1 + clip_epsilon) * adv[i]
            surr += -min(s1, s2) / n_ind
            eloss += -fw["entropy"] / n_ind
            if (1 - clip_epsilon) <= r <= (1 + clip_epsilon) or s1 < s2:
                g_lp = -adv[i] * r / n_ind
            g_en = -entropy_coef / n_ind
        Gi = ON.backward(P, g, fw, value_pred_coef * gv[i] / B, g_lp, g_en)
        for k in Gtot:
            Gtot[k] += Gi[k]
    vloss = vl_terms.sum() / B
    grad = np.zeros(PL.NUM_PARAMS)
    for s in PL.SLOTS.values():
        grad[s.offset:s.offset + s.size] = Gtot[s.name].reshape(-1)
    return dict(loss=surr + value_pred_coef * vloss + entropy_coef * eloss, value_loss=vloss, surr_loss=surr,
                entropy_loss=eloss, value=vals, grad=grad, value_loss_sum=vl_terms.sum(), clipped=clipped.sum())


class PortAgent(TP.PortAgent):
    """oracle/torch_port.PortAgent whose value loss is clipped_value_loss against `old_values` (set per step)."""

    def __init__(self, flat, value_clip, **kw):
        super().__init__(flat, **kw)
        self.value_clip, self.old_values = value_clip, None

    def backward(self, b, actions, advantages, returns, fixed_log_probs, ind):
        surr, _, el = TP.ppo_losses(self.P, b, actions, advantages, returns, fixed_log_probs, ind, self.clip_epsilon)
        vl = clipped_value_loss(TP.value(self.P, b), returns, self.old_values, self.value_clip)
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el
        self.opt.zero_grad()
        loss.backward()
        return loss.item(), vl.item(), surr.item(), el.item()


class MLPPortAgent(MP.MLPPortAgent):
    """oracle/mlp_port.MLPPortAgent with the clipped value loss against `old_values` (set per step)."""

    def __init__(self, flat, value_clip, **kw):
        super().__init__(flat, **kw)
        self.value_clip, self.old_values = value_clip, None

    def backward(self, b, actions, adv, ret, fixed, ind):
        surr, _, el = MP.ppo_losses(self.P, b, actions, adv, ret, fixed, ind, self.clip_epsilon)
        v = MP.value(self.P, b)
        vl = clipped_value_loss(v, ret.to(v.dtype), self.old_values.to(v.dtype), self.value_clip)
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el
        self.opt.zero_grad()
        loss.backward()
        return loss.item(), vl.item(), surr.item(), el.item()
