"""Float64 oracle of the EWMA proximal policy (PPO-EWMA, upb_set_prox_ewma) for both models, and the fp32 replay of its
parameter average.

Per graph with exps != 0, lp its log-prob at the step's parameters, lp_b the behaviour (fixed) log-prob and lp_p its
log-prob at the proximal parameters:
    r = exp(lp - lp_p),  w = exp(lp_p - lp_b) (a constant),  surr = -w min(r A, clamp(r, lo, hi) A)
Since w > 0, w min(r A, clamp(r) A) = min(r A', clamp(r) A') with A' = w A (and likewise the dual clip's bound), so the
decoupled minibatch is the existing oracle run at the anchor lp_p with advantages A'.  The value loss and the entropy
do not see w."""
from __future__ import annotations

import numpy as np
import torch

import lossopt_oracle as LO
from drl_urban_planning_b200 import params as PL
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON


def weights64(lp_p, lp_b):
    """float64 per-graph behaviour weight w = exp(lp_p - lp_b) and the KL estimate expm1(d) - d (slots 23, 24)."""
    d = np.asarray(lp_p, np.float64).reshape(-1) - np.asarray(lp_b, np.float64).reshape(-1)
    return np.exp(d), np.expm1(d) - d


def sgnn_log_probs(flat, states, actions):
    """float64 log-probs of the SGNN at `flat` (oracle/sgnn_numpy.forward)."""
    n = len(states)
    r = ON.ppo_minibatch(flat, states, actions, np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n), want_grad=False)
    return r["log_prob"]


def sgnn_minibatch(flat, prox_flat, states, actions, advantages, returns, fixed_log_probs, exps, **kw):
    """The SGNN's decoupled minibatch: lossopt_oracle.ppo_minibatch (its dual_clip, huber_delta, old_values,
    value_clip, clip_epsilon and loss coefficients in kw) at the anchor lp_p with A' = w A, plus the slot sums
    prox_weight / prox_kl and lp_p itself."""
    lp_p = sgnn_log_probs(prox_flat, states, actions)
    w, kl = weights64(lp_p, fixed_log_probs)
    adv = np.asarray(advantages, np.float64).reshape(-1)
    out = LO.ppo_minibatch(flat, states, actions, w * adv, returns, lp_p, exps, **kw)
    ind = np.asarray(exps).reshape(-1) != 0
    out.update(prox_weight=w[ind].sum(), prox_kl=kl[ind].sum(), prox_log_prob=lp_p)
    return out


def mlp_minibatch(flat, prox_flat, states, actions, advantages, returns, fixed_log_probs, exps, clip_epsilon=0.2,
                  value_pred_coef=0.5, entropy_coef=0.01, dual_clip=None):
    """The rl-mlp's decoupled minibatch in float64 torch autograd (oracle/mlp_port), through the same identity:
    losses, the flat gradient and the slot sums."""
    b = MP.stack_states(states)
    act = torch.as_tensor(np.asarray(actions))
    ind = torch.as_tensor(np.flatnonzero(np.asarray(exps).reshape(-1) != 0))
    with torch.no_grad():
        lp_p = MP.log_prob_entropy(MP.params_from_flat(prox_flat, torch.float64), b, act)[0].reshape(-1)
    lp_b = torch.as_tensor(np.asarray(fixed_log_probs, np.float64).reshape(-1))
    w = torch.exp(lp_p - lp_b)
    P = MP.params_from_flat(flat, torch.float64, requires_grad=True)
    v = MP.value(P, b).reshape(-1)
    lp, ent = (x.reshape(-1) for x in MP.log_prob_entropy(P, b, act))
    ratio = torch.exp(lp[ind] - lp_p[ind])
    a = w[ind] * torch.as_tensor(np.asarray(advantages, np.float64).reshape(-1))[ind]
    surr = LO.surrogate(ratio, a, clip_epsilon, dual_clip)
    vl = (v - torch.as_tensor(np.asarray(returns, np.float64).reshape(-1))).pow(2).mean()
    el = -ent[ind].mean()
    loss = surr + value_pred_coef * vl + entropy_coef * el
    loss.backward()
    grad = PL.MLP.flatten({k: (x.grad.numpy() if x.grad is not None else np.zeros(tuple(x.shape)))
                           for k, x in P.items()})
    wk, kl = weights64(lp_p.numpy(), lp_b.numpy())
    m = np.asarray(exps).reshape(-1) != 0
    return dict(loss=loss.item(), value_loss=vl.item(), surr_loss=surr.item(), entropy_loss=el.item(), grad=grad,
                prox_weight=wk[m].sum(), prox_kl=kl[m].sum(), prox_log_prob=lp_p.numpy())


def fma32(b, x, y):
    """fp32 fmaf(b, x, y) with one rounding, for fp32 arrays b, x, y: b x is exact in float64, the sum is TwoSum's
    float64 value plus its error, and a float64 sum that lands exactly halfway between two fp32 neighbours is moved
    towards the error before the rounding to fp32."""
    p = np.float64(b) * np.asarray(x, np.float32).astype(np.float64)
    q = np.asarray(y, np.float32).astype(np.float64)
    s = p + q
    bb = s - p
    e = (p - (s - bb)) + (q - bb)
    r = s.astype(np.float32).astype(np.float64)
    up = np.nextafter(r.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(r.astype(np.float32), np.float32(-np.inf)).astype(np.float64)
    tie = ((s - r) == (up - r) / 2) | ((r - s) == (r - dn) / 2)
    s = np.where(tie & (e != 0), np.nextafter(s, s + e), s)
    return s.astype(np.float32)


def ewma_replay(prox, trajectory, beta):
    """theta_prox after the parameter vectors `trajectory` (each the parameters an applied step left), in the kernels'
    fp32 arithmetic: fmaf(fp32(beta), fp32(prox - theta), theta)."""
    b = np.float32(beta)
    p = np.asarray(prox, np.float32).copy()
    for theta in trajectory:
        th = np.asarray(theta, np.float32)
        p = fma32(b, (p - th).astype(np.float32), th)
    return p
