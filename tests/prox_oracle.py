"""The fp32 replay of the EWMA proximal policy's parameter average (PPO-EWMA, upb_set_prox_ewma).  The minibatch with
the proximal policy is tests/ppo_oracle.py's."""
from __future__ import annotations

import numpy as np

from oracle import sgnn_numpy as ON


def sgnn_log_probs(flat, states, actions):
    """float64 log-probs of the SGNN at `flat` (oracle/sgnn_numpy.forward)."""
    n = len(states)
    r = ON.ppo_minibatch(flat, states, actions, np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n), want_grad=False)
    return r["log_prob"]


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
