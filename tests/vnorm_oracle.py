"""Value-target normalisation (MAPPO's ValueNorm with per_element_update=False) and PopArt's output-preserving rescale
of the value head's last layer, in float64, for the tests; the oracles themselves know neither.

The state is {m1, m2, d}; its statistics S are (0, 1) while d == 0, else mean = m1 / max(d, 1e-5) and
std = sqrt(max(m2 / max(d, 1e-5) - mean^2, 1e-2)).  Every operation here is one IEEE double operation in the order the
kernels use (include/upb200.h: upb_set_value_norm), so given the same state the fp32 outputs below are the kernels'
bits; the state update itself sums the returns in another order, which moves it by round-off only."""
from __future__ import annotations

import math

import numpy as np


def stats(m1, m2, d):
    """S(m1, m2, d) -> (mean, std) in float64."""
    if d == 0.0:
        return 0.0, 1.0
    dd = max(float(d), 1e-5)
    mu = float(m1) / dd
    return mu, math.sqrt(max(float(m2) / dd - mu * mu, 1e-2))


def update(state, returns, beta):
    """The state after one update from `returns` (all of them); the unchanged state when one is not finite."""
    r = np.asarray(returns, np.float32).astype(np.float64).reshape(-1)
    if not np.isfinite(r).all():
        return tuple(float(x) for x in state)
    m1, m2, d = (float(x) for x in state)
    b1, b2 = math.fsum(r) / r.size, math.fsum(r * r) / r.size
    w = 1.0 - beta
    return beta * m1 + w * b1, beta * m2 + w * b2, beta * d + w


def rescale(w2, b2, old, new, dtype=np.float32):
    """PopArt: the last layer (w2 (32,), b2 scalar) that maps the new statistics' normalised output onto the same
    denormalised value, formed in float64 from the `dtype` values and rounded once to `dtype`."""
    (mo, so), (mn, sn) = old, new
    w = np.asarray(w2, dtype).astype(np.float64)
    b = float(dtype(b2))
    return (w * so / sn).astype(dtype), dtype(((so * b + mo) - mn) / sn)


def normalize(x, st):
    """(x - fp32(mean)) / fp32(std) in fp32."""
    mu, sd = np.float32(st[0]), np.float32(st[1])
    with np.errstate(invalid="ignore", over="ignore"):
        return (np.asarray(x, np.float32) - mu) / sd


def fmaf(a, x, b):
    """fp32 fma(a, x, b), correctly rounded: a * x is exact in float64; the float64 sum's rounding error is recovered
    (TwoSum) to settle a sum that lands exactly half-way between two fp32 values."""
    a, x, b = (np.asarray(v, np.float32).astype(np.float64) for v in (a, x, b))
    p = a * x
    s = p + b
    bv = s - p
    err = (p - (s - bv)) + (b - bv)
    f = s.astype(np.float32)
    f64 = f.astype(np.float64)
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    tie_up, tie_dn = s == (f64 + up) / 2, s == (f64 + dn) / 2
    f = np.where(tie_up & (err > 0), up.astype(np.float32), f)
    f = np.where(tie_dn & (err < 0), dn.astype(np.float32), f)
    return f


def denormalize(n, state):
    """The value in reward units of the head's normalised outputs n: fmaf(fp32(std), n, fp32(mean)), n itself while
    d == 0."""
    n = np.asarray(n, np.float32)
    if state[2] == 0.0:
        return n.copy()
    mu, sd = stats(*state)
    return fmaf(np.float32(sd), n, np.float32(mu))


def step(state, returns, values, w2, b2, beta, new_state=None):
    """One upb_value_norm_update: the new state, the rescaled (w2, b2) and the normalised returns / values.  With
    `new_state` (the kernel's), the fp32 outputs are formed from it, so they are the kernel's bits."""
    new = update(state, returns, beta) if new_state is None else tuple(new_state)
    moved = bool(np.isfinite(np.asarray(returns, np.float32)).all())
    old_st, new_st = stats(*state), stats(*new)
    if moved:
        w2, b2 = rescale(w2, b2, old_st, new_st)
    return dict(state=new, stats=new_st, w2=np.asarray(w2, np.float32), b2=np.float32(b2),
                returns=normalize(returns, new_st), values=None if values is None else normalize(values, new_st))
