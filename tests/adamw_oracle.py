"""torch 2.11's _single_tensor_adam with betas, eps, amsgrad and decoupled_weight_decay on flat arrays: a float64 oracle
and an fp32 replay in the step kernels' operation order (optim_kernels.cuh: pg_adam_step).

The replay forms what the kernels form: the moment weights 1.f - fp32(beta), the bias corrections in double from
fp32(beta) by repeated squaring (layout.h: ipow), the step size (float)(lr / bc1), the decoupled factor fp32(1 - lr * wd)
in double and the coupled term as one fused multiply-add."""
import math
from fractions import Fraction

import numpy as np

F32 = np.float32


def adam64(p, g, m, v, vmax, step, lr, wd, beta1, beta2, eps, amsgrad=False, decoupled=False):
    """One float64 Adam step at count `step` (the count after it); returns (p, m, v, vmax)."""
    p, g, m, v = (np.asarray(x, np.float64) for x in (p, g, m, v))
    vmax = np.asarray(vmax, np.float64)
    if wd != 0.0:
        if decoupled:
            p = p * (1.0 - lr * wd)
        else:
            g = g + wd * p
    m = m + (1.0 - beta1) * (g - m)
    v = v * beta2 + (1.0 - beta2) * g * g
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    d = v
    if amsgrad:
        vmax = np.maximum(vmax, v)
        d = vmax
    p = p - (lr / bc1) * (m / (np.sqrt(d) / math.sqrt(bc2) + eps))
    return p, m, v, vmax


def ipow(b: float, n: int) -> float:
    r = 1.0
    while n > 0:
        if n & 1:
            r *= b
        b *= b
        n >>= 1
    return r


def _round_f32(x: Fraction) -> F32:
    """x rounded once to fp32 (nearest, ties to even)."""
    d = float(x)                                   # nearest double
    r = F32(d)
    if float(r) != d:
        other = np.nextafter(r, F32(np.inf) if d > float(r) else F32(-np.inf))
        mid = (Fraction(float(r)) + Fraction(float(other))) / 2
        if Fraction(d) == mid and x != mid:        # d sits on a tie that x does not: round x itself
            return other if abs(x - Fraction(float(other))) < abs(x - Fraction(float(r))) else r
    return r


def fma32(a, b, c) -> np.ndarray:
    """Element-wise fp32 a * b + c with one rounding (the kernels' __fmaf_rn)."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, F32) for x in (a, b, c)))
    out = np.empty(a.shape, F32)
    for i in np.ndindex(a.shape):
        x, y, z = float(a[i]), float(b[i]), float(c[i])
        if not all(map(math.isfinite, (x, y, z))):
            out[i] = F32(F32(x) * F32(y) + F32(z))
        else:
            out[i] = _round_f32(Fraction(x) * Fraction(y) + Fraction(z))
    return out


def adam32(p, g, m, v, vmax, step, lr, wd, beta1, beta2, eps, amsgrad=False, decoupled=False):
    """The kernels' fp32 Adam step on a tensor at count `step` (after it); returns (p, m, v, vmax) as float32 copies.
    vmax is returned unchanged without amsgrad."""
    p, g, m, v, vmax = (np.array(x, F32) for x in (p, g, m, v, vmax))
    b1, b2, e = F32(beta1), F32(beta2), F32(eps)
    w1, w2 = F32(1.0) - b1, F32(1.0) - b2
    step_size = F32(lr / (1.0 - ipow(float(b1), step)))
    bc2_sqrt = F32(math.sqrt(1.0 - ipow(float(b2), step)))
    with np.errstate(all="ignore"):
        if wd != 0.0 and decoupled:
            p = p * F32(1.0 - lr * wd)
        elif wd != 0.0:
            g = fma32(F32(wd), p, g)
        m = m + w1 * (g - m)
        v = v * b2 + (w2 * g) * g
        d = v
        if amsgrad:
            vmax = np.where((v > vmax) | np.isnan(v), v, vmax).astype(F32)
            d = vmax
        denom = np.sqrt(d) / bc2_sqrt + e
        p = p + (-step_size) * (m / denom)
    return p, m, v, vmax
