"""PPO diagnostics per minibatch from the sums the step kernels leave in the gradient buffer.

The step kernels add, per graph, the terms of statistics slots 8-12 (include/upb200.h) next to the loss statistics, and
`upb_grad_norms` gives each gradient buffer's squared norms over the three clip groups.  Every input is a sum over
graphs or a function of the globally reduced gradient, so shards of a minibatch on several GPUs sum to the same
diagnostics as one GPU running the whole minibatch.
"""
from __future__ import annotations

import numpy as np

NAMES = ("approx_kl", "clip_fraction", "explained_variance", "grad_norm_policy", "grad_norm_value")


def grad_clip_coef(norm, max_norm):
    """torch.nn.utils.clip_grad_norm_'s coefficient clamp(max_norm / (norm + 1e-6), max=1) in fp32 as torch forms it
    (a Python float over a tensor is reciprocal(tensor) * float); a NaN norm gives NaN."""
    n = np.asarray(norm, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = (np.float32(1.0) / (n + np.float32(1e-6))) * np.float32(max_norm)
    return np.where(c > np.float32(1.0), np.float32(1.0), c)


def ppo_diagnostics(stats, sq_norms) -> dict:
    """Per-minibatch diagnostics, each a float64 array of shape (minibatches,).

    stats:    (minibatches, >= 13) summed statistics rows, slot layout of include/upb200.h.
    sq_norms: (minibatches, 3) sums of squares of the minibatch's gradient over the shared encoder, the policy heads and
              the value head (upb_grad_norms).

    approx_kl and clip_fraction are means over the graphs with exps != 0, divided by max(n_ind, 1) as the losses are.
    explained_variance = 1 - Var(V - R) / Var(R), both variances over the minibatch's B graphs, with V the value at the
    parameters the step started from; NaN when Var(R) is zero, that is, not above 1e-5 of mean(R^2), the cancellation
    error of a variance formed from fp32 sums of R and R^2.  grad_norm_policy = sqrt(encoder + policy) and
    grad_norm_value = sqrt(encoder + value) are the totals the reference's two clip_grad_norm_ calls measure
    (agent_ppo.py:43-46), before any clipping and without weight decay.  On a step that clips, the reference's second
    call sees the encoder already scaled by the first; the value reported here is the unscaled one.
    """
    st = np.asarray(stats, np.float64)
    sq = np.asarray(sq_norms, np.float64)
    st = st.reshape(-1, st.shape[-1])
    sq = sq.reshape(-1, 3)
    n_b = np.maximum(st[:, 3], 1.0)
    n_i = np.maximum(st[:, 4], 1.0)
    mean_r = st[:, 10] / n_b
    var_r = st[:, 11] / n_b - mean_r * mean_r
    mean_e = st[:, 12] / n_b
    var_e = st[:, 0] / n_b - mean_e * mean_e
    # Var(R) from the sums: a constant R leaves only the rounding of the sums, which is not a spread of the returns
    flat_r = var_r <= 1e-5 * (st[:, 11] / n_b)
    with np.errstate(divide="ignore", invalid="ignore"):
        ev = np.where(flat_r, np.nan, 1.0 - var_e / np.where(flat_r, 1.0, var_r))
    return dict(approx_kl=st[:, 8] / n_i, clip_fraction=st[:, 9] / n_i, explained_variance=ev,
                grad_norm_policy=np.sqrt(sq[:, 0] + sq[:, 1]), grad_norm_value=np.sqrt(sq[:, 0] + sq[:, 2]))
