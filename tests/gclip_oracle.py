"""The global gradient-norm clip (`max_grad_norm`, torch.nn.utils.clip_grad_norm_(actor_critic.parameters(), m)) for the
oracles, and a host replay of the order in which the step kernels form its norm (optim_kernels.cuh: gclip_*)."""
from __future__ import annotations

import numpy as np

from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.diagnostics import grad_clip_coef

SLICE = 128
SGNN_ROW, MLP_ROW = 14592, 10304          # per-CTA gradient rows (layout.h: G_ROW; mlp_kernel.cuh: MG_ROW)


def clip64(grad, max_norm):
    """clip_grad_norm_ in float64 on a flat gradient (every parameter once): g * min(m / (||g|| + 1e-6), 1)."""
    g = np.asarray(grad, np.float64)
    norm = np.sqrt(np.sum(g * g))
    return g * min(max_norm / (norm + 1e-6), 1.0), norm


def _sgnn_chain():
    """The attention chain's flat columns in its element order (optim_kernels.cuh: chain_dst) and the chain-owned mask."""
    s = PL.SGNN.slots
    dst = np.concatenate([s[n].offset + np.arange(256) for n in ("att_q_w", "att_k_w", "att_v_w")] +
                         [s["mha_in_w"].offset + np.arange(768)] +
                         [s[n].offset + np.arange(16) for n in ("att_q_b", "att_k_b", "att_v_b")] +
                         [s["mha_in_b"].offset + np.arange(48)])
    owned = np.zeros(PL.NUM_PARAMS, bool)
    owned[dst] = True
    return dst, owned


def _halve(x):
    while x.shape[-1] > 1:
        h = x.shape[-1] // 2
        x = x[..., :h] + x[..., h:]
    return x[..., 0]


def replay_norm(grad_buffer, model):
    """The fp32 norm the kernels form from a step's reduced gradient buffer, bit for bit: float64 squares of each
    128-column slice's real-parameter columns added by halving, the SGNN's chain partial (thread sums of 4 elements
    512 apart, a halving tree per warp, the 16 warps in order), all partials in slice order, sqrt in double."""
    g = np.asarray(grad_buffer, np.float32).astype(np.float64)
    mlp = model == "mlp"
    n, row = (PL.MLP.num_params, MLP_ROW) if mlp else (PL.NUM_PARAMS, SGNN_ROW)
    x = np.zeros(-(-row // SLICE) * SLICE)           # the rl-mlp row's last slice is half a slice
    x[:n] = g[:n] * g[:n]
    if not mlp:
        dst, owned = _sgnn_chain()
        x[:n][owned] = 0.0
    parts = list(_halve(x.reshape(-1, SLICE)))
    if not mlp:
        c = np.zeros(2048)
        c[:dst.size] = g[dst] * g[dst]
        c = c.reshape(4, 512)
        thread = ((c[0] + c[1]) + c[2]) + c[3]
        warps = _halve(thread.reshape(16, 32))
        chain = 0.0
        for w in warps:
            chain += w
        parts.append(chain)
    total = 0.0
    for p in parts:
        total += p
    return np.float32(np.sqrt(total))


def coef(norm, max_norm):
    return grad_clip_coef(norm, max_norm)
