"""The bf16-tile build (libupb200_bf16.so, -DUPB_TILE_BF16) for the oracles: float64 with the kernel's rounding at the
three products it runs as tensor-core tiles.

That build replaces the 3xTF32 tiles of the SGNN backward (csrc/sgnn_kernel.cuh, mma_3x) by one TF32 pass on operands
rounded to bfloat16 with round-to-nearest-even from their fp32 values.  A bf16 x bf16 product is exact in TF32 and in
float64, so the oracle rounds the operands exactly as the kernel does and multiplies and accumulates in float64:
  * g_W = GPQ^T h^l   (gw_partial): A = GPQ, the unscaled (gP | gQ) rows of the pull; B = the layer input h^l;
  * g_h = g_h' + GPQ Wpq   (gh_phase_tc): A = GPQ, B = the layer's weights; the g_h' term is the accumulator's initial
    value and is not rounded;
  * g_We = g_h0^T X   (encoder backward): A = g_h0, B = the node features; the g_hc x_cur^T term is added outside the
    tile and is not rounded.
Everything else -- the g_hc outer product, enc_b, the gcn*_b sums, EPQ, h^0 -- stays exact, as it does in the kernel.
An operand is rounded from the fp32 value the kernel holds (float64 -> fp32 -> bf16), so an operand the fp32 kernel
carries exactly rounds the same way here."""
from __future__ import annotations

import numpy as np

from oracle import sgnn_numpy as ON

# the tensors the tiles reach: every other gradient tensor is formed before the first tile of the backward (gcn1_b is
# the bias sum of the last layer's pull, which comes before that layer's g_h and g_W tiles)
TILE_TENSORS = ("gcn0_w", "gcn0_b", "gcn1_w", "enc_w", "enc_b")


def bf16_round(x) -> np.ndarray:
    """fp32 -> bf16 with round-to-nearest-even, as torch's .to(torch.bfloat16) and the kernel's bf16_round: float32
    values whose low 16 bits are clear.  A NaN becomes the quiet NaN 0x7fc0 (c10::BFloat16's; torch's vectorised CPU
    conversion gives 0xffff, another NaN); +-inf stays; finite values past the largest bf16 round to +-inf."""
    x = np.asarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7fff + ((u >> 16) & 1)) & 0xffff0000).astype(np.uint32)
    r = np.where(np.isnan(x), np.uint32(0x7fc00000), r)
    return r.view(np.float32)


def bf16_operand(a) -> np.ndarray:
    """A tile operand as the kernel feeds it: the float64 value at fp32, rounded to bf16, back in float64."""
    return bf16_round(np.asarray(a, np.float64).astype(np.float32)).astype(np.float64)


def bf16_tile(a, b) -> np.ndarray:
    """A @ B with both operands rounded as the bf16-tile build rounds them, accumulated in float64."""
    return bf16_operand(a) @ bf16_operand(b)


def ppo_minibatch(*args, **kw):
    """oracle/sgnn_numpy.ppo_minibatch with the bf16 tiles."""
    return ON.ppo_minibatch(*args, tile=bf16_tile, **kw)
