// Flat parameter / gradient layout (ActorCritic.parameters() order, SURVEY.md appendix A.5).
// Mirrors drl_urban_planning_b200/params.py; tests/test_abi.py checks both against upb_param_slot().
#pragma once
#include "../../include/upb200.h"

namespace upb {

constexpr int D = 16;           // gcn_node_dim
constexpr int F = 23;           // node feature dim
constexpr int FS = 24;          // padded node feature stride
constexpr int NUMD = 52;        // numerical feature dim
constexpr int NH0 = 64;         // numeric encoder hidden
constexpr int HID = 32;         // policy / value head hidden
constexpr int SVD = 67;         // value-head input: 16 + 16 + 16 + 16 + 3

// ---- parameter offsets (floats)
constexpr int P_NUM_W0 = 0;         // [64][52]
constexpr int P_NUM_B0 = 3328;      // [64]
constexpr int P_NUM_W1 = 3392;      // [16][64]
constexpr int P_NUM_B1 = 4416;      // [16]
constexpr int P_ENC_W = 4432;       // [16][23]
constexpr int P_ENC_B = 4800;       // [16]
constexpr int P_GCN0_W = 4816;      // [16][32]
constexpr int P_GCN0_B = 5328;      // [16]
constexpr int P_GCN1_W = 5344;
constexpr int P_GCN1_B = 5856;
constexpr int P_MHA_IN_W = 5872;    // [48][16]
constexpr int P_MHA_IN_B = 6640;    // [48]
constexpr int P_MHA_OUT_W = 6688;   // [16][16]
constexpr int P_MHA_OUT_B = 6944;   // [16]
constexpr int P_ATT_Q_W = 6960;
constexpr int P_ATT_Q_B = 7216;
constexpr int P_ATT_K_W = 7232;
constexpr int P_ATT_K_B = 7488;
constexpr int P_ATT_V_W = 7504;
constexpr int P_ATT_V_B = 7760;
constexpr int P_LU_W0 = 7776;       // [32][64]
constexpr int P_LU_B0 = 9824;       // [32]
constexpr int P_LU_W1 = 9856;       // [1][32]
constexpr int P_RD_W0 = 9888;       // [32][16]
constexpr int P_RD_B0 = 10400;      // [32]
constexpr int P_RD_W1 = 10432;      // [1][32]
constexpr int P_VAL_W0 = 10464;     // [32][67]
constexpr int P_VAL_B0 = 12608;     // [32]
constexpr int P_VAL_W1 = 12640;     // [32][32]
constexpr int P_VAL_B1 = 13664;     // [32]
constexpr int P_VAL_W2 = 13696;     // [1][32]
constexpr int P_VAL_B2 = 13728;     // [1]
constexpr int NUM_PARAMS = 13729;

constexpr int ENCODER_END = P_LU_W0;   // [0, ENCODER_END) shared encoder
constexpr int POLICY_END = P_VAL_W0;   // [ENCODER_END, POLICY_END) policy heads; rest value head

// ---- per-CTA partial gradient row: real parameters, then "virtual" gradients of the composed attention
// projections (chained to the real tensors once per step by attention_chain, optim_kernels.cuh), then loss statistics.
constexpr int G_QC = 13744;            // [16][16]  d/d(Win_q Wq)
constexpr int G_QBC = G_QC + 256;      // [16]      d/d(Win_q bq + bin_q)
constexpr int G_KC = G_QBC + 16;       // [16][16]  d/d(Win_k Wk)
constexpr int G_VC = G_KC + 256;       // [16][16]  d/d(Win_v Wv)
constexpr int G_VBC = G_VC + 256;      // [16]      d/d(Win_v bv + bin_v)
constexpr int G_STATS = G_VBC + 16;    // 14544: [STATS_USED] statistics (see upb200.h)
constexpr int G_ROW = 14592;           // row stride (multiple of 64)

// statistics slots the step kernels fill (upb200.h); the reductions copy [0, STATS_USED) into the gradient buffer and
// write the rest of its UPB_STAT_COUNT slots as zeros.  Both models' per-CTA rows hold at least this many.
constexpr int STATS_USED = 13;
// The clipped value loss (upb_set_value_clip) adds two sums beyond the KL stop's slots 13 / 14: the value loss the step
// optimised and the number of graphs whose clipped branch won.  The reductions copy them like [0, STATS_USED).
constexpr int VCLIP_LOSS_SLOT = 15, VCLIP_COUNT_SLOT = 16;
// The KL penalty (upb_set_kl_penalty) adds the sum of the exact per-graph KL(pi_old || pi) after the global clip's norm
// (slot 17, not a sum).
constexpr int KLPEN_SLOT = 18;
// Dual-clip PPO (upb_set_dual_clip) counts the graphs whose bound c A was strictly active (slot 20); the Huber value
// loss (upb_set_huber_delta) counts the graphs whose chosen value term is in its linear branch (slot 21) and, like value
// clipping, sums the value loss the step optimised in slot 15.
constexpr int DUAL_COUNT_SLOT = 20, HUBER_COUNT_SLOT = 21;
// The KL-adaptive learning rate (upb_set_adaptive_lr) writes the step's decision, +1 / -1 / 0, into slot 22 once (not a
// sum: the reductions write it as 0 and the optimiser step overwrites it).
constexpr int LR_DECISION_SLOT = 22;
// The EWMA proximal policy (upb_set_prox_ewma) sums the behaviour weights w = exp(lp_p - lp_b) (slot 23) and the
// behaviour-to-proximal KL estimate expm1(d) - d, d = lp_p - lp_b (slot 24) over ind.
constexpr int PROX_WEIGHT_SLOT = 23, PROX_KL_SLOT = 24;
#ifdef __CUDACC__
__host__ __device__
#endif
constexpr bool stat_summed(int slot) {
  return slot < STATS_USED || slot == VCLIP_LOSS_SLOT || slot == VCLIP_COUNT_SLOT || slot == KLPEN_SLOT ||
         slot == DUAL_COUNT_SLOT || slot == HUBER_COUNT_SLOT || slot == PROX_WEIGHT_SLOT || slot == PROX_KL_SLOT;
}

// The fused step tails cut a gradient row into slices of SLICE columns, each owned by one CTA.
constexpr int SLICE = 128;

// Gradient-row layout of a model as the reductions and the fused step tail read it (SgnnRow here, MlpRow in
// mlp_kernel.cuh).  A per-CTA partial row of `row` floats holds the parameters' gradients [0, num_params) and the
// statistics from column `stats`; the flat gradient buffer holds [num_params gradients | pad | UPB_STAT_COUNT
// statistics at stat_offset].  The columns [chain0_begin, chain0_end) and [chain1_begin, chain1_end) are written by an
// attention chain rule instead of being copied from the column sums (empty ranges: none).  [lu_begin, rd_begin) and
// [rd_begin, policy_end) are the land-use and road heads, whose Adam step is skipped when no graph of their stage ran.
struct SgnnRow {
  static constexpr int row = G_ROW, nslice = G_ROW / SLICE, num_params = NUM_PARAMS, policy_end = POLICY_END;
  static constexpr int lu_begin = P_LU_W0, rd_begin = P_RD_W0, stats = G_STATS, stat_offset = UPB_STAT_OFFSET;
  static constexpr int chain0_begin = P_MHA_IN_W, chain0_end = P_MHA_OUT_W, chain1_begin = P_ATT_Q_W,
                       chain1_end = P_LU_W0;     // in_proj weight + bias; the q / k / v projections
};

// beta^n for an integer step count by repeated squaring in double (a handful of multiplies; libdevice pow(double) costs
// thousands of cycles in a one-thread critical path)
#ifdef __CUDACC__
__host__ __device__
#endif
inline double ipow(double b, long long n) {
  double r = 1.0;
  while (n > 0) {
    if (n & 1) r *= b;
    b *= b;
    n >>= 1;
  }
  return r;
}

}  // namespace upb
