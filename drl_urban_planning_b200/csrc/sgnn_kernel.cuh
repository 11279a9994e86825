// Fused SGNN policy/value forward(+backward) kernel: one CTA walks one rollout graph at a time and keeps
// the whole graph on chip (node embeddings, exp-transformed edge-MLP pre-activations, CSR adjacency).
//
// Reference dataflow replaced (all fp32):
//   urban_planning/models/state_encoder.py:184-214  encoder (node Linear, 2x {gather -> edge MLP -> scatter},
//                                                    masked means, 1-query attention, numeric MLP)
//   urban_planning/models/policy.py:45-104           masked categorical heads (log-prob, entropy, argmax)
//   urban_planning/models/value.py:36-39             value head
//   khrylib/rl/agents/agent_pg.py:19-23 + urban_planning/agents/urban_planning_agent.py:363-371   losses
//   autograd of all of the above (urban_planning_agent.py:335), hand-derived (SURVEY.md appendix A.7)
//
// Algebra used (exact in real arithmetic, SURVEY.md A.3):
//   * W_l [h_u | h_v] = P_u + Q_v with node-level P = h W_l[:, :16]^T + b, Q = h W_l[:, 16:]^T;
//   * tanh(P_u + Q_v) = 1 - 2 / (exp(2 P_u) exp(2 Q_v) + 1): exp(2P), exp(2Q) are taken once per NODE, an edge
//     costs one FMA + one MUFU.RCP per channel and direction;  he = (t1 + t2)/2 = 1 - r1 - r2;
//   * he is symmetric in (u, v), so the scatter-add becomes an atomics-free PULL over a symmetrised CSR;
//   * attention with one query: softmax_i(q'.k'_i/4) only needs (Kc^T q').h_i, and sum_i a_i v'_i = Vc hbar + vbc;
//   * land-use head first layer on [he | hc | he*hc | he-hc] = Weff he + ceff with a per-graph 32x16 Weff;
//   * only mask-true candidates need the head: masked logits are exactly 0-probability.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "blob.h"
#include "layout.h"
#include "optim_kernels.cuh"

namespace upb {

constexpr int NT = 512;          // threads per CTA (1024 would cap the per-graph body at 64 registers: spills)
constexpr int NW = NT / 32;      // warps per CTA
constexpr int NS = 464;          // nodes kept in shared memory
constexpr int AS = 5632;         // directed adjacency entries kept in shared memory
constexpr int KS = 160;          // action candidates kept in shared memory
constexpr int CH = 96;           // candidate chunk of the head backward
constexpr float MASK_FILL = -4294967296.0f;   // float32(-2**32 + 1), policy.py:50
constexpr float EPS_DEG = 1e-6f;               // state_encoder.py:11

// ---- shared memory map (floats) -----------------------------------------------------------------------
// weights (per CTA, loaded once per launch)
constexpr int S_WET = 0;                   // [24][16]  enc_w^T (row 23 zero)
constexpr int S_BE = S_WET + 384;          // [16]
constexpr int S_WPQ0 = S_BE + 16;          // [32][16]  rows 0-15: gcn_w[o][0:16] (P), rows 16-31: gcn_w[o-16][16:32] (Q)
constexpr int S_B0 = S_WPQ0 + 512;         // [16]
constexpr int S_WPQ1 = S_B0 + 16;
constexpr int S_B1 = S_WPQ1 + 512;
constexpr int S_QC = S_B1 + 16;            // [16][16]  Win_q Wq
constexpr int S_QBC = S_QC + 256;          // [16]      Win_q bq + bin_q
constexpr int S_KC = S_QBC + 16;           // [16][16]  Win_k Wk
constexpr int S_VC = S_KC + 256;           // [16][16]  Win_v Wv
constexpr int S_VBC = S_VC + 256;          // [16]
constexpr int S_WO = S_VBC + 16;           // [16][16]
constexpr int S_BO = S_WO + 256;           // [16]
constexpr int S_LUW0 = S_BO + 16;          // [32][64]
constexpr int S_LUB0 = S_LUW0 + 2048;      // [32]
constexpr int S_LUW1 = S_LUB0 + 32;        // [32]
constexpr int S_RDW0 = S_LUW1 + 32;        // [32][16]
constexpr int S_RDW0T = S_RDW0 + 512;      // [16][32]
constexpr int S_RDB0 = S_RDW0T + 512;      // [32]
constexpr int S_RDW1 = S_RDB0 + 32;        // [32]
constexpr int S_WPQT0 = S_RDW1 + 32;       // [16][32]  transpose of S_WPQ0 (bank-conflict-free EPQ phase)
constexpr int S_WPQT1 = S_WPQT0 + 512;
constexpr int S_QCT = S_WPQT1 + 512;       // [16][16] transposes of Qc, Kc, Vc, Wo (conflict-free lane-per-row matvecs)
constexpr int S_KCT = S_QCT + 256;
constexpr int S_VCT = S_KCT + 256;
constexpr int S_WOT = S_VCT + 256;
constexpr int S_WEND = S_WOT + 256;

// per-graph small vectors
constexpr int V_X52 = 0;        // [52] numerical features (padded to 56)
constexpr int V_XCUR = 56;      // [24]
constexpr int V_HC = 80;        // [16]
constexpr int V_A0 = 96;        // [64] numeric hidden
constexpr int V_SV = 160;       // [67] value features: hnum | mean_h | mean_he | att | stage (padded to 68)
constexpr int V_QP = 228;       // [16] q'
constexpr int V_QK = 244;       // [16] Kc^T q' / 4
constexpr int V_HBAR = 260;     // [16]
constexpr int V_VP = 276;       // [16] v' = Vc hbar + vbc
constexpr int V_Y0 = 292;       // [32]
constexpr int V_Y1 = 324;       // [32]
constexpr int V_WEFFT = 356;    // [16][32] Weff^T (land use)
constexpr int V_CEFF = 868;     // [32]
constexpr int V_GSV = 900;      // [68]
constexpr int V_D0 = 968;       // [32]
constexpr int V_D1 = 1000;      // [32]
constexpr int V_DN0 = 1032;     // [64]
constexpr int V_DN1 = 1096;     // [16]
constexpr int V_GVP = 1112;     // [16]
constexpr int V_GHBAR = 1128;   // [16]
constexpr int V_GSH = 1144;     // [16]
constexpr int V_GQP = 1160;     // [16]
constexpr int V_GHC = 1176;     // [16]
constexpr int V_CE = 1192;      // [16] g_mean_he / e
constexpr int V_GMN = 1208;     // [16] g_mean_h / n
constexpr int V_GWEFF = 1224;   // [32][16]
constexpr int V_GC = 1736;      // [32]
constexpr int V_GW2 = 1768;     // [32]
constexpr int V_TMP16 = 1800;   // [16] block-reduce results
constexpr int V_TMP16B = 1816;  // [16]
constexpr int V_SC = 1832;      // [24] scalars
constexpr int V_WEFF = 1856;    // [32][16] Weff (land use), row-major copy for the head backward
constexpr int V_TMP32 = 2368;   // [32] block-reduce results
constexpr int V_END = 2400;
// scalar slots
constexpr int SC_VALUE = 0, SC_MAX = 1, SC_SUM = 2, SC_LSE = 3, SC_ENT = 4, SC_LOGP = 5, SC_GV = 6, SC_GLP = 7,
              SC_GH = 8, SC_Z = 9, SC_SLOT = 10, SC_BEST = 11, SC_GDOT = 12, SC_ACT = 13, SC_RET = 14, SC_EXP = 15,
              SC_FLP = 16, SC_ADV = 17, SC_QUEUE = 18, SC_VOLD = 19, SC_PLP = 20;

constexpr int S_VEC = S_WEND;
constexpr int S_RED = S_VEC + V_END;             // [NW][20] block-reduce scratch
constexpr int S_INV = S_RED + NW * 20;           // [NS]
constexpr int S_ALPHA = S_INV + NS;              // [NS]
constexpr int S_RP = S_ALPHA + NS;               // [(NS+8)/2] u16 pairs: CSR row pointers (live to the end: g_h reads degrees)
// from here to S_EPQ everything is dead after the last pull; the encoder backward's node features land here early
constexpr int S_Z = S_RP + (NS + 8) / 2;         // [KS]
constexpr int S_GZ = S_Z + KS;                   // [KS]
constexpr int S_GHEAD = S_GZ + KS;               // [KS][16]
constexpr int S_CUV = S_GHEAD + KS * 16;         // [KS] u32
constexpr int S_CIDX = S_CUV + KS;               // [KS] i32
constexpr int ORD_ROUNDS = ((NS + 7) / 8 + NW - 1) / NW + 1;   // pull-schedule rounds kept in shared memory
constexpr int S_ORD = S_CIDX + KS;               // [ORD_ROUNDS][NW][8] u16: pull schedule (blob.h)
constexpr int S_ADJ = S_ORD + ORD_ROUNDS * NW * 4;   // [AS] u32
constexpr int S_EPQ = S_ADJ + AS;                // [NS][32]
constexpr int S_GPQ = S_EPQ + NS * 32;           // [NS][32]   (aliased by the head-backward chunk buffers)
constexpr int S_H = S_GPQ + NS * 32;             // [NS][16]
constexpr int S_TOTAL = S_H + NS * 16;
constexpr size_t SMEM_BYTES = (size_t)S_TOTAL * 4;
static_assert(SMEM_BYTES <= 232448, "shared memory budget (227 KB)");
constexpr int KW = 16;            // warps that share the K dimension of the g_W tile reduction
constexpr int XEARLY_NODES = (S_EPQ - S_Z) / FS;        // feature rows that fit in the candidate + CSR + adjacency stretch
static_assert(S_Z % 4 == 0 && S_EPQ % 4 == 0, "bulk copies need 16-byte aligned shared addresses");
constexpr int HIN_NODES = (NS * 32 - KW * 512) / 16;   // h rows that fit behind the g_W reduction buffer in the EPQ region
static_assert(KW * 512 <= NS * 32 && NW * 384 <= NS * 32, "cross-warp reduction buffers alias the EPQ region");
static_assert(NS == 464 && AS == 5632 && KS == 160 && CH == 96 && XEARLY_NODES == 381 && HIN_NODES == 416,
              "tests/shape_cases.py (used by tests/test_gpu_shapes.py) puts graphs on both sides of these limits: "
              "move its cases with them");
static_assert(NW == kPullWarps, "the packer lays the pull schedule out for NT / 32 warps");
static_assert(NT >= 512 && KW <= NW, "thread (r, c) = (tid >> 4, tid & 15) mappings use the first 512 threads");
// The bulk copies of a fast-path graph round every blob section up to 16 bytes (graph_body staging).  At the largest
// fast-path sizes (n = NS, 2e = AS, k = KS, ord_rounds = ORD_ROUNDS) each rounded copy still ends inside its region:
static_assert((NS + 1 + 7) / 8 * 16 <= (NS + 8) / 2 * 4, "row-pointer copy at n = NS overruns S_RP");
static_assert((AS + 3) / 4 * 16 <= AS * 4, "adjacency copy at 2e = AS (e odd or even) overruns S_ADJ");
static_assert((KS + 3) / 4 * 16 <= KS * 4, "candidate copies at k = KS overrun S_CUV / S_CIDX");
static_assert(ORD_ROUNDS * NW * 16 <= (S_ADJ - S_ORD) * 4, "pull-schedule copy overruns S_ORD");
static_assert(NS * FS <= S_GPQ - S_EPQ && NS * 32 <= S_GPQ - S_EPQ, "feature / EPQ copies at n = NS overrun S_EPQ");
static_assert(S_Z + XEARLY_NODES * FS <= S_EPQ, "early feature copy at n = XEARLY_NODES overruns the list stretch");
static_assert(KW * 512 + HIN_NODES * 16 <= NS * 32, "h-row copy at n = HIN_NODES overruns the EPQ region");
// GPQ region while it is not holding GPQ (whole forward; backward until the first pull): value-head and numeric-
// encoder weights (re-staged per graph, padded row strides = conflict-free lane-per-row access), then the policy-head
// backward buffers.
constexpr int VN_VW0 = 0;                  // [32][67]   val_w0 (stride 67 is odd: conflict-free both ways)
constexpr int VN_VB0 = VN_VW0 + 2144;      // [32]
constexpr int VN_VW1 = VN_VB0 + 32;        // [32][33]   val_w1, row stride 33
constexpr int VN_VB1 = VN_VW1 + 1056;      // [32]
constexpr int VN_VW2 = VN_VB1 + 32;        // [32]
constexpr int VN_VB2 = VN_VW2 + 32;        // [1] (+3 pad)
constexpr int VN_NW0 = VN_VB2 + 4;         // [64][53]   num_w0, row stride 53
constexpr int VN_NB0 = VN_NW0 + 3392;      // [64]
constexpr int VN_NW1 = VN_NB0 + 64;        // [16][65]   num_w1, row stride 65
constexpr int VN_NB1 = VN_NW1 + 1040;      // [16]
constexpr int VN_END = VN_NB1 + 16;
constexpr int HB_GU = (VN_END + 3) & ~3;   // [CH][32] g_u of the chunk's candidates
constexpr int HB_X = HB_GU + CH * 32;      // [CH][16] head inputs
constexpr int HB_PGC = HB_X + CH * 16;     // [32 half-warps][32] partial sums of g_u
constexpr int HB_PGW2 = HB_PGC + 1024;     // [32 half-warps][32] partial sums of g_z t
constexpr int HB_END = HB_PGW2 + 1024;
static_assert(HB_END <= NS * 32, "value/numeric weights + head-backward buffers alias the GPQ region");

// per-CTA global scratch (floats): saved layer inputs + big-graph arrays
__host__ __device__ inline size_t scratch_floats(int n_cap, int e_cap) {
  const size_t kcap = (size_t)(e_cap > n_cap ? e_cap : n_cap);
  return (size_t)n_cap * (16 + 16 + 32 + 32 + 32 + 16 + 2) + kcap * 18 + 64;
}

struct StepArgs {
  const uint8_t* blob;
  const int* ids;
  int count;
  const float* params;
  const float* actions;
  const float* adv;
  const float* ret;
  const float* fixed_lp;
  const float* exps;
  float inv_batch, inv_ind;
  float clip_lo, clip_hi;      // the clip range [fp32(1 - eps), fp32(1 + eps)], each bound rounded once (upb_set_clip_range)
  float c_value, c_entropy;
  int diagnostics;             // 1: add the PPO diagnostic sums, statistics slots 8-12 (upb_set_diagnostics)
  float* out_value;
  float* out_logp;
  float* out_entropy;
  int* out_greedy;
  const float* uniforms;   // optional [blob count]: one uniform in [0, 1) per graph -> out_sample (forward kernel only)
  int* out_sample;         // action index drawn by inverse CDF over the candidates in index order
  float* gpart;        // [gridDim.x][G_ROW]
  float* scratch;      // [gridDim.x][scratch_stride]
  size_t scratch_stride;
  int n_cap, e_cap;
  // fused tail (single GPU, no clipping this step): cross-CTA gradient reduction + attention chain + Adam inside
  // the same launch, separated by grid barriers (cooperative launch: all CTAs are co-resident)
  int fuse_tail;
  float* params_rw;            // == params, writable
  float* grad_out;             // [UPB_GRAD_STRIDE]
  float* adam_m;
  float* adam_v;
  const long long* steps_in;   // [4]
  long long* steps_out;        // [4]
  unsigned int* gridbar;       // [8]: [0] cumulative arrival counter (never reset), [2], [3] stage bits by launch
                               // parity, [6] sticky count of CTAs that gave up on a peer
  unsigned int bar_target;     // value of gridbar[0] once every CTA of this launch has arrived
  float beta1, beta2, adam_eps;  // the learning rate is `lr`, last in the struct
  float weight_decay;          // Adam's coupled L2 term (upb_set_weight_decay); 0 = off
  // exchange buffers of the fused tail (one GPU: world = 1, own buffer only; upb_peer_connect: all ranks', mapped over
  // NVLink).  Layout per rank (floats): [2 parities][MAX_PEERS sources][G_ROW] sums, then u32 flags
  // [2][MAX_PEERS][FLAG_STRIDE] = (sequence << 2) | stage bits of the source rank.
  int world, rank;
  unsigned int seq;            // sequence number of this fused step (same on all ranks, starts at 1)
  float* const* peers;         // device array [world] of the ranks' exchange buffers (own buffer at [rank])
  long long* stamps;   // optional [384]: [0,64) clock64() phase stamps, [64,224) busy cycles per CTA, [224,384) prologue cycles; of the first graph of CTA 0 (tools/phase_times.py)
  // masked logit rows (policy.py:45-65, forward kernel only; upb_policy_logits): logit_rows[gid] = the graph's row in its
  // stage's matrix, < 0 = none; lu_logits [*][e_cap], rd_logits [*][n_cap], either may be NULL.  Last in the struct,
  // so the fields above keep their parameter offsets.
  const int* logit_rows;
  float* lu_logits;
  float* rd_logits;
  // KL stop of the training kernels (upb_set_target_kl; NULL = off): the model's stop word.  While it is set a step
  // returns at entry (skip_step); the fused tail sets it when the step's reduced statistics pass kl_exceeds(kl_limit).
  unsigned int* kl_stop;
  float kl_limit;
  // clipped value loss of the training kernels (upb_set_value_clip; NULL = off): the values V_old the update's pre-pass
  // computed, indexed by blob position, and the clip range c > 0 (value_seed)
  const float* old_values;
  float value_clip;
  // global gradient-norm clip of the fused tails (upb_set_max_grad_norm; 0 = off): tail_gclip
  float max_norm;
  // forward kernel only (upb_forward_cand; NULL = off): every candidate's log-softmax z_j - lse, at the graph's
  // candidate position cand_off + j of the blob
  float* out_cand_logp;
  // KL penalty of the training kernels (upb_set_kl_penalty; NULL = off): the pre-pass candidate log-probs, laid out as
  // out_cand_logp, and the coefficient beta > 0 (softmax_seeds)
  const float* old_cand_logp;
  float kl_coef;
  // non-finite guard of the fused tails (upb_set_nonfinite_guard; 0 = off): read by tail_gclip only
  int nonfinite_guard;
  // Adam's learning rate of the fused tails (upb_set_lr): a double, as torch keeps it, so that the step size is formed as
  // (float)(lr / bias_correction1)
  double lr;
  // parameter groups of the fused tails (upb_set_param_groups; NULL = none): read by k_sgnn_pg / k_mlp_pg, whose tail
  // is tail_gclip<L, true>, and by skip_step; each tensor's count goes tsteps_in -> tsteps_out
  const ParamGroups* pg;
  const long long* tsteps_in;
  long long* tsteps_out;
  // dual-clip PPO of the training kernels (upb_set_dual_clip; 0 = off): the bound c > 1 on a negative advantage's
  // surrogate (softmax_seeds).  Huber value loss (upb_set_huber_delta; 0 = off): the threshold delta > 0 (value_seed)
  float dual_clip;
  float huber_delta;
  // KL-adaptive lr of the fused tails (upb_set_adaptive_lr; alr.in NULL = off): the gate (tail_kl_gate) decides and
  // re-forms the staged step sizes from alr.in, and the statistics slice's owner writes alr.out (tail_write_lr).  The
  // host then passes a stop word even while the KL stop is off (a word nothing sets, with kl_limit = +inf), so the step
  // kernels fill slot 8 and the tails run the gate exactly as they do for the KL stop.
  AdaptiveLr alr;
  // EWMA proximal policy (upb_set_prox_ewma; NULL = off).  Training kernels: prox_lp = the log-probs at theta_prox by
  // position in ids (softmax_seeds), and the fused tails' EWMA of every element into prox_params with weight prox_beta
  // (adam_elem, prox_keep).  Forward kernel: out_pos_logp receives each graph's log-prob by position in ids, and the
  // launch returns at entry while kl_stop is set (the proximal forward of a skipped step).
  const float* prox_lp;
  float* out_pos_logp;
  float* prox_params;
  float prox_beta;
};

// ---- small device helpers ------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exp(2a) with 2a clamped to +-80 so products of two factors stay finite and non-zero.  The clamp changes the product
// of two clamped factors (e^{2P} e^{2Q} with P = 50, Q = -45 gives e^0, not e^10): graphs whose factors pass |a| = 40
// keep the raw pre-activations instead (tier 2 of the EPQ phase) and take exp2a of the sum.
__device__ __forceinline__ float exp2a(float a) {
  const float t = fminf(fmaxf(a * 2.8853900817779268f, -115.41560327111707f), 115.41560327111707f);
  return ex2_approx(t);
}
// 16-byte asynchronous global -> shared copies (LDGSTS): no register staging, every copy of a phase is in flight at once
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// ---- bulk asynchronous copies (TMA, 1-D): one elected thread issues cp.async.bulk global -> shared for a whole blob
// section; completion is counted in bytes on an mbarrier that every thread then waits on (UBLKCP / SYNCS in SASS).
// Sources and destinations are 16-byte aligned and sizes multiples of 16 (blob sections are padded for this).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy accesses (ordinary loads / stores) before this fence are ordered before later async-proxy (bulk copy)
// accesses to the same memory
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 f4(float a) { return make_float4(a, a, a, a); }
__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 operator*(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 operator*(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float comp(const float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }

// fp32 pairs: channels (x,y) and (z,w) of a float4.  sm_90 has no paired fp32 instruction, so each pair operation is
// two round-to-nearest scalar ones (the _rn forms are never contracted or reassociated by the compiler).
struct F2x2 { float2 a, b; };
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ F2x2 ldp(const float* p) {
  const float4 v = ld4(p);
  F2x2 r; r.a = make_float2(v.x, v.y); r.b = make_float2(v.z, v.w);
  return r;
}
// Row access of the pulls.  SM (the graph lives in shared memory): a per-thread 32-bit shared base address and ONE
// shift-add per neighbour row (ld.shared.v4 through inline PTX; left to itself the compiler rebuilds float indices with
// three more integer instructions per load).  Otherwise (large graphs, rows in global memory): ordinary loads.
template <bool SM>
struct RowBase {
  const float* p;
  unsigned a;
  __device__ __forceinline__ explicit RowBase(const float* base) : p(base), a(SM ? smem_u32(base) : 0u) {}
  __device__ __forceinline__ F2x2 row(unsigned k, int shift) const {      // 16 bytes at base + (k << shift) BYTES
    if constexpr (SM) {
      float4 v;
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a + (k << shift)));
      F2x2 r; r.a = make_float2(v.x, v.y); r.b = make_float2(v.z, v.w);
      return r;
    } else {
      return ldp(reinterpret_cast<const float*>(reinterpret_cast<const char*>(p) + ((size_t)k << shift)));
    }
  }
};
__device__ __forceinline__ float2 rcp2(float2 v) { return make_float2(rcp_approx(v.x), rcp_approx(v.y)); }
__device__ __forceinline__ float2 neg2(float2 v) { return make_float2(-v.x, -v.y); }

// Denominator 1 + e^{2(P_i + Q_k)} of one directed entry.  Tiers 0 and 1: EPQ rows hold the factors e^{2P}, e^{2Q};
// tier 2: the raw P, Q (the factors would have been clamped), summed before the exponential.
template <int TIER>
__device__ __forceinline__ float2 edge_den(float2 p, float2 q) {
  if constexpr (TIER == 2) {
    const float2 x = fadd2(p, q);
    return make_float2(__fadd_rn(exp2a(x.x), 1.f), __fadd_rn(exp2a(x.y), 1.f));
  } else {
    return ffma2(p, q, make_float2(1.f, 1.f));
  }
}
// Forward message of one directed entry, two channels: accumulates r1 + r2 into s, where
//   r1 = 1/(EP_i EQ_k + 1), r2 = 1/(EP_k EQ_i + 1),  he = 1 - r1 - r2.
// Fast form (tier 0): r1 + r2 = (a + b) / (a b) -> ONE reciprocal per channel; valid while a b cannot overflow, which
// the EPQ phase guarantees by flagging graphs with |pre-activation| > 10.9 (tiers 1 and 2 use two reciprocals).
template <int TIER>
__device__ __forceinline__ void fwd_term(float2 epi, float2 eqi, float2 epk, float2 eqk, float2& s) {
  const float2 a = edge_den<TIER>(epi, eqk), b = edge_den<TIER>(epk, eqi);
  if (TIER > 0) s = fadd2(s, fadd2(rcp2(a), rcp2(b)));
  else s = ffma2(fadd2(a, b), rcp2(fmul2(a, b)), s);
}
// Backward of the same entry: aP += ge2 r1 (1 - r1), aQ += ge2 r2 (1 - r2) with ge2 = 2 g_he
// (1 - tanh^2 = 4 r (1 - r) and g1 = g_he/2 (1 - t1^2)).
template <int TIER>
__device__ __forceinline__ void bwd_term(float2 epi, float2 eqi, float2 epk, float2 eqk, float2 ge2, float2& aP,
                                         float2& aQ) {
  const float2 one = make_float2(1.f, 1.f);
  const float2 a = edge_den<TIER>(epi, eqk), b = edge_den<TIER>(epk, eqi);
  float2 r1, r2;
  if (TIER > 0) { r1 = rcp2(a); r2 = rcp2(b); }
  else { const float2 R = rcp2(fmul2(a, b)); r1 = fmul2(b, R); r2 = fmul2(a, R); }
  aP = ffma2(ge2, fmul2(r1, fadd2(one, neg2(r1))), aP);
  aQ = ffma2(ge2, fmul2(r2, fadd2(one, neg2(r2))), aQ);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Deterministic block reductions.  `red` is NW*20 floats of scratch; results land in out[] (shared).
// All threads must call; two __syncthreads inside.
__device__ __forceinline__ float block_sum1(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < NW; ++w) s += red[w];
  __syncthreads();
  return s;
}
__device__ __forceinline__ float block_max1(float v, float* red) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = red[0];
#pragma unroll
  for (int w = 1; w < NW; ++w) s = fmaxf(s, red[w]);
  __syncthreads();
  return s;
}
// thread holds 4 channels (4q..4q+3, q = tid & 3) of a 16-vector partial sum -> out16[16]
__device__ __forceinline__ void block_sum_q4(float4 v, float* red, float* out16) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o);
    v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < 4) st4(red + warp * 16 + lane * 4, v);
  __syncthreads();
  if (threadIdx.x < 16) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) s += red[w * 16 + threadIdx.x];
    out16[threadIdx.x] = s;
  }
  __syncthreads();
}

// two float4 partials per thread (channels 4q..4q+3 of two 16-vectors) -> out32[0..15], out32[16..31]
__device__ __forceinline__ void block_sum_q8(float4 v, float4 w, float* red, float* out32) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o); v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o); v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
    w.x += __shfl_xor_sync(0xffffffffu, w.x, o); w.y += __shfl_xor_sync(0xffffffffu, w.y, o);
    w.z += __shfl_xor_sync(0xffffffffu, w.z, o); w.w += __shfl_xor_sync(0xffffffffu, w.w, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < 4) { st4(red + warp * 20 + lane * 4, v); }
  __syncthreads();
  float keep = 0.f;
  if (threadIdx.x < 16) {
#pragma unroll
    for (int x = 0; x < NW; ++x) keep += red[x * 20 + threadIdx.x];
  }
  __syncthreads();
  if (lane < 4) { st4(red + warp * 20 + lane * 4, w); }
  if (threadIdx.x < 16) out32[threadIdx.x] = keep;
  __syncthreads();
  if (threadIdx.x < 16) {
    float s = 0.f;
#pragma unroll
    for (int x = 0; x < NW; ++x) s += red[x * 20 + threadIdx.x];
    out32[16 + threadIdx.x] = s;
  }
  __syncthreads();
}
// a float4 partial (channels 4q..) plus one scalar per thread -> out32[0..15], out32[16]
__device__ __forceinline__ void block_sum_q4p1(float4 v, float sc1, float* red, float* out32) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o); v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o); v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
  }
  sc1 = warp_sum(sc1);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < 4) st4(red + warp * 20 + lane * 4, v);
  if (lane == 0) red[warp * 20 + 16] = sc1;
  __syncthreads();
  if (threadIdx.x < 17) {
    float s = 0.f;
#pragma unroll
    for (int x = 0; x < NW; ++x) s += red[x * 20 + threadIdx.x];
    out32[threadIdx.x] = s;
  }
  __syncthreads();
}

// y[row] = act(b[row] + W[row][:] . x) for row < rows; 8 lanes per row; rows must be a multiple of 4.
// W, b in global memory (read through L1/L2), x and y in shared memory.  No barrier inside.
template <bool TANH>
__device__ __forceinline__ void matvec8(const float* __restrict__ W, const float* __restrict__ b, int rows, int cols,
                                        const float* x, float* y) {
  const int p = threadIdx.x & 7;
  for (int row = threadIdx.x >> 3; row < rows; row += NT / 8) {
    const float* w = W + (size_t)row * cols;
    float acc = 0.f;
#pragma unroll 9
    for (int k = p; k < cols; k += 8) acc = fmaf(__ldg(w + k), x[k], acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (p == 0) {
      acc += __ldg(b + row);
      y[row] = TANH ? tanhf(acc) : acc;
    }
  }
}

// ---- once per launch: parameters -> shared memory (with the composed attention projections) --------------
__device__ __forceinline__ void load_weights(const float* __restrict__ P, float* sW) {
  // Every global load is issued before the first shared store (one L2/HBM round trip per launch, not one per loop).
  const int t = threadIdx.x;
  static_assert(NT == 512, "load_weights is laid out for 512 threads");
  const int o = t >> 4, c = t & 15;
  const int src = o < 16 ? o * 32 + c : (o - 16) * 32 + 16 + c;          // (P | Q) split of a gcn weight row
  const float wet = (t < 384 && (t >> 4) < F) ? __ldg(P + P_ENC_W + c * F + (t >> 4)) : 0.f;
  const float g0 = __ldg(P + P_GCN0_W + src), g1 = __ldg(P + P_GCN1_W + src);
  const float in0 = __ldg(P + P_MHA_IN_W + t), in1 = t < 256 ? __ldg(P + P_MHA_IN_W + 512 + t) : 0.f;
  float wq = 0.f, wk = 0.f, wv = 0.f, wo = 0.f;
  if (t < 256) {
    wq = __ldg(P + P_ATT_Q_W + t); wk = __ldg(P + P_ATT_K_W + t); wv = __ldg(P + P_ATT_V_W + t);
    wo = __ldg(P + P_MHA_OUT_W + t);
  }
  float lu[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) lu[j] = __ldg(P + P_LU_W0 + t + NT * j);
  const float rd = __ldg(P + P_RD_W0 + t);
  float sm0 = 0.f, sm1 = 0.f, sm2 = 0.f;     // small vectors, one element per thread group
  if (t < 16) { sm0 = __ldg(P + P_ENC_B + t); sm1 = __ldg(P + P_GCN0_B + t); sm2 = __ldg(P + P_GCN1_B + t); }
  else if (t < 32) { sm0 = __ldg(P + P_MHA_OUT_B + t - 16); sm1 = __ldg(P + P_ATT_Q_B + t - 16); sm2 = __ldg(P + P_ATT_V_B + t - 16); }
  else if (t < 64) { sm0 = __ldg(P + P_LU_B0 + t - 32); sm1 = __ldg(P + P_LU_W1 + t - 32); }
  else if (t < 96) { sm0 = __ldg(P + P_RD_B0 + t - 64); sm1 = __ldg(P + P_RD_W1 + t - 64); }
  else if (t < 112) { sm0 = __ldg(P + P_MHA_IN_B + t - 96); sm1 = __ldg(P + P_MHA_IN_B + 32 + t - 96); }

  float* tmp = sW + S_EPQ;                   // staging (the EPQ region is idle at launch time):
                                             // in_proj_weight [48][16] | Wq | Wk | Wv | bq | bv | bin_q | bin_v
  if (t < 384) sW[S_WET + t] = wet;
  sW[S_WPQ0 + t] = g0; sW[S_WPQ1 + t] = g1;
  sW[S_WPQT0 + c * 32 + o] = g0; sW[S_WPQT1 + c * 32 + o] = g1;
  tmp[t] = in0;
  if (t < 256) {
    tmp[512 + t] = in1;
    tmp[768 + t] = wq; tmp[1024 + t] = wk; tmp[1280 + t] = wv;
    sW[S_WO + t] = wo;
    sW[S_WOT + c * 16 + o] = wo;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) sW[S_LUW0 + t + NT * j] = lu[j];
  sW[S_RDW0 + t] = rd;
  sW[S_RDW0T + c * 32 + o] = rd;
  if (t < 16) { sW[S_BE + t] = sm0; sW[S_B0 + t] = sm1; sW[S_B1 + t] = sm2; }
  else if (t < 32) { sW[S_BO + t - 16] = sm0; tmp[1536 + t - 16] = sm1; tmp[1552 + t - 16] = sm2; }
  else if (t < 64) { sW[S_LUB0 + t - 32] = sm0; sW[S_LUW1 + t - 32] = sm1; }
  else if (t < 96) { sW[S_RDB0 + t - 64] = sm0; sW[S_RDW1 + t - 64] = sm1; }
  else if (t < 112) { tmp[1568 + t - 96] = sm0; tmp[1584 + t - 96] = sm1; }
  __syncthreads();
  // composed attention projections: Qc = Win_q Wq, Kc = Win_k Wk, Vc = Win_v Wv (+ transposes), qbc, vbc
  if (t < 256) {
    float q = 0.f, k = 0.f, v = 0.f;
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      q = fmaf(tmp[o * 16 + m], tmp[768 + m * 16 + c], q);
      k = fmaf(tmp[(16 + o) * 16 + m], tmp[1024 + m * 16 + c], k);
      v = fmaf(tmp[(32 + o) * 16 + m], tmp[1280 + m * 16 + c], v);
    }
    sW[S_QC + t] = q; sW[S_KC + t] = k; sW[S_VC + t] = v;
    const int tr = c * 16 + o;
    sW[S_QCT + tr] = q; sW[S_KCT + tr] = k; sW[S_VCT + tr] = v;
  } else if (t < 272) {
    const int r = t - 256;
    float q = tmp[1568 + r], v = tmp[1584 + r];
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      q = fmaf(tmp[r * 16 + m], tmp[1536 + m], q);
      v = fmaf(tmp[(32 + r) * 16 + m], tmp[1552 + m], v);
    }
    sW[S_QBC + r] = q;
    sW[S_VBC + r] = v;
  }
}

// ---- per-graph view ---------------------------------------------------------------------------------------
struct GraphView {
  int n, e, k, stage, gid;
  const float* x;          // [n][24] global
  float* H0g;              // [n][16] global scratch: h^0
  float* H1g;              // [n][16] global scratch: h^1
  float* EPQ;              // [n][32]
  float* GPQ;              // [n][32]
  float* H;                // [n][16]
  float* inv;              // [n]
  float* alpha;            // [n]
  float* z;                // [k]
  float* gz;               // [k]
  float* ghead;            // [k][16]
  const uint16_t* rp;      // [n+1]
  const uint16_t* ord;     // [ord_rounds][16][8] pull schedule: node ids, 0xFFFF = none (blob.h)
  int ord_rounds;
  const uint32_t* adj;     // [2e]
  const uint32_t* cuv;     // [k]
  const int* cidx;         // [k]
};

// ---- tensor-core tiles for the dense per-node blocks (mma.sync m16n8k8 TF32, "3xTF32" error compensation) -------
// fp32 parity (1e-4) rules out a single TF32 pass; splitting both operands into a TF32 head and a TF32 tail and
// accumulating a_lo b_hi + a_hi b_lo + a_hi b_hi in fp32 gives ~2^-21 relative error per product.
// The tail x - head is exact in fp32 and goes to the tensor core as it is: the TF32 multiplier reads only its upper 19
// bits, so a second cvt (several instructions on sm_90) would only round where the hardware truncates.
#ifdef UPB_TILE_BF16
// NON-PARITY build (BASELINE.json configs[2] "fp32 vs bf16 MLP tiles", libupb200_bf16.so): the tensor-core tiles take
// their operands rounded to bfloat16 (8-bit mantissa) and run ONE pass instead of the three of the 3xTF32 scheme.  A
// bf16 value is exactly representable in TF32, so the m16n8k8 TF32 instruction computes the bf16 x bf16 -> fp32 product
// exactly; results no longer meet the 1e-4 parity bar and bench.py labels the line accordingly.
// fp32 -> bf16 with round-to-nearest-even, as torch's .to(torch.bfloat16): a NaN stays a NaN, the quiet NaN 0x7fc0 of
// c10::BFloat16 (the rounding add would carry a NaN's mantissa into its exponent and sign: 0x7fffffff -> -0.0), +-inf
// stays, and finite values past the largest bf16 round to +-inf.  Returned as the fp32 bit pattern, low 16 bits clear.
__device__ __forceinline__ uint32_t bf16_round(float x) {
  if (x != x) return 0x7fc00000u;
  uint32_t u = __float_as_uint(x);
  u += 0x7fffu + ((u >> 16) & 1u);
  return u & 0xffff0000u;
}
// the B fragments reach mma_3x as their fp32 value (the tail is unused), so that mma_3x rounds them to bf16 once, as it
// does A: a TF32 head rounded again to bf16 would differ from one rounding by a bf16 ulp on ~6 % of values
__device__ __forceinline__ void tf32_split(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x);
  lo = 0u;
}
#else
__device__ __forceinline__ void tf32_split(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  lo = __float_as_uint(x - __uint_as_float(hi));
}
#endif
__device__ __forceinline__ void mma_tf32(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// one k-tile (8 columns) of a 16-row A tile held as four floats (rows g, g+8; tile columns t, t+4) times a B fragment
// given as hi/lo pairs
#ifdef UPB_TILE_BF16
// bf16 build: one pass on both operands rounded to bf16 from fp32 (bh0, bh1: fp32 bit patterns from tf32_split)
__device__ __forceinline__ void mma_3x(float (&c)[4], float a0, float a1, float a2, float a3, uint32_t bh0, uint32_t bh1,
                                       uint32_t bl0, uint32_t bl1) {
  (void)bl0; (void)bl1;
  mma_tf32(c, bf16_round(a0), bf16_round(a1), bf16_round(a2), bf16_round(a3),
           bf16_round(__uint_as_float(bh0)), bf16_round(__uint_as_float(bh1)));
}
#else
__device__ __forceinline__ void mma_3x(float (&c)[4], float a0, float a1, float a2, float a3, uint32_t bh0, uint32_t bh1,
                                       uint32_t bl0, uint32_t bl1) {
  uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
  tf32_split(a0, h0, l0); tf32_split(a1, h1, l1); tf32_split(a2, h2, l2); tf32_split(a3, h3, l3);
  mma_tf32(c, l0, l1, l2, l3, bh0, bh1);
  mma_tf32(c, h0, h1, h2, h3, bl0, bl1);
  mma_tf32(c, h0, h1, h2, h3, bh0, bh1);
}
#endif

// g_h = g_h' + GPQ . Wpq on the tensor cores, in place over H (which holds gs = g_h' / (deg + eps)); 16 nodes per
// warp-task, K = 32 permuted as above (two 128-bit row segments per row).  Wpq is [32 o][16 c].  If `rescale`, the
// result is stored scaled by 1 / (deg + eps) again (the next pull wants that form).
__device__ __forceinline__ void gh_phase_tc(const GraphView& g, const float* Wpq, bool rescale) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gq = lane >> 2, t = lane & 3;
  uint32_t bh[2][8], bl[2][8];         // [n-tile][k index: j<4 -> 4t+j, j>=4 -> 16+4t+(j-4)]
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = (j < 4 ? 0 : 16) + 4 * t + (j & 3);
      tf32_split(Wpq[k * 16 + nt * 8 + gq], bh[nt][j], bl[nt][j]);
    }
  const int n = g.n;
  for (int m0 = warp * 16; m0 < n; m0 += NW * 16) {
    const int r0 = min(m0 + gq, n - 1), r1 = min(m0 + gq + 8, n - 1);
    const float4 v0 = ld4(g.GPQ + r0 * 32 + 4 * t), v1 = ld4(g.GPQ + r0 * 32 + 16 + 4 * t);
    const float4 w0 = ld4(g.GPQ + r1 * 32 + 4 * t), w1 = ld4(g.GPQ + r1 * 32 + 16 + 4 * t);
    const float rd0 = (float)(g.rp[r0 + 1] - g.rp[r0]) + EPS_DEG, rd1 = (float)(g.rp[r1 + 1] - g.rp[r1]) + EPS_DEG;
    float acc[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const float2 h0 = *reinterpret_cast<const float2*>(g.H + r0 * 16 + nt * 8 + 2 * t);
      const float2 h1 = *reinterpret_cast<const float2*>(g.H + r1 * 16 + nt * 8 + 2 * t);
      acc[nt][0] = h0.x * rd0; acc[nt][1] = h0.y * rd0; acc[nt][2] = h1.x * rd1; acc[nt][3] = h1.y * rd1;
      mma_3x(acc[nt], v0.x, w0.x, v0.y, w0.y, bh[nt][0], bh[nt][1], bl[nt][0], bl[nt][1]);
      mma_3x(acc[nt], v0.z, w0.z, v0.w, w0.w, bh[nt][2], bh[nt][3], bl[nt][2], bl[nt][3]);
      mma_3x(acc[nt], v1.x, w1.x, v1.y, w1.y, bh[nt][4], bh[nt][5], bl[nt][4], bl[nt][5]);
      mma_3x(acc[nt], v1.z, w1.z, v1.w, w1.w, bh[nt][6], bh[nt][7], bl[nt][6], bl[nt][7]);
    }
    const float s0 = rescale ? g.inv[r0] : 1.f, s1 = rescale ? g.inv[r1] : 1.f;
    __syncwarp();                                   // every lane has read its H inputs before any lane overwrites
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      if (m0 + gq < n)
        *reinterpret_cast<float2*>(g.H + (m0 + gq) * 16 + nt * 8 + 2 * t) = make_float2(acc[nt][0] * s0, acc[nt][1] * s0);
      if (m0 + gq + 8 < n)
        *reinterpret_cast<float2*>(g.H + (m0 + gq + 8) * 16 + nt * 8 + 2 * t) = make_float2(acc[nt][2] * s1, acc[nt][3] * s1);
    }
  }
}

// exp-transformed edge-MLP pre-activations of one layer: EPQ[i][o] = exp(2 (Wpq[o] . h_i + b[o]))  (b only for o<16).
// 8 lanes per node PAIR, 4 outputs per lane.  Each lane keeps its 16x4 slice of the transposed weights WT[c][o] in
// registers for the whole phase (64 floats), so a pair costs only the 8 row loads of the two h vectors.
// RAW: store the pre-activations themselves (tier 2).  Returns this thread's tier of the largest |pre-activation| it
// saw: 0 up to 10.9 (the one-reciprocal pull), 1 up to exp2a's clamp at 40, 2 beyond it (or NaN).
template <bool RAW>
__device__ __forceinline__ int epq_phase(const GraphView& g, const float* hsrc, const float* WT, const float* b) {
  const int og = threadIdx.x & 7;
  const float4 bias = og < 4 ? ld4(b + og * 4) : f4(0.f);
  float2 wlo[16], whi[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const float4 w = ld4(WT + c * 32 + og * 4);
    wlo[c] = make_float2(w.x, w.y); whi[c] = make_float2(w.z, w.w);
  }
  const int npair = (g.n + 1) >> 1;
  float amax = 0.f;
  for (int task = threadIdx.x; task < npair * 8; task += NT) {
    const int i0 = (task >> 3) * 2;
    const int i1 = min(i0 + 1, g.n - 1);
    float4 ha[4], hb[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { ha[j] = ld4(hsrc + i0 * 16 + j * 4); hb[j] = ld4(hsrc + i1 * 16 + j * 4); }
    float2 a0 = make_float2(bias.x, bias.y), a1 = make_float2(bias.z, bias.w), b0 = a0, b1 = a1;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float xa = comp(ha[c >> 2], c & 3), xb = comp(hb[c >> 2], c & 3);
      const float2 xa2 = make_float2(xa, xa), xb2 = make_float2(xb, xb);
      a0 = ffma2(wlo[c], xa2, a0); a1 = ffma2(whi[c], xa2, a1);
      b0 = ffma2(wlo[c], xb2, b0); b1 = ffma2(whi[c], xb2, b1);
    }
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(a0.x), fabsf(a0.y)), fmaxf(fabsf(a1.x), fabsf(a1.y))));
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(b0.x), fabsf(b0.y)), fmaxf(fabsf(b1.x), fabsf(b1.y))));
    if constexpr (RAW) {
      st4(g.EPQ + i0 * 32 + og * 4, make_float4(a0.x, a0.y, a1.x, a1.y));
      if (i1 != i0) st4(g.EPQ + i1 * 32 + og * 4, make_float4(b0.x, b0.y, b1.x, b1.y));
    } else {
      st4(g.EPQ + i0 * 32 + og * 4, make_float4(exp2a(a0.x), exp2a(a0.y), exp2a(a1.x), exp2a(a1.y)));
      if (i1 != i0) st4(g.EPQ + i1 * 32 + og * 4, make_float4(exp2a(b0.x), exp2a(b0.y), exp2a(b1.x), exp2a(b1.y)));
    }
  }
  return !(amax <= 10.9f) + !(amax <= 40.f);      // NaN: 2
}

// Bank-conflict-free row access for the pulls.  An EPQ row is 32 floats: EP in banks 0-15, EQ in banks 16-31.  A
// 128-bit shared load is served per quarter-warp (8 lanes = two 4-lane node groups); if both groups read the EP half
// of their neighbour rows they collide.  So the odd group of every pair reads the halves in the opposite order:
//   X = row[offX..], Y = row[offY..] with (offX, offY) = odd ? (16, 0) : (0, 16), and the node's own factors are
//   swapped to match, m1 = A X + 1, m2 = B Y + 1 with (A, B) = odd ? (EP_i, EQ_i) : (EQ_i, EP_i).
// {m1, m2} = {a, b} = {EP_i EQ_k + 1, EP_k EQ_i + 1}: the forward is symmetric in them; the backward un-swaps its
// two accumulators once per node.

// one GCN layer forward, in place: H[i] += (sum over the CSR row of he(i,k)) / (deg_i + eps).  4 lanes per node.
template <int TIER, bool SM>
__device__ __forceinline__ void pull_forward(const GraphView& g, int q, bool save_h1, float* h1g, bool want_sums,
                                             float4& msum, float4& hsum) {
  const int odd = (threadIdx.x >> 2) & 1;
  const int offX = (odd ? 16 : 0) + q * 4, offY = (odd ? 0 : 16) + q * 4;
  const RowBase<SM> rX(g.EPQ + offX), rY(g.EPQ + offY);      // EPQ rows are 128 bytes
  for (int task = threadIdx.x; task < g.ord_rounds * NT; task += NT) {
    const int i = g.ord[task >> 2];
    if (i == kNoNode) continue;
    const F2x2 A = rY.row((unsigned)i, 7), B = rX.row((unsigned)i, 7);
    const int beg = g.rp[i], end = g.rp[i + 1];
    float2 s0 = make_float2(0.f, 0.f), s1 = s0, s2 = s0, s3 = s0;
    int t = beg;
    for (; t + 1 < end; t += 2) {       // two neighbours per trip: four independent dependency chains
      const unsigned k0 = g.adj[t] & 0xffffu, k1 = g.adj[t + 1] & 0xffffu;
      const F2x2 X0 = rX.row(k0, 7), Y0 = rY.row(k0, 7);
      const F2x2 X1 = rX.row(k1, 7), Y1 = rY.row(k1, 7);
      fwd_term<TIER>(A.a, B.a, Y0.a, X0.a, s0);
      fwd_term<TIER>(A.b, B.b, Y0.b, X0.b, s1);
      fwd_term<TIER>(A.a, B.a, Y1.a, X1.a, s2);
      fwd_term<TIER>(A.b, B.b, Y1.b, X1.b, s3);
    }
    if (t < end) {
      const unsigned k0 = g.adj[t] & 0xffffu;
      const F2x2 X0 = rX.row(k0, 7), Y0 = rY.row(k0, 7);
      fwd_term<TIER>(A.a, B.a, Y0.a, X0.a, s0);
      fwd_term<TIER>(A.b, B.b, Y0.b, X0.b, s1);
    }
    const float cnt = (float)(end - beg);
    const float4 acc = make_float4(cnt - (s0.x + s2.x), cnt - (s0.y + s2.y), cnt - (s1.x + s3.x), cnt - (s1.y + s3.y));
    const float iv = g.inv[i];
    float4 h = ld4(g.H + i * 16 + q * 4);
    h.x = fmaf(acc.x, iv, h.x); h.y = fmaf(acc.y, iv, h.y); h.z = fmaf(acc.z, iv, h.z); h.w = fmaf(acc.w, iv, h.w);
    st4(g.H + i * 16 + q * 4, h);
    if (save_h1) st4(h1g + i * 16 + q * 4, h);
    if (want_sums) { msum = msum + acc; hsum = hsum + h; }
  }
}

// one GCN layer backward (pull).  H holds the SCALED incoming gradient gs_i = g_h'_i / (deg_i + eps); writes
// GPQ[i] = (gP_i | gQ_i) using EPQ and, on the last layer, the mean / head gradients of the edge activations.
// Returns this thread's share of sum_i gP_i (bias gradient).
template <int TIER, bool SM>
__device__ __forceinline__ float4 pull_backward(const GraphView& g, int q, float4 ce4, bool use_head) {
  float4 bsum = f4(0.f);
  const float2 two = make_float2(2.f, 2.f);
  const int odd = (threadIdx.x >> 2) & 1;
  const int offX = (odd ? 16 : 0) + q * 4, offY = (odd ? 0 : 16) + q * 4;
  const RowBase<SM> rX(g.EPQ + offX), rY(g.EPQ + offY), rH(g.H + q * 4);      // EPQ rows: 128 bytes, H rows: 64
  for (int task = threadIdx.x; task < g.ord_rounds * NT; task += NT) {
    const int i = g.ord[task >> 2];
    if (i == kNoNode) continue;
    const F2x2 A = rY.row((unsigned)i, 7), B = rX.row((unsigned)i, 7);
    const float4 gsi4 = (ld4(g.H + i * 16 + q * 4) + ce4) * 2.f;                  // 2 (gs_i + g_me/e)
    const float2 gsa = make_float2(gsi4.x, gsi4.y), gsb = make_float2(gsi4.z, gsi4.w);
    const int beg = g.rp[i], end = g.rp[i + 1];
    float2 u0 = make_float2(0.f, 0.f), u1 = u0, v0 = u0, v1 = u0;    // u: terms of m1, v: terms of m2
    float2 w0 = u0, w1 = u0, z0 = u0, z1 = u0;                      // second chain (odd entries)
    int t = beg;
    for (; t + 1 < end; t += 2) {
      const uint32_t e0 = g.adj[t], e1 = g.adj[t + 1];
      const unsigned k0 = e0 & 0xffffu, k1 = e1 & 0xffffu;
      const F2x2 X0 = rX.row(k0, 7), Y0 = rY.row(k0, 7), h0 = rH.row(k0, 6);
      const F2x2 X1 = rX.row(k1, 7), Y1 = rY.row(k1, 7), h1 = rH.row(k1, 6);
      float2 ga0 = ffma2(h0.a, two, gsa), gb0 = ffma2(h0.b, two, gsb);
      float2 ga1 = ffma2(h1.a, two, gsa), gb1 = ffma2(h1.b, two, gsb);
      if (use_head) {
        if ((e0 >> 16) & kAdjSlotMask) {
          const F2x2 gh = ldp(g.ghead + (size_t)(((e0 >> 16) & kAdjSlotMask) - 1) * 16 + q * 4);
          ga0 = ffma2(gh.a, two, ga0); gb0 = ffma2(gh.b, two, gb0);
        }
        if ((e1 >> 16) & kAdjSlotMask) {
          const F2x2 gh = ldp(g.ghead + (size_t)(((e1 >> 16) & kAdjSlotMask) - 1) * 16 + q * 4);
          ga1 = ffma2(gh.a, two, ga1); gb1 = ffma2(gh.b, two, gb1);
        }
      }
      bwd_term<TIER>(A.a, B.a, Y0.a, X0.a, ga0, u0, v0);
      bwd_term<TIER>(A.b, B.b, Y0.b, X0.b, gb0, u1, v1);
      bwd_term<TIER>(A.a, B.a, Y1.a, X1.a, ga1, w0, z0);
      bwd_term<TIER>(A.b, B.b, Y1.b, X1.b, gb1, w1, z1);
    }
    if (t < end) {
      const uint32_t e0 = g.adj[t];
      const unsigned k0 = e0 & 0xffffu;
      const F2x2 X0 = rX.row(k0, 7), Y0 = rY.row(k0, 7), h0 = rH.row(k0, 6);
      float2 ga0 = ffma2(h0.a, two, gsa), gb0 = ffma2(h0.b, two, gsb);
      if (use_head && ((e0 >> 16) & kAdjSlotMask)) {
        const F2x2 gh = ldp(g.ghead + (size_t)(((e0 >> 16) & kAdjSlotMask) - 1) * 16 + q * 4);
        ga0 = ffma2(gh.a, two, ga0); gb0 = ffma2(gh.b, two, gb0);
      }
      bwd_term<TIER>(A.a, B.a, Y0.a, X0.a, ga0, u0, v0);
      bwd_term<TIER>(A.b, B.b, Y0.b, X0.b, gb0, u1, v1);
    }
    // bwd_term(epi:=A, eqi:=B, epk:=Y, eqk:=X): first accumulator <- terms of A X + 1, second <- terms of Y B + 1.
    // odd group:  A X = EP_i EQ_k (= a -> gP),  Y B = EP_k EQ_i (= b -> gQ);   even group: the other way round.
    const float4 t1 = make_float4(u0.x + w0.x, u0.y + w0.y, u1.x + w1.x, u1.y + w1.y);
    const float4 t2 = make_float4(v0.x + z0.x, v0.y + z0.y, v1.x + z1.x, v1.y + z1.y);
    const float4 aP = odd ? t1 : t2, aQ = odd ? t2 : t1;
    st4(g.GPQ + i * 32 + q * 4, aP);
    st4(g.GPQ + i * 32 + 16 + q * 4, aQ);
    bsum = bsum + aP;
  }
  return bsum;
}

// own-thread read-modify-write on this CTA's private gradient row (same thread always owns the same element)
// contribution of this graph to the CTA-private gradient row.  `red.global.add` has no return value, so the
// thread does not wait for the L2 round trip; the row is private to the CTA and every element is always updated
// by the same thread, so the summation order stays fixed (deterministic).
__device__ __forceinline__ void gacc(float* gp, int idx, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(gp + idx), "f"(v) : "memory");
}


// ---- small dense blocks run by single warps from shared-memory weights ------------------------------------------
// value-head and numeric-encoder weights -> the (currently free) GPQ region, with padded row strides
__device__ __forceinline__ void stage_vn_weights(const float* __restrict__ P, float* vn) {
  // all global loads are issued before the first shared store, so the thread waits for one L2 round trip, not 18
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  float a[5], b[2], c[8], d[2], e = 0.f;
#pragma unroll
  for (int j = 0; j < 5; ++j) a[j] = (t + NT * j < HID * SVD) ? __ldg(P + P_VAL_W0 + t + NT * j) : 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j) b[j] = __ldg(P + P_VAL_W1 + t + NT * j);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int u = warp + NW * j;
    c[2 * j] = __ldg(P + P_NUM_W0 + u * NUMD + lane);
    c[2 * j + 1] = lane < NUMD - 32 ? __ldg(P + P_NUM_W0 + u * NUMD + 32 + lane) : 0.f;
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) d[j] = __ldg(P + P_NUM_W1 + t + NT * j);
  if (t < 32) e = __ldg(P + P_VAL_B0 + t);
  else if (t < 64) e = __ldg(P + P_VAL_B1 + t - 32);
  else if (t < 96) e = __ldg(P + P_VAL_W2 + t - 64);
  else if (t < 160) e = __ldg(P + P_NUM_B0 + t - 96);
  else if (t < 176) e = __ldg(P + P_NUM_B1 + t - 160);
  else if (t == 176) e = __ldg(P + P_VAL_B2);
#pragma unroll
  for (int j = 0; j < 5; ++j) if (t + NT * j < HID * SVD) vn[VN_VW0 + t + NT * j] = a[j];       // same [32][67] layout
#pragma unroll
  for (int j = 0; j < 2; ++j) { const int i = t + NT * j; vn[VN_VW1 + (i >> 5) * 33 + (i & 31)] = b[j]; }
#pragma unroll
  for (int j = 0; j < 4; ++j) {                                                                  // [64][52] -> stride 53
    const int u = warp + NW * j;
    vn[VN_NW0 + u * 53 + lane] = c[2 * j];
    if (lane < NUMD - 32) vn[VN_NW0 + u * 53 + 32 + lane] = c[2 * j + 1];
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) { const int i = t + NT * j; vn[VN_NW1 + (i >> 6) * 65 + (i & 63)] = d[j]; }
  if (t < 32) vn[VN_VB0 + t] = e;
  else if (t < 64) vn[VN_VB1 + t - 32] = e;
  else if (t < 96) vn[VN_VW2 + t - 64] = e;
  else if (t < 160) vn[VN_NB0 + t - 96] = e;
  else if (t < 176) vn[VN_NB1 + t - 160] = e;
  else if (t == 176) vn[VN_VB2] = e;
}
static_assert(NT == 512 && NW == 16, "stage_vn_weights is laid out for 512 threads");

__device__ __forceinline__ void group_bar(int id, int nthreads) {      // named barrier of a warp group
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// numeric feature encoder (state_encoder.py:35-57,187).  Layer 0: all 512 threads, 8 lanes per hidden unit (two warps
// alone would arrive late at the next barrier).
__device__ __forceinline__ void numeric_l0(const float* vn, const float* x52, float* a0, int tid) {
  const int u = tid >> 3, p = tid & 7;
  const float* w = vn + VN_NW0 + u * 53;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const int c = p + 8 * k;
    if (c < NUMD) s = fmaf(w[c], x52[c], s);
  }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (p == 0) a0[u] = tanhf(s + vn[VN_NB0 + u]);
}
// Layer 1: one warp, 16 units x 2 halves of the 64 inputs
__device__ __forceinline__ void numeric_l1(const float* vn, const float* a0, float* hnum, int lane) {
  const int r = lane & 15, half = lane >> 4;
  const float* w = vn + VN_NW1 + r * 65 + half * 32;
  const float* x = a0 + half * 32;
  float s0 = 0.f, s1 = 0.f;
#pragma unroll 16
  for (int k = 0; k < 32; k += 2) { s0 = fmaf(w[k], x[k], s0); s1 = fmaf(w[k + 1], x[k + 1], s1); }
  float s = s0 + s1;
  s += __shfl_xor_sync(0xffffffffu, s, 16);
  if (lane < 16) hnum[r] = tanhf(s + vn[VN_NB1 + r]);
}

// Attention tail (hbar, v' = Vc hbar + vbc, att = Wo v' + bo) in one warp's registers; lane & 15 = component.
// `tmp` holds the block reduction of pass 2: tmp[0..15] = sum_i a_i h_i, tmp[16] = sum_i a_i.
__device__ __forceinline__ void attention_tail(const float* sW, const float* tmp, int lane, float& hbar, float& vp,
                                               float& at) {
  const int c = lane & 15;
  hbar = tmp[c] / tmp[16];
  vp = sW[S_VBC + c];
#pragma unroll
  for (int j = 0; j < 16; ++j) vp = fmaf(sW[S_VCT + j * 16 + c], __shfl_sync(0xffffffffu, hbar, j), vp);
  at = sW[S_BO + c];
#pragma unroll
  for (int j = 0; j < 16; ++j) at = fmaf(sW[S_WOT + j * 16 + c], __shfl_sync(0xffffffffu, vp, j), at);
}

// Value head (value.py:15-39) by the 256 threads of warps 0..7: 8 lanes per hidden unit, named barrier 1.
__device__ __forceinline__ void value_head_group(float* sV, const float* vn, float* sc, int tid) {
  const int r = tid >> 3, p = tid & 7, lane = tid & 31;
  {
    const float* w = vn + VN_VW0 + r * SVD;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      const int k = p + 8 * j;
      if (k < SVD) s = fmaf(w[k], sV[V_SV + k], s);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if (p == 0) sV[V_Y0 + r] = tanhf(s + vn[VN_VB0 + r]);
  }
  group_bar(1, 256);
  {
    const float* w = vn + VN_VW1 + r * 33;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) s = fmaf(w[p + 8 * j], sV[V_Y0 + p + 8 * j], s);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if (p == 0) sV[V_Y1 + r] = tanhf(s + vn[VN_VB1 + r]);
  }
  group_bar(1, 256);
  if (tid < 32) {
    const float v = warp_sum(vn[VN_VW2 + lane] * sV[V_Y1 + lane]) + vn[VN_VB2];
    if (lane == 0) sc[SC_VALUE] = v;
  }
}

// Backward of the value head and of the numeric encoder by the 256 threads of warps 0..7 (named barrier 2);
// leaves g_sv in sV[V_GSV..] and adds the weight gradients to the CTA's gradient row.
__device__ __forceinline__ void value_numeric_bwd_group(float* sV, const float* vn, float gV, float* gp, int tid) {
  const int r = tid >> 3, p = tid & 7;
  if (tid < 32) {
    const float y1 = sV[V_Y1 + tid];
    sV[V_D1 + tid] = gV * vn[VN_VW2 + tid] * (1.f - y1 * y1);
  }
  group_bar(2, 256);
  {   // d0[c] = (sum_q W1[q][c] d1[q]) (1 - y0[c]^2): c = r, 8 lanes x 4 q
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) s = fmaf(vn[VN_VW1 + (p + 8 * j) * 33 + r], sV[V_D1 + p + 8 * j], s);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    const float y0 = sV[V_Y0 + r];
    if (p == 0) sV[V_D0 + r] = s * (1.f - y0 * y0);
    // W1 / biases / W2 gradients need d1, y0, y1 only
#pragma unroll
    for (int j = 0; j < 4; ++j) gacc(gp, P_VAL_W1 + r * 32 + p + 8 * j, sV[V_D1 + r] * sV[V_Y0 + p + 8 * j]);
    if (tid < 32) {
      gacc(gp, P_VAL_B1 + tid, sV[V_D1 + tid]);
      gacc(gp, P_VAL_W2 + tid, gV * sV[V_Y1 + tid]);
    }
    if (tid == 32) gacc(gp, P_VAL_B2, gV);
  }
  group_bar(2, 256);
  if (tid < SVD) {   // g_sv[k] = sum_r W0[r][k] d0[r]
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
    for (int q = 0; q < 32; q += 2) {
      s0 = fmaf(vn[VN_VW0 + q * SVD + tid], sV[V_D0 + q], s0);
      s1 = fmaf(vn[VN_VW0 + (q + 1) * SVD + tid], sV[V_D0 + q + 1], s1);
    }
    sV[V_GSV + tid] = s0 + s1;
  }
  {   // W0 gradient: row r, columns p, p+8, ...
    const float d0 = sV[V_D0 + r];
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      const int k = p + 8 * j;
      if (k < SVD) gacc(gp, P_VAL_W0 + r * SVD + k, d0 * sV[V_SV + k]);
    }
    if (tid < 32) gacc(gp, P_VAL_B0 + tid, sV[V_D0 + tid]);
  }
  group_bar(2, 256);
  if (tid < 16) {
    const float hn = sV[V_SV + tid];
    sV[V_DN1 + tid] = sV[V_GSV + tid] * (1.f - hn * hn);
  }
  group_bar(2, 256);
  {   // dn0[u] = (sum_r NW1[r][u] dn1[r]) (1 - a0[u]^2): u = tid >> 2 (64 units), 4 lanes x 4 r
    const int u = tid >> 2, pp = tid & 3;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) s = fmaf(vn[VN_NW1 + (pp + 4 * j) * 65 + u], sV[V_DN1 + pp + 4 * j], s);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    const float a0 = sV[V_A0 + u];
    if (pp == 0) sV[V_DN0 + u] = s * (1.f - a0 * a0);
#pragma unroll
    for (int j = 0; j < 4; ++j) {          // NW1 gradient: 16 x 64 = 1024 = 256 threads x 4
      const int idx = tid + 256 * j;
      gacc(gp, P_NUM_W1 + idx, sV[V_DN1 + (idx >> 6)] * sV[V_A0 + (idx & 63)]);
    }
    if (tid < 16) gacc(gp, P_NUM_B1 + tid, sV[V_DN1 + tid]);
  }
  group_bar(2, 256);
  {   // NW0 gradient: unit u = tid >> 2, columns pp, pp+4, ... (52 = 4 x 13)
    const int u = tid >> 2, pp = tid & 3;
    const float d = sV[V_DN0 + u];
#pragma unroll
    for (int j = 0; j < 13; ++j) gacc(gp, P_NUM_W0 + u * NUMD + pp + 4 * j, d * sV[V_X52 + pp + 4 * j]);
    if (tid < NH0) gacc(gp, P_NUM_B0 + tid, sV[V_DN0 + tid]);
  }
}

// Policy head on one candidate by a HALF-warp: lane c16 owns input channel c16 and hidden units c16, c16 + 16.
// Returns the two tanh units and the candidate's input channel (he of the edge, or h^L of the node).
struct HeadLane {
  float w0[16], w1[16];      // rows c16 and c16+16 of the (effective) first-layer matrix
  float cb0, cb1, w20, w21;
  unsigned mask;             // the half-warp's lanes
};
__device__ __forceinline__ void head_lane_init(HeadLane& hl, const GraphView& g, const float* sW, const float* sV,
                                               int lane) {
  const int c16 = lane & 15;
  hl.mask = 0xFFFFu << (lane & 16);
  const float* WT = g.stage == 0 ? sV + V_WEFFT : sW + S_RDW0T;      // [16][32]: conflict-free for lane = unit
#pragma unroll
  for (int c = 0; c < 16; ++c) { hl.w0[c] = WT[c * 32 + c16]; hl.w1[c] = WT[c * 32 + c16 + 16]; }
  if (g.stage == 0) {
    hl.cb0 = sV[V_CEFF + c16]; hl.cb1 = sV[V_CEFF + c16 + 16];
    hl.w20 = sW[S_LUW1 + c16]; hl.w21 = sW[S_LUW1 + c16 + 16];
  } else {
    hl.cb0 = sW[S_RDB0 + c16]; hl.cb1 = sW[S_RDB0 + c16 + 16];
    hl.w20 = sW[S_RDW1 + c16]; hl.w21 = sW[S_RDW1 + c16 + 16];
  }
}
__device__ __forceinline__ void head_units(const HeadLane& hl, const GraphView& g, int j, int lane, bool raw, float& t0,
                                           float& t1, float& xin) {
  const int c16 = lane & 15;
  const uint32_t uv = g.cuv[j];
  if (g.stage == 0) {
    const int u = uv & 0xffffu, v = uv >> 16;
    const float epu = g.EPQ[u * 32 + c16], equ = g.EPQ[u * 32 + 16 + c16];
    const float epv = g.EPQ[v * 32 + c16], eqv = g.EPQ[v * 32 + 16 + c16];
    float a, b;
    if (raw) { a = exp2a(epu + eqv) + 1.f; b = exp2a(epv + equ) + 1.f; }
    else { a = fmaf(epu, eqv, 1.f); b = fmaf(epv, equ, 1.f); }
    xin = (1.f - rcp_approx(a)) - rcp_approx(b);
  } else {
    xin = g.H[(int)uv * 16 + c16];
  }
  float p0 = hl.cb0, p1 = hl.cb1;
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const float x = __shfl_sync(hl.mask, xin, c, 16);
    p0 = fmaf(hl.w0[c], x, p0);
    p1 = fmaf(hl.w1[c], x, p1);
  }
  t0 = tanhf(p0);
  t1 = tanhf(p1);
}
__device__ __forceinline__ float half_sum(float v, unsigned mask) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o, 16);
  return v;
}

// Graph gid's masked logit row, or nullptr when it has none (no row number, or no matrix for its stage).  The row is
// `width` floats: the context's cap of the stage, the reference's max_num_edges / max_num_nodes padding.
__device__ __forceinline__ float* logit_row(const StepArgs& a, int gid, int stage, int& width) {
  width = stage == 0 ? a.e_cap : a.n_cap;
  float* base = stage == 0 ? a.lu_logits : a.rd_logits;
  const int row = a.logit_rows[gid];
  return row < 0 || base == nullptr ? nullptr : base + (size_t)row * width;
}

// dst[0, width) = v by the threads t0, t0 + step, ...: float4 stores when dst is 16-byte aligned
__device__ __forceinline__ void fill_row(float* dst, int width, float v, int t0, int step) {
  int i = t0;
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (; i < width >> 2; i += step) d4[i] = make_float4(v, v, v, v);
    i = ((width >> 2) << 2) + t0;
  }
  for (; i < width; i += step) dst[i] = v;
}

// One warp: the graph's row of the reference's masked logits (policy.py:48-61): the fill value everywhere, then each
// candidate's logit at its index.  The fill covers the whole padded width, whatever the graph's own e or n.
__device__ __forceinline__ void write_logit_row(const StepArgs& a, const GraphView& g, int lane) {
  int width;
  float* dst = logit_row(a, g.gid, g.stage, width);
  if (dst == nullptr) return;
  fill_row(dst, width, MASK_FILL, lane, 32);
  __syncwarp();
  for (int j = lane; j < g.k; j += 32) dst[g.cidx[j]] = g.z[j];
}

// The whole CTA: a NaN row for a graph the kernel skips (larger than the context's caps), as its value and log-prob
template <int NTHREADS>
__device__ __forceinline__ void write_skipped_logit_row(const StepArgs& a, int gid, int stage) {
  if (a.logit_rows == nullptr) return;
  int width;
  float* dst = logit_row(a, gid, stage, width);
  if (dst != nullptr) fill_row(dst, width, CUDART_NAN_F, threadIdx.x, NTHREADS);
}

// Value-loss seed of one graph: g = c_v / B * d(loss)/dV, the loss term it adds to statistics slot 0 or 15, and whether
// the clipped branch won (slot 16).  Both places that form g_V call this: softmax_seeds and the SGNN's value-backward
// warps.  Off (old_values NULL): (V - R)^2, today's arithmetic.  On: the clipped value loss of OpenAI baselines' ppo2 /
// CleanRL's clip_vloss, in torch's fp32 operations and order,
//   d = V - V_old,  Vc = V_old + clamp(d, -c, c),  a = (V - R)^2,  b = (Vc - R)^2,  loss = max(a, b),
// with the gradient of torch.maximum (a tie sends half to each input) and of the inclusive clamp.  V_old + d need not
// round back to V, so a and b can differ in the last bits inside the clamp: the branch is taken as torch takes it.
// Huber (huber_delta = delta > 0) replaces each square e^2 by h(e) = 2 huber_loss(e; delta) and its gradient 2 e by
// 2 clamp(e, -delta, delta) (huber_term, huber_clamp); `linear` is 1 where the chosen term (a on a tie) has |e| > delta
// (slot 21).  The seed keeps the order 2 c_v e (1/B), so a delta above every |V - R| gives the step without Huber.
struct ValueSeed {
  float g, loss, clipped, linear;
};
// 2 * torch.nn.functional.huber_loss in fp32 as torch forms it: z^2 (= e * e) for z = |e| < delta, else
// 2 (delta (z - delta / 2)); NaN stays NaN
__device__ __forceinline__ float huber_term(float e, float delta) {
  const float z = fabsf(e);
  return z < delta ? z * z : 2.f * (delta * (z - 0.5f * delta));
}
// torch.clamp(e, -delta, delta) (huber_loss's backward): NaN passes through
__device__ __forceinline__ float huber_clamp(float e, float delta) {
  return e < -delta ? -delta : (e > delta ? delta : e);
}
__device__ __forceinline__ ValueSeed value_seed(const StepArgs& a, float V, float R, float V_old) {
  const float dv = V - R, hd = a.huber_delta;
  if (a.old_values == nullptr) {
    if (hd == 0.f) return {2.f * a.c_value * dv * a.inv_batch, dv * dv, 0.f, 0.f};
    return {2.f * a.c_value * huber_clamp(dv, hd) * a.inv_batch, huber_term(dv, hd), 0.f,
            fabsf(dv) > hd ? 1.f : 0.f};
  }
  const float c = a.value_clip;
  const float d = V - V_old, Vc = V_old + fminf(fmaxf(d, -c), c), dvc = Vc - R;
  const float la = hd == 0.f ? dv * dv : huber_term(dv, hd), lb = hd == 0.f ? dvc * dvc : huber_term(dvc, hd);
  const float ga = 2.f * (hd == 0.f ? dv : huber_clamp(dv, hd));
  const float gb = (d >= -c && d <= c) ? 2.f * (hd == 0.f ? dvc : huber_clamp(dvc, hd)) : 0.f;
  const float g = la > lb ? ga : (lb > la ? gb : 0.5f * ga + 0.5f * gb);
  return {a.c_value * g * a.inv_batch, lb > la ? lb : la, lb > la ? 1.f : 0.f,
          hd != 0.f && fabsf(lb > la ? dvc : dv) > hd ? 1.f : 0.f};
}

// first element of graph gid's candidates in the blob's candidate section (and in the per-candidate log-prob arrays)
__device__ __forceinline__ int cand_offset(const StepArgs& a, const BlobHeader& hd, int gid) {
  return reinterpret_cast<const GraphDesc*>(a.blob + hd.off_desc)[gid].cand_off;
}

// The whole CTA: NaN log-probs for the candidates of a graph the kernel skips (larger than the context's caps)
template <int NTHREADS>
__device__ __forceinline__ void write_skipped_cand_logp(const StepArgs& a, const GraphDesc& d) {
  if (a.out_cand_logp == nullptr) return;
  for (int j = threadIdx.x; j < d.k; j += NTHREADS) a.out_cand_logp[d.cand_off + j] = CUDART_NAN_F;
}

// One warp: masked softmax over the k candidates (log-softmax over the candidates equals log-softmax over all
// padded logits: masked entries have probability exactly 0), outputs, PPO seeds and the logit gradients.
template <bool TRAIN>
__device__ __forceinline__ void softmax_seeds(const StepArgs& a, const BlobHeader& hd, const GraphView& g, float* sc,
                                              float* stats, int lane, int item) {   // stats: the CTA's statistics slots;
                                                                                    // item: the graph's position in ids
  const int k = g.k, gid = g.gid;
  float lmax = -CUDART_INF_F;
  int lbest = 0x7fffffff;
  for (int j = lane; j < k; j += 32) {
    const float zj = g.z[j];
    if (zj > lmax) { lmax = zj; lbest = j; }     // first index wins inside a lane (j ascending)
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {             // arg-max with first-index tie break (policy.py:72 `probs.argmax`)
    const float om = __shfl_xor_sync(0xffffffffu, lmax, o);
    const int ob = __shfl_xor_sync(0xffffffffu, lbest, o);
    if (om > lmax || (om == lmax && ob < lbest)) { lmax = om; lbest = ob; }
  }
  const float zmax = lmax;
  float lsum = 0.f;
  for (int j = lane; j < k; j += 32) lsum += expf(g.z[j] - zmax);
  const float lse = zmax + logf(warp_sum(lsum));
  const int aidx = a.actions ? (int)sc[SC_ACT] : -1;
  float lent = 0.f;
  int slot = -1;
  for (int j = lane; j < k; j += 32) {
    const float lp = g.z[j] - lse;
    lent -= expf(lp) * lp;
    if (g.cidx[j] == aidx) slot = j;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) slot = max(slot, __shfl_xor_sync(0xffffffffu, slot, o));
  float H = warp_sum(lent), logp = 0.f;
  int greedy = 0;
  if (k > 0) {
    greedy = g.cidx[lbest];
    if (a.actions) logp = slot >= 0 ? g.z[slot] - lse : MASK_FILL - lse;
  } else {      // every logit equals the fill value -2^32+1.  The distribution is uniform over the padded width, but the
                // reference's fp32 log-softmax returns 0 for every entry (logsumexp = fill + log(width) rounds back to
                // fill, ulp 512): log_prob = 0, entropy = 0 -- measured on the unmodified reference
                // (tests/golden/edge_empty.npz) and reproduced here
    H = 0.f;
    logp = 0.f;
  }
  const float V = sc[SC_VALUE];
  if (lane == 0) {
    sc[SC_LSE] = lse; sc[SC_ENT] = H; sc[SC_LOGP] = logp; sc[SC_SLOT] = (float)(slot + 1);
    if (a.out_value) a.out_value[gid] = V;
    if (a.out_logp) a.out_logp[gid] = logp;
    if (a.out_entropy) a.out_entropy[gid] = H;
    if (a.out_greedy) a.out_greedy[gid] = greedy;
    if (!TRAIN && a.out_pos_logp) a.out_pos_logp[item] = logp;
  }
  if constexpr (!TRAIN) {
    if (a.logit_rows != nullptr) write_logit_row(a, g, lane);
    if (a.out_cand_logp != nullptr) {
      float* dst = a.out_cand_logp + cand_offset(a, hd, gid);
      for (int j = lane; j < k; j += 32) dst[j] = g.z[j] - lse;
    }
    // Sampled action (policy.py:81-83 `dist.sample()`), from a caller-supplied uniform u in [0, 1): the first
    // candidate, in index order, of positive fp32 probability exp(z - zmax) / sum whose cumulative term sum exceeds
    // u * sum.  A zero-probability candidate (logit gap beyond ~104, where the probability rounds to 0) is never
    // picked, as Categorical.sample never returns one: not at u = 0 (hence the strict '>'), not where the scan's
    // per-lane association rounds its cumulative sum above its predecessor's (hence the explicit test), and not when
    // u * sum rounds to or above the scan's total (then the last candidate of positive probability).  (torch's sampler
    // consumes its generator differently, so sampled rollouts are reproducible per uniform stream, not bit-equal to
    // Categorical.sample.)
    if (a.uniforms != nullptr && a.out_sample != nullptr) {
      const float u = a.uniforms[gid];
      int pick = -1;
      if (k > 0) {
        const float S = warp_sum(lsum), target = u * S;
        float run = 0.f;
        int last = -1;                                    // the last candidate of positive probability so far
        for (int base = 0; base < k && pick < 0; base += 32) {
          const int j = base + lane;
          const float ej = j < k ? expf(g.z[j] - zmax) : 0.f;
          float c = ej;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, c, o);
            if (lane >= o) c += t;
          }
          c += run;
          const unsigned pos = __ballot_sync(0xffffffffu, ej / S > 0.f);
          const unsigned hit = pos & __ballot_sync(0xffffffffu, c > target);
          if (hit) pick = base + __ffs(hit) - 1;
          if (pos) last = base + 31 - __clz(pos);
          run = __shfl_sync(0xffffffffu, c, 31);
        }
        if (pick < 0) pick = last;                        // u * sum rounded to or above the scan's total; the arg-max
                                                          // has probability 1 / sum >= 1 / k, so `last` is set
        pick = g.cidx[pick];
      } else {                                            // empty mask: uniform over the padded width
        const int cap = g.stage == 0 ? hd.e_cap : hd.n_cap;
        pick = min(cap - 1, max(0, (int)(u * (float)cap)));
      }
      if (lane == 0) a.out_sample[gid] = pick;
    }
  }
  if constexpr (TRAIN) {
    const float R = sc[SC_RET], dv = V - R;
    float glp = 0.f, gH = 0.f, surr = 0.f, negent = 0.f, in_ind = 0.f, kl = 0.f, clipped = 0.f, dual = 0.f;
    float pw = 0.f, pkl = 0.f;
    if (sc[SC_EXP] != 0.f) {
      in_ind = 1.f;
      const float dlp = logp - sc[SC_FLP];
      // EWMA proximal policy (a.prox_lp): the clip acts on r = exp(lp - lp_p), and the constant behaviour weight
      // w = exp(lp_p - lp_b) multiplies the surrogate and its gradient below.  Off, r = exp(lp - lp_b) as before.
      const float r = expf(a.prox_lp != nullptr ? logp - sc[SC_PLP] : dlp), A = sc[SC_ADV];
      const float lo = a.clip_lo, hi = a.clip_hi;
      const float s1 = r * A, s2 = fminf(fmaxf(r, lo), hi) * A;
      const bool inside = r >= lo && r <= hi;
      surr = -fminf(s1, s2);
      if (inside || s1 < s2) glp = -A * r * a.inv_ind;
      // dual clip (Ye et al. 2020, Tianshou's dual_clip): for A < 0 the surrogate is max(clip1, c A), c A constant.
      // torch.maximum's gradient: none where c A wins, half on an exact tie; a NaN clip1 stays (no branch taken)
      if (a.dual_clip != 0.f && A < 0.f) {
        const float cA = a.dual_clip * A, clip1 = fminf(s1, s2);
        if (cA > clip1) {
          surr = -cA; glp = 0.f; dual = 1.f;
        } else if (cA == clip1) {
          glp *= 0.5f;
        }
      }
      gH = -a.c_entropy * a.inv_ind;
      negent = -H;
      kl = expm1f(dlp) - dlp;       // (r - 1) - log r >= 0, an estimate of KL(old || new), without r - 1's cancellation
      clipped = inside ? 0.f : 1.f;
      if (a.prox_lp != nullptr) {   // slot 8 above stays against the behaviour log-probs; slots 9 and 20 use r
        const float d = sc[SC_PLP] - sc[SC_FLP];
        pw = expf(d);
        pkl = expm1f(d) - d;
        surr *= pw;
        glp *= pw;
      }
    }
    if (lane == 0) {
      const ValueSeed vs = value_seed(a, V, R, sc[SC_VOLD]);
      sc[SC_GV] = vs.g;
      // fire-and-forget adds (gacc): a read-modify-write would park this warp on an L2 round trip before the
      // logit-gradient loop below; same thread, same addresses, so the summation order is still fixed
      gacc(stats, 0, dv * dv); gacc(stats, 1, surr); gacc(stats, 2, negent); gacc(stats, 3, 1.f); gacc(stats, 4, in_ind);
      gacc(stats, 5, g.stage == 0 ? 1.f : 0.f); gacc(stats, 6, g.stage == 1 ? 1.f : 0.f);
      gacc(stats, 7, (isfinite(V) && isfinite(logp) && isfinite(H)) ? 0.f : 1.f);
      if (a.diagnostics || a.kl_stop) gacc(stats, 8, kl);       // the KL stop decides on slot 8
      if (a.diagnostics) {
        gacc(stats, 9, clipped); gacc(stats, 10, R); gacc(stats, 11, R * R); gacc(stats, 12, dv);
      }
      if (a.old_values || a.huber_delta != 0.f) gacc(stats, VCLIP_LOSS_SLOT, vs.loss);
      if (a.old_values) gacc(stats, VCLIP_COUNT_SLOT, vs.clipped);
      if (a.dual_clip != 0.f) gacc(stats, DUAL_COUNT_SLOT, dual);
      if (a.huber_delta != 0.f) gacc(stats, HUBER_COUNT_SLOT, vs.linear);
      if (a.prox_lp != nullptr) { gacc(stats, PROX_WEIGHT_SLOT, pw); gacc(stats, PROX_KL_SLOT, pkl); }
    }
    // logits gradient: g_z = g_lp (delta_a - p) - g_H p (logp + H)
    const float* lpo = (a.old_cand_logp != nullptr && in_ind != 0.f) ? a.old_cand_logp + cand_offset(a, hd, gid)
                                                                       : nullptr;
    if (lpo == nullptr) {
      for (int j = lane; j < k; j += 32) {
        const float lp = g.z[j] - lse, p = expf(lp);
        g.gz[j] = glp * ((j == slot ? 1.f : 0.f) - p) - gH * p * (lp + H);
      }
    } else {
      // KL penalty beta * KL(pi_old || pi), exact over the candidates: KL_g = sum_c p_old (lp_old - lp), taken in log
      // space (a new probability that underflows gives a large finite term, not inf; a p_old that underflows adds 0),
      // and its logit gradient beta / |ind| (p - p_old)
      const float kpen = a.kl_coef * a.inv_ind;
      float lkl = 0.f;
#pragma unroll 1      // not unrolled: this path's code stays small in the graph loop's instruction footprint
      for (int j = lane; j < k; j += 32) {
        const float lp = g.z[j] - lse, p = expf(lp);
        const float lo = lpo[j], po = expf(lo);
        if (po > 0.f) lkl += po * (lo - lp);
        g.gz[j] = glp * ((j == slot ? 1.f : 0.f) - p) - gH * p * (lp + H) + kpen * (p - po);
      }
      const float klg = warp_sum(lkl);
      if (lane == 0) {
        gacc(stats, KLPEN_SLOT, klg);
        if (!isfinite(klg)) gacc(stats, 7, 1.f);
      }
    }
  }
}

// pull the NEXT graph of this CTA into L2 while the current one is processed (its first touches are then L2 hits):
// feature rows, adjacency, row pointers, pull schedule, and the sample's small rows (numerical / current-node features,
// action, return, ...).  Out of line: once per graph, and its address arithmetic stays out of the graph body's
// register allocation.
template <bool TRAIN>
__device__ __noinline__ void prefetch_next_graph(const StepArgs& a, int nitem) {
  const int T0 = threadIdx.x, TN = NT;
  const BlobHeader& hd = *reinterpret_cast<const BlobHeader*>(a.blob);
  const GraphDesc* descs = reinterpret_cast<const GraphDesc*>(a.blob + hd.off_desc);
  const int ng = a.ids ? a.ids[nitem] : nitem;
  const GraphDesc& nd = descs[ng];
  const char* px = reinterpret_cast<const char*>(a.blob + hd.off_x) + (size_t)nd.x_row * FS * 4;
  const char* pa = reinterpret_cast<const char*>(a.blob + hd.off_adj) + (size_t)nd.adj_off * 4;
  const char* pr = reinterpret_cast<const char*>(a.blob + hd.off_rowptr) + (size_t)nd.rp_off * 2;
  const char* po = reinterpret_cast<const char*>(a.blob + hd.off_order) + (size_t)nd.ord_off * 2;
  const int bx = nd.n * FS * 4, ba = nd.e * 8, br = (nd.n + 1) * 2, bo = nd.ord_rounds * NW * 16;
  for (int o = T0 * 128; o < bx; o += TN * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(px + o));
  for (int o = T0 * 128; o < ba; o += TN * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pa + o));
  for (int o = T0 * 128; o < br; o += TN * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pr + o));
  for (int o = T0 * 128; o < bo; o += TN * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(po + o));
  if (T0 >= TN - 32) {
    const int w = T0 - (TN - 32);
    const void* q = nullptr;
    if (w < 3) q = reinterpret_cast<const char*>(a.blob + hd.off_num) + (size_t)ng * NUMD * 4 + min(w * 128, NUMD * 4 - 4);
    else if (w < 5) q = reinterpret_cast<const char*>(a.blob + hd.off_cur) + (size_t)ng * FS * 4 + (w - 3) * (FS * 4 - 4);
    else if (w == 5) q = a.actions ? a.actions + (size_t)ng * 2 : nullptr;
    else if (TRAIN && w == 6) q = a.ret + ng;
    else if (TRAIN && w == 7) q = a.exps + ng;
    else if (TRAIN && w == 8) q = a.fixed_lp + ng;
    else if (TRAIN && w == 9) q = a.adv + ng;
    else if (TRAIN && w == 10) q = a.old_values ? a.old_values + ng : nullptr;
    if (q) asm volatile("prefetch.global.L2 [%0];" ::"l"(q));
  }
}

// partial g_W tile of one warp on the tensor cores: redbuf[warp][o][c] = sum over this warp's nodes of GPQ[i][o] h[i][c],
// i.e. A = GPQ^T (32 x K: two m-tiles) times B = h (K x 16: two n-tiles), K = nodes, 3xTF32 (mma_3x).  A k-step takes
// 8 consecutive nodes (tile column t -> node 8 kc + t); the warp takes k-steps kc = warp, warp + KW, ..., two per trip.
// Tile rows and columns are permuted so that every fragment is one vector load: A row 8 j + g is output o = 4 g + j, B
// column 8 j + g is channel c = 2 g + j.  Lane (g, t) then loads GPQ[node][4g .. 4g+3] (a warp reads four whole 128 B rows:
// four wavefronts, the least 512 B can take) and h[node][2g, 2g+1] (four whole 64 B rows), and its accumulators hold
// the 4 x 4 tile o in [4g, 4g+4), c in [4t, 4t+4).  SMEM: h rows staged in shared memory, else read from the global
// scratch (L2).
template <bool SMEM>
__device__ __forceinline__ void gw_partial(const GraphView& g, const float* hin, int n, float* redbuf) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gq = lane >> 2, t = lane & 3;
  float acc[2][2][4];   // [m-tile][n-tile][fragment]
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mt][nt][q] = 0.f;
  for (int kc = warp; kc * 8 < n; kc += 2 * KW) {   // two k-steps per trip: all their rows are in flight together
    float4 ga[2][2];    // [k-step][tile column t, t + 4]
    float2 hb[2][2];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int i = (kc + u * KW) * 8 + s * 4 + t;
        const bool ok = i < n;
        if constexpr (SMEM) hb[u][s] = ok ? *reinterpret_cast<const float2*>(hin + i * 16 + 2 * gq) : make_float2(0.f, 0.f);
        else hb[u][s] = ok ? __ldcg(reinterpret_cast<const float2*>(hin + (size_t)i * 16 + 2 * gq)) : make_float2(0.f, 0.f);
        ga[u][s] = ok ? ld4(g.GPQ + i * 32 + 4 * gq) : f4(0.f);
      }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      uint32_t bh[2][2], bl[2][2];   // [n-tile][tile row t, t + 4]
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        tf32_split(hb[u][s].x, bh[0][s], bl[0][s]);
        tf32_split(hb[u][s].y, bh[1][s], bl[1][s]);
      }
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        mma_3x(acc[0][nt], ga[u][0].x, ga[u][0].y, ga[u][1].x, ga[u][1].y, bh[nt][0], bh[nt][1], bl[nt][0], bl[nt][1]);
        mma_3x(acc[1][nt], ga[u][0].z, ga[u][0].w, ga[u][1].z, ga[u][1].w, bh[nt][0], bh[nt][1], bl[nt][0], bl[nt][1]);
      }
    }
  }
  // acc[mt][nt][q] is o = 4 gq + 2 mt + (q >> 1), c = 4 t + 2 (q & 1) + nt
#pragma unroll
  for (int x = 0; x < 4; ++x) {
    const int mt = x >> 1, r = 2 * (x & 1);
    st4(redbuf + warp * 512 + (gq * 4 + x) * 16 + t * 4,
        make_float4(acc[mt][0][r], acc[mt][1][r], acc[mt][0][r + 1], acc[mt][1][r + 1]));
  }
}

#define UPB_STAMP(ID)                                                                      \
  do {                                                                                     \
    if (a.stamps != nullptr && blockIdx.x == 0 && threadIdx.x == 0 && first_item) a.stamps[ID] = clock64(); \
  } while (0)

// probe: arrival time of every warp at one point of the graph body (moved around while tuning; tools/phase_times.py)
#define UPB_WSTAMP()                                                                                         \
  do {                                                                                                       \
    if (a.stamps != nullptr && blockIdx.x == 0 && (threadIdx.x & 31) == 0 && first_item)                      \
      a.stamps[46 + (threadIdx.x >> 5)] = clock64();                                                         \
  } while (0)

#define UPB_WSTAMP_B()                                                                                       \
  do {                                                                                                       \
    if (a.stamps != nullptr && blockIdx.x == 0 && (threadIdx.x & 31) == 0 && first_item && threadIdx.x < 384) \
      a.stamps[212 + (threadIdx.x >> 5)] = clock64();                                                        \
  } while (0)

// VALUES (with !TRAIN): the value-only sweep (k_sgnn_values): the body stops once the value head has written the value;
// the policy head, its candidate staging and the softmax warp do not run.
template <bool TRAIN, bool BIG, bool VALUES = false>
__device__ void graph_body(const StepArgs& a, const BlobHeader& hd, const GraphDesc& d, int gid, int item, float* smem,
                           float* gp, float* scr, bool first_item, uint64_t* mbar, unsigned mpar) {
  static_assert(!(TRAIN && VALUES), "the value-only sweep is a forward");
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q = tid & 3;
  UPB_STAMP(0);
  float* sW = smem;
  float* sV = smem + S_VEC;
  float* sRed = smem + S_RED;
  float* sc = sV + V_SC;
  const float* P = a.params;

  GraphView g;
  g.n = d.n; g.e = d.e; g.k = d.k; g.stage = d.stage; g.gid = gid;
  g.x = reinterpret_cast<const float*>(a.blob + hd.off_x) + (size_t)d.x_row * FS;
  const float* gnum = reinterpret_cast<const float*>(a.blob + hd.off_num) + (size_t)gid * NUMD;
  const float* gcur = reinterpret_cast<const float*>(a.blob + hd.off_cur) + (size_t)gid * FS;
  const uint16_t* rp_g = reinterpret_cast<const uint16_t*>(a.blob + hd.off_rowptr) + d.rp_off;
  const uint16_t* ord_g = reinterpret_cast<const uint16_t*>(a.blob + hd.off_order) + d.ord_off;
  g.ord_rounds = d.ord_rounds;
  const uint32_t* adj_g = reinterpret_cast<const uint32_t*>(a.blob + hd.off_adj) + d.adj_off;
  const uint32_t* cuv_g = reinterpret_cast<const uint32_t*>(a.blob + hd.off_cand_uv) + d.cand_off;
  const int* cidx_g = reinterpret_cast<const int*>(a.blob + hd.off_cand_idx) + d.cand_off;
  const int n = g.n, e = g.e, k = g.k;
  g.H0g = scr;
  g.H1g = scr + (size_t)a.n_cap * 16;
  float* E0g = scr + (size_t)a.n_cap * 32;        // [n][32] saved EPQ of layer 0 (reloaded by the backward pass)
  if constexpr (BIG) {
    float* b = scr + (size_t)a.n_cap * 64;
    g.EPQ = b;  b += (size_t)a.n_cap * 32;
    g.GPQ = b;  b += (size_t)a.n_cap * 32;
    g.H = b;    b += (size_t)a.n_cap * 16;
    g.inv = b;  b += a.n_cap;
    g.alpha = b; b += a.n_cap;
    const size_t kcap = (size_t)(a.e_cap > a.n_cap ? a.e_cap : a.n_cap);
    g.z = b;    b += kcap;
    g.gz = b;   b += kcap;
    g.ghead = b;
    g.rp = rp_g; g.adj = adj_g; g.cuv = cuv_g; g.cidx = cidx_g; g.ord = ord_g;
  } else {
    g.EPQ = smem + S_EPQ; g.GPQ = smem + S_GPQ; g.H = smem + S_H; g.inv = smem + S_INV;
    g.alpha = smem + S_ALPHA; g.z = smem + S_Z; g.gz = smem + S_GZ; g.ghead = smem + S_GHEAD;
    uint16_t* rp_s = reinterpret_cast<uint16_t*>(smem + S_RP);
    uint32_t* adj_s = reinterpret_cast<uint32_t*>(smem + S_ADJ);
    uint32_t* cuv_s = reinterpret_cast<uint32_t*>(smem + S_CUV);
    int* cidx_s = reinterpret_cast<int*>(smem + S_CIDX);
    // stage the graph's neighbourhood lists and node features in shared memory: one bulk copy (TMA) per blob section,
    // issued by one thread, all in flight together; blob sections are padded to 16 bytes.  The features park in the EPQ
    // region, which is idle until the first EPQ phase.  (reference op being staged: the per-sample gathers of
    // state_encoder.py:110-148 read these neighbourhoods from padded (B, E, .) tensors)
    if (tid == 0) {
      const unsigned b_rp = (unsigned)((n + 1 + 7) / 8) * 16u, b_ord = (unsigned)(d.ord_rounds * NW) * 16u;
      const unsigned b_adj = (unsigned)((2 * e + 3) / 4) * 16u, b_k = VALUES ? 0u : (unsigned)((k + 3) / 4) * 16u;
      const unsigned b_x = (unsigned)n * (FS * 4u);
      fence_proxy_async();                     // the previous graph's ordinary accesses to these regions come first
      mbar_expect_tx(mbar, b_rp + b_ord + b_adj + 2u * b_k + b_x);
      bulk_g2s(rp_s, rp_g, b_rp, mbar);
      if (b_ord) bulk_g2s(smem + S_ORD, ord_g, b_ord, mbar);
      if (b_adj) bulk_g2s(adj_s, adj_g, b_adj, mbar);
      if (b_k) { bulk_g2s(cuv_s, cuv_g, b_k, mbar); bulk_g2s(cidx_s, cidx_g, b_k, mbar); }
      bulk_g2s(smem + S_EPQ, g.x, b_x, mbar);
    }
    g.rp = rp_s; g.adj = adj_s; g.cuv = cuv_s; g.cidx = cidx_s;
    g.ord = reinterpret_cast<const uint16_t*>(smem + S_ORD);
  }
  float* vn = smem + S_GPQ;          // value-head / numeric-encoder weights live in the idle GPQ region
  // per-graph vectors and scalars (numerical features, current-node features, action / return / ... of this sample):
  // one word per thread, LOADED before the weight staging and stored after it, so this round trip (DRAM-cold for the
  // per-sample arrays) overlaps the staging's instead of following it -- the slowest warp sets the barrier below
  const float* psrc = nullptr;
  float* pdst = nullptr;
  if (tid < NUMD) { psrc = gnum + tid; pdst = sV + V_X52 + tid; }
  else if (tid >= 64 && tid < 64 + FS) { psrc = gcur + (tid - 64); pdst = sV + V_XCUR + (tid - 64); }
  else if (tid >= 96 && tid < 109) pdst = sc + (tid - 96);                             // zeroed scalar slots
  else if (tid == 109) { if (a.actions) { psrc = a.actions + ((size_t)gid * 2 + g.stage); pdst = sc + SC_ACT; } }
  else if (tid == 114) pdst = sc + SC_QUEUE;                                           // candidate queue head = 0
  else if (TRAIN && tid == 110) { psrc = a.ret + gid; pdst = sc + SC_RET; }            // consumed by the softmax warp
  else if (TRAIN && tid == 111) { psrc = a.exps + gid; pdst = sc + SC_EXP; }
  else if (TRAIN && tid == 112) { psrc = a.fixed_lp + gid; pdst = sc + SC_FLP; }
  else if (TRAIN && tid == 113) { psrc = a.adv + gid; pdst = sc + SC_ADV; }
  else if (TRAIN && tid == 115) { if (a.old_values) psrc = a.old_values + gid; pdst = sc + SC_VOLD; }   // 0 when off
  else if (TRAIN && tid == 116) { if (a.prox_lp) { psrc = a.prox_lp + item; pdst = sc + SC_PLP; } }
  const float pval = psrc ? __ldg(psrc) : 0.f;
  stage_vn_weights(P, vn);
  if (pdst) *pdst = pval;
  if constexpr (!BIG) mbar_wait(mbar, mpar);
  __syncthreads();
  UPB_STAMP(1);

  // ================================================================================ forward
  numeric_l0(vn, sV + V_X52, sV + V_A0, tid);                        // numeric encoder, layer 0 (state_encoder.py:35-57)
  for (int i = tid; i < n; i += NT) g.inv[i] = 1.0f / ((float)(g.rp[i + 1] - g.rp[i]) + EPS_DEG);
  // h^0 = X We^T + be (state_encoder.py:189)
  if constexpr (BIG) {   // 4 lanes per node, 4 channels per lane, features from global memory
    for (int task = tid; task < n * 4; task += NT) {
      const int i = task >> 2;
      const float* xr = g.x + (size_t)i * FS;
      float4 xv[6];
#pragma unroll
      for (int f4i = 0; f4i < 6; ++f4i) xv[f4i] = __ldg(reinterpret_cast<const float4*>(xr) + f4i);
      float4 acc = ld4(sW + S_BE + q * 4);
#pragma unroll
      for (int f4i = 0; f4i < 6; ++f4i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float xs = comp(xv[f4i], j);
          const float4 w = ld4(sW + S_WET + (f4i * 4 + j) * 16 + q * 4);
          acc.x = fmaf(w.x, xs, acc.x); acc.y = fmaf(w.y, xs, acc.y);
          acc.z = fmaf(w.z, xs, acc.z); acc.w = fmaf(w.w, xs, acc.w);
        }
      }
      st4(g.H + i * 16 + q * 4, acc);
      if (TRAIN) st4(g.H0g + i * 16 + q * 4, acc);
    }
  } else {   // 8 lanes per node, 2 channels per lane: the lane's 24x2 weight slice stays in registers, features from
             // the staged rows (4 consecutive nodes per warp load: conflict-free), packed FMAs
    const int c2 = (lane & 7) * 2;
    float2 w[24];
#pragma unroll
    for (int f = 0; f < 24; ++f) w[f] = *reinterpret_cast<const float2*>(sW + S_WET + f * 16 + c2);
    const float2 be = *reinterpret_cast<const float2*>(sW + S_BE + c2);
    const float* xs = smem + S_EPQ;
    for (int i = warp * 4 + (lane >> 3); i < n; i += NW * 4) {
      const float4* xr = reinterpret_cast<const float4*>(xs + i * FS);
      float2 acc = be;
#pragma unroll
      for (int f4i = 0; f4i < 6; ++f4i) {
        const float4 xv = xr[f4i];
        acc = ffma2(w[f4i * 4 + 0], make_float2(xv.x, xv.x), acc);
        acc = ffma2(w[f4i * 4 + 1], make_float2(xv.y, xv.y), acc);
        acc = ffma2(w[f4i * 4 + 2], make_float2(xv.z, xv.z), acc);
        acc = ffma2(w[f4i * 4 + 3], make_float2(xv.w, xv.w), acc);
      }
      *reinterpret_cast<float2*>(g.H + i * 16 + c2) = acc;
      if (TRAIN) *reinterpret_cast<float2*>(g.H0g + i * 16 + c2) = acc;
    }
  }
  if (warp == NW - 1 && lane < 16) {   // current node through the same encoder (state_encoder.py:190-191)
    float s = sW[S_BE + lane];
#pragma unroll
    for (int f = 0; f < F; ++f) s = fmaf(sW[S_WET + f * 16 + lane], sV[V_XCUR + f], s);
    sV[V_HC + lane] = s;
  }
  __syncthreads();
  UPB_STAMP(2);
  if (warp == 0) numeric_l1(vn, sV + V_A0, sV + V_SV, lane);          // numeric encoder, layer 1 -> sv[0..15]
  if (!VALUES && g.stage == 0 && tid < 512) {
    // Weff = Wa + Wd + Wc diag(hc), ceff = b + (Wb - Wd) hc   (state_encoder.py:207-210 folded into the head)
    const int r = tid >> 4, c = tid & 15;
    const float* w = sW + S_LUW0 + r * 64;
    const float weff = w[c] + w[48 + c] + w[32 + c] * sV[V_HC + c];
    sV[V_WEFFT + c * 32 + r] = weff;
    sV[V_WEFF + r * 16 + c] = weff;
    if (tid < 32) {
      const float* wr = sW + S_LUW0 + tid * 64;
      float s = sW[S_LUB0 + tid];
#pragma unroll
      for (int cc = 0; cc < 16; ++cc) s = fmaf(wr[16 + cc] - wr[48 + cc], sV[V_HC + cc], s);
      sV[V_CEFF + tid] = s;
    }
  }

  // GCN layers (state_encoder.py:194-197): h <- h + (sum_{nbr} he) / (deg + eps), pull over the CSR
  int tier_last = 0, tier_first = 0;
  for (int l = 0; l < 2; ++l) {
    const float* WT = sW + (l == 0 ? S_WPQT0 : S_WPQT1);
    const float* bl = sW + (l == 0 ? S_B0 : S_B1);
    const int bad = epq_phase<false>(g, g.H, WT, bl);
    int tier = __syncthreads_or(bad) != 0;       // any pre-activation outside the one-reciprocal range?
    if (tier && __syncthreads_or(bad == 2)) {    // beyond exp2a's clamp: the same phase again, keeping raw values
      tier = 2;
      epq_phase<true>(g, g.H, WT, bl);
      __syncthreads();
    }
    UPB_STAMP(3+l*2);
    if (l == 1) tier_last = tier;
    else tier_first = tier;
    if (TRAIN && l == 0) {   // keep layer 0's EPQ for the backward pass (cheaper to reload than to recompute)
      for (int i = tid; i < n * 8; i += NT) __stcg(reinterpret_cast<float4*>(E0g) + i, ld4(g.EPQ + i * 4));
    }
    float4 msum = f4(0.f), hsum = f4(0.f);
    if (tier == 2) pull_forward<2, !BIG>(g, q, TRAIN && l == 0, g.H1g, l == 1, msum, hsum);
    else if (tier) pull_forward<1, !BIG>(g, q, TRAIN && l == 0, g.H1g, l == 1, msum, hsum);
    else pull_forward<0, !BIG>(g, q, TRAIN && l == 0, g.H1g, l == 1, msum, hsum);
    if (l == 1) {   // masked means (state_encoder.py:179-182,199-200); sum_j he_j = 1/2 sum_i acc_i
      block_sum_q8(msum, hsum, sRed, sV + V_TMP32);
      if (tid < 16) {
        sV[V_SV + 32 + tid] = (0.5f * sV[V_TMP32 + tid]) / (float)e;
        sV[V_SV + 16 + tid] = sV[V_TMP32 + 16 + tid] / (float)n;
      }
    } else {
      __syncthreads();
    }
    UPB_STAMP(4+l*2);
  }

  // attention of the current node over all nodes (state_encoder.py:150-161).  q' and Kc^T q'/4 are small enough
  // for every warp to compute for itself in registers (lane & 15 = component): no barriers, no smem round trip.
  float qk_c;
  {
    const int c = lane & 15;
    float qp = sW[S_QBC + c];
#pragma unroll
    for (int j = 0; j < 16; ++j) qp = fmaf(sW[S_QCT + j * 16 + c], sV[V_HC + j], qp);        // q'[c] = Qc[c][:] . hc
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) s = fmaf(sW[S_KC + r * 16 + c], __shfl_sync(0xffffffffu, qp, r), s);
    qk_c = 0.25f * s;     // 1/sqrt(head_dim)
    if (warp == 0 && lane < 16) { sV[V_QP + c] = qp; sV[V_QK + c] = qk_c; }
  }
  {
    const float4 qk4 = make_float4(__shfl_sync(0xffffffffu, qk_c, q * 4), __shfl_sync(0xffffffffu, qk_c, q * 4 + 1),
                                   __shfl_sync(0xffffffffu, qk_c, q * 4 + 2), __shfl_sync(0xffffffffu, qk_c, q * 4 + 3));
    float lmax = -CUDART_INF_F;
    for (int task = tid; task < ((n * 4 + 31) & ~31); task += NT) {
      const int i = task >> 2;
      float s = i < n ? dot4(qk4, ld4(g.H + i * 16 + q * 4)) : 0.f;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      if (i < n) {
        if (q == 0) g.alpha[i] = s;
        lmax = fmaxf(lmax, s);
      }
    }
    const float smax = block_max1(lmax, sRed);   // (alpha[i] is re-read below only by the warp that wrote it)
    float4 hb = f4(0.f);
    float asum = 0.f;
    for (int task = tid; task < ((n * 4 + 31) & ~31); task += NT) {
      const int i = task >> 2;
      const float ai = i < n ? expf(g.alpha[i] - smax) : 0.f;
      if (i < n) hb = hb + ld4(g.H + i * 16 + q * 4) * ai;
      __syncwarp();                               // all four lanes of the node have read the score
      if (i < n && q == 0) { g.alpha[i] = ai; asum += ai; }
    }
    block_sum_q4p1(hb, asum, sRed, sV + V_TMP32);   // -> [0..15] sum a_i h_i, [16] sum a_i
  }
  UPB_STAMP(7);

  // attention tail in every warp's registers; warp 0 publishes it
  {
    float hbar, vp, at;
    attention_tail(sW, sV + V_TMP32, lane, hbar, vp, at);
    if (warp == 0) {
      if (lane < 16) { sV[V_HBAR + lane] = hbar; sV[V_VP + lane] = vp; sV[V_SV + 48 + lane] = at; }
      if (lane < 3) sV[V_SV + 64 + lane] = (lane == g.stage) ? 1.f : 0.f;
      if (lane == 0) sc[SC_Z] = sV[V_TMP32 + 16];
    }
  }
  if (warp < 8) {
    group_bar(1, 256);                             // sv published by warp 0
    value_head_group(sV, vn, sc, tid);             // value head (value.py:15-39): warps 0..7
  }
  if constexpr (VALUES) {
    if (tid == 0) a.out_value[gid] = sc[SC_VALUE];    // the thread that wrote it
    return;
  }
  {   // policy head on the mask-true candidates (policy.py:45-65): half-warps pull candidates from a shared queue
    HeadLane hl;
    head_lane_init(hl, g, sW, sV, lane);
    int* queue = reinterpret_cast<int*>(sc) + SC_QUEUE;
    for (;;) {
      int j = 0;
      if ((lane & 15) == 0) j = atomicAdd(queue, 1);
      j = __shfl_sync(hl.mask, j, 0, 16);
      if (j >= k) break;
      float t0, t1, xin;
      head_units(hl, g, j, lane, tier_last == 2, t0, t1, xin);
      if (TRAIN && j < CH) {   // the backward pass starts from these instead of recomputing its first chunk (the buffers sit
                               // behind the value-head weights in the GPQ region, idle until the backward pulls)
        float* cGU = smem + S_GPQ + HB_GU;
        cGU[j * 32 + (lane & 15)] = t0;
        cGU[j * 32 + (lane & 15) + 16] = t1;
        smem[S_GPQ + HB_X + j * 16 + (lane & 15)] = xin;
      }
      const float zj = half_sum(hl.w20 * t0 + hl.w21 * t1, hl.mask);
      if ((lane & 15) == 0) g.z[j] = zj;
    }
  }
  __syncthreads();
  UPB_STAMP(9);
  // softmax / outputs / PPO seeds by warp NW-1; meanwhile (TRAIN) warps 0..7 run the value-head and numeric-encoder
  // backward, which only needs the value
  // (code order: the eight value-backward warps fall straight into their work; the softmax warp's 30 KB of code come
  // last, so only idle warps branch over them)
  if constexpr (TRAIN) {
    if (warp < 8) {
      const float gV = value_seed(a, sc[SC_VALUE], sc[SC_RET], sc[SC_VOLD]).g;
      value_numeric_bwd_group(sV, vn, gV, gp, tid);
    }
    if (tid >= 256 && tid < 272) sV[V_GHC + tid - 256] = 0.f;
  }
  if (warp == NW - 1) softmax_seeds<TRAIN>(a, hd, g, sc, TRAIN ? gp + G_STATS : nullptr, lane, item);
  if constexpr (!TRAIN) return;
  __syncthreads();
  UPB_STAMP(10);

  // ================================================================================ backward (SURVEY A.7)
  // ---- policy head backward, CH candidates at a time
  {
    float* cGU = smem + S_GPQ + HB_GU;        // [CH][32] g_u
    float* cX = smem + S_GPQ + HB_X;          // [CH][16] head input
    float* pGC = smem + S_GPQ + HB_PGC;       // [32][32] per-half-warp partial sums of g_u
    float* pGW2 = smem + S_GPQ + HB_PGW2;     // [32][32] per-half-warp partial sums of g_z t
    float G = 0.f, gcr = 0.f, gw2r = 0.f;     // thread (r = tid>>4, c = tid&15)
    const int r_ = (tid >> 4) & 31, c_ = tid & 15;
    const float* WR = g.stage == 0 ? sV + V_WEFF : sW + S_RDW0;     // [32][16] row-major
    int base = 0;
    do {
      const int cn = min(CH, k - base);
      {
        const int hw = warp * 2 + (lane >> 4), c16 = lane & 15;
        float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
        if (base == 0) {   // first chunk: hidden activations t and head inputs were left in cGU / cX by the forward pass
          const float* w2 = g.stage == 0 ? sW + S_LUW1 : sW + S_RDW1;
          const float w20 = w2[c16], w21 = w2[c16 + 16];
          for (int jj = hw; jj < cn; jj += 2 * NW) {
            const float t0 = cGU[jj * 32 + c16], t1 = cGU[jj * 32 + c16 + 16];
            const float gzj = g.gz[jj];
            const float gu0 = gzj * w20 * (1.f - t0 * t0), gu1 = gzj * w21 * (1.f - t1 * t1);
            cGU[jj * 32 + c16] = gu0;
            cGU[jj * 32 + c16 + 16] = gu1;
            a00 += gu0; a01 += gu1; a10 = fmaf(gzj, t0, a10); a11 = fmaf(gzj, t1, a11);
          }
        } else {           // later chunks: recompute the candidates' hidden units
          HeadLane hl;
          head_lane_init(hl, g, sW, sV, lane);
          for (int jj = hw; jj < cn; jj += 2 * NW) {
            float t0, t1, xin;
            head_units(hl, g, base + jj, lane, tier_last == 2, t0, t1, xin);
            const float gzj = g.gz[base + jj];
            const float gu0 = gzj * hl.w20 * (1.f - t0 * t0), gu1 = gzj * hl.w21 * (1.f - t1 * t1);
            cGU[jj * 32 + c16] = gu0;
            cGU[jj * 32 + c16 + 16] = gu1;
            cX[jj * 16 + c16] = xin;
            a00 += gu0; a01 += gu1; a10 = fmaf(gzj, t0, a10); a11 = fmaf(gzj, t1, a11);
          }
        }
        pGC[hw * 32 + c16] = a00; pGC[hw * 32 + c16 + 16] = a01;
        pGW2[hw * 32 + c16] = a10; pGW2[hw * 32 + c16 + 16] = a11;
      }
      __syncthreads();
      UPB_STAMP(12);
      if (tid < 512) {
        float g0 = 0.f, g1 = 0.f;
        int jj = 0;
        for (; jj + 1 < cn; jj += 2) {
          g0 = fmaf(cGU[jj * 32 + r_], cX[jj * 16 + c_], g0);
          g1 = fmaf(cGU[(jj + 1) * 32 + r_], cX[(jj + 1) * 16 + c_], g1);
        }
        if (jj < cn) g0 = fmaf(cGU[jj * 32 + r_], cX[jj * 16 + c_], g0);
        G += g0 + g1;
        if (tid < 64) {       // sums over the 32 half-warps: tid < 32 -> g_c[tid], 32..63 -> g_w2[tid-32]
          const float* src = tid < 32 ? pGC + tid : pGW2 + (tid - 32);
          float sacc = 0.f;
#pragma unroll 8
          for (int h = 0; h < 32; ++h) sacc += src[h * 32];
          if (tid < 32) gcr += sacc; else gw2r += sacc;
        }
      }
      for (int task = tid; task < cn * 16; task += NT) {   // g_x = W^T g_u
        const int jj = task >> 4, c = task & 15;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
        for (int r = 0; r < 32; r += 2) {
          s0 = fmaf(WR[r * 16 + c], cGU[jj * 32 + r], s0);
          s1 = fmaf(WR[(r + 1) * 16 + c], cGU[jj * 32 + r + 1], s1);
        }
        g.ghead[(size_t)(base + jj) * 16 + c] = s0 + s1;
      }
      base += CH;
      if (base < k) __syncthreads();               // chunk buffers are reused
    } while (base < k);
    if (tid < 512) sV[V_GWEFF + tid] = G;
    if (tid < 32) sV[V_GC + tid] = gcr;
    if (tid >= 32 && tid < 64) sV[V_GW2 + tid - 32] = gw2r;
  }
  // ---- attention backward.  g_v' = Wo^T g_att and g_hbar = Vc^T g_v' per warp in registers (lane & 15 = component).
  // Runs BEFORE the barrier that closes the head backward: it needs nothing from it (value-path gradients, alpha and
  // h^L only; every head-backward read of h^L lies before that loop's last internal barrier), so its dependent chains
  // and the node loop overlap the other warps' last head-backward chunk instead of following the barrier.
  float gvp_c, ghbar_c;
  float4 gsh = f4(0.f);
  {
    const int c = lane & 15;
    const float gatt = sV[V_GSV + 48 + c];
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) s = fmaf(sW[S_WO + r * 16 + c], __shfl_sync(0xffffffffu, gatt, r), s);
    gvp_c = s;
    s = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) s = fmaf(sW[S_VC + r * 16 + c], __shfl_sync(0xffffffffu, gvp_c, r), s);
    ghbar_c = s;
    if (warp == 0 && lane < 16) {
      sV[V_GVP + c] = gvp_c;
      sV[V_CE + c] = e > 0 ? sV[V_GSV + 32 + c] / (float)e : 0.f;
    }
  }
  {
    const float4 gh4 = make_float4(__shfl_sync(0xffffffffu, ghbar_c, q * 4), __shfl_sync(0xffffffffu, ghbar_c, q * 4 + 1),
                                   __shfl_sync(0xffffffffu, ghbar_c, q * 4 + 2), __shfl_sync(0xffffffffu, ghbar_c, q * 4 + 3));
    // g_hbar . hbar in exactly the arithmetic of each node's dp below: in a peaked softmax hbar is h_max bit for bit
    // and dp - gdot must be exactly 0 there (another summation order leaves an ulp, which large keys amplify)
    float gdot = dot4(gh4, ld4(sV + V_HBAR + q * 4));
    gdot += __shfl_xor_sync(0xffffffffu, gdot, 1);
    gdot += __shfl_xor_sync(0xffffffffu, gdot, 2);
    const float4 qk4 = make_float4(__shfl_sync(0xffffffffu, qk_c, q * 4), __shfl_sync(0xffffffffu, qk_c, q * 4 + 1),
                                   __shfl_sync(0xffffffffu, qk_c, q * 4 + 2), __shfl_sync(0xffffffffu, qk_c, q * 4 + 3));
    const float4 gmn4 = ld4(sV + V_GSV + 16 + q * 4) * (1.f / (float)n);
    const float invZ = 1.f / sc[SC_Z];
    for (int task = tid; task < ((n * 4 + 31) & ~31); task += NT) {
      const int i = task >> 2;
      const float4 h = i < n ? ld4(g.H + i * 16 + q * 4) : f4(0.f);
      float dp = dot4(gh4, h);
      dp += __shfl_xor_sync(0xffffffffu, dp, 1);
      dp += __shfl_xor_sync(0xffffffffu, dp, 2);
      if (i < n) {
        const float ai = g.alpha[i] * invZ;
        const float gs = ai * (dp - gdot);
        gsh = gsh + h * gs;
        // g_h^L = g_mean/n + a_i g_hbar (value path) + g_s qk (key path); stored scaled by 1/(deg+eps), over h^L
        st4(g.H + i * 16 + q * 4, (gmn4 + gh4 * ai + qk4 * gs) * g.inv[i]);
      }
    }
  }
  __syncthreads();
  UPB_STAMP(13);
  if (g.stage == 0) {
    if (tid < 512) {
      const int r_ = tid >> 4, c_ = tid & 15;
      const float G = sV[V_GWEFF + tid], hc = sV[V_HC + c_], gc = sV[V_GC + r_];
      const int o = P_LU_W0 + r_ * 64 + c_;
      gacc(gp, o, G);
      gacc(gp, o + 16, gc * hc);
      gacc(gp, o + 32, G * hc);
      gacc(gp, o + 48, G - gc * hc);
    }
    if (tid < 32) { gacc(gp, P_LU_B0 + tid, sV[V_GC + tid]); gacc(gp, P_LU_W1 + tid, sV[V_GW2 + tid]); }
    if (warp == 1) {   // d/d hc through ceff and through Wc diag(hc): 16 components x 2 halves of the 32 units
      const int c = lane & 15, r0 = (lane >> 4) * 16;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        const float* w = sW + S_LUW0 + (r0 + r) * 64;
        s0 = fmaf(w[16 + c] - w[48 + c], sV[V_GC + r0 + r], s0);
        s1 = fmaf(w[32 + c], sV[V_GWEFF + (r0 + r) * 16 + c], s1);
      }
      float s = s0 + s1;
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      if (lane < 16) sV[V_GHC + c] = s;
    }
  } else {
    if (tid < 512) gacc(gp, P_RD_W0 + tid, sV[V_GWEFF + tid]);
    if (tid < 32) { gacc(gp, P_RD_B0 + tid, sV[V_GC + tid]); gacc(gp, P_RD_W1 + tid, sV[V_GW2 + tid]); }
  }

  block_sum_q4(gsh, sRed, sV + V_GSH);
  if (warp == 0) {   // g_q' = Kc gsh / 4, g_hc += Qc^T g_q', composed-projection gradients
    const int c = lane & 15;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) s = fmaf(sW[S_KCT + j * 16 + c], sV[V_GSH + j], s);
    const float gqp = 0.25f * s;
    float t = sV[V_GHC + c];
#pragma unroll
    for (int r = 0; r < 16; ++r) t = fmaf(sW[S_QC + r * 16 + c], __shfl_sync(0xffffffffu, gqp, r), t);
    __syncwarp();                                  // lanes c and c + 16 both read V_GHC[c] above (racecheck)
    if (lane < 16) { sV[V_GHC + c] = t; sV[V_GQP + c] = gqp; }
  }
  if (g.stage == 1) {   // road head feeds h^L of its candidate nodes directly
    for (int task = tid; task < k * 16; task += NT) {
      const int j = task >> 4, c = task & 15;
      const int node = (int)g.cuv[j];
      g.H[node * 16 + c] += g.ghead[(size_t)j * 16 + c] * g.inv[node];
    }
  }
  __syncthreads();
  UPB_STAMP(14);
  if (tid < 256) {   // composed-projection ("virtual") gradients, chained to the real tensors in k_reduce_finish
    const int r = tid >> 4, cc = tid & 15;
    gacc(gp, G_QC + tid, sV[V_GQP + r] * sV[V_HC + cc]);
    gacc(gp, G_KC + tid, 0.25f * sV[V_QP + r] * sV[V_GSH + cc]);
    gacc(gp, G_VC + tid, sV[V_GVP + r] * sV[V_HBAR + cc]);
    gacc(gp, P_MHA_OUT_W + tid, sV[V_GSV + 48 + r] * sV[V_VP + cc]);
  } else if (tid < 272) {
    const int c = tid - 256;
    gacc(gp, G_QBC + c, sV[V_GQP + c]);
    gacc(gp, G_VBC + c, sV[V_GVP + c]);
    gacc(gp, P_MHA_OUT_B + c, sV[V_GSV + 48 + c]);
  }

  // ---- GCN layers, last to first
  for (int l = 1; l >= 0; --l) {
    const float* Wpq = sW + (l == 0 ? S_WPQ0 : S_WPQ1);
    const float* hin = l == 0 ? g.H0g : g.H1g;     // layer input h^l (global scratch)
    int tier = tier_last;
    if (l == 0) {   // EPQ of layer 0 was overwritten by layer 1: reload the copy saved by the forward pass
      if constexpr (BIG) {
#pragma unroll 2
        for (int i = tid; i < n * 8; i += NT) st4(g.EPQ + i * 4, __ldcg(reinterpret_cast<const float4*>(E0g) + i));
      } else {   // one bulk copy; the forward pass's __stcg stores to E0g were ordered by the barriers since
        if (tid == 0) {
          fence_proxy_async();
          mbar_expect_tx(mbar + 1, (unsigned)n * 128u);
          bulk_g2s(g.EPQ, E0g, (unsigned)n * 128u, mbar + 1);
        }
        mbar_wait(mbar + 1, mpar);
      }
      tier = tier_first;
      __syncthreads();
      UPB_STAMP(17);
    }
    const bool last = (l == 1);
    const float4 ce4 = last ? ld4(sV + V_CE + q * 4) : f4(0.f);
    const bool use_head = last && g.stage == 0;
    // (the backward pull keeps compiler-generated addressing)
    const float4 bsum = tier == 2 ? pull_backward<2, false>(g, q, ce4, use_head)
                        : tier ? pull_backward<1, false>(g, q, ce4, use_head) : pull_backward<0, false>(g, q, ce4, use_head);
    block_sum_q4(bsum, sRed, sV + V_TMP16);     // barriers inside: GPQ complete, EPQ dead
    UPB_STAMP(15+(1-l)*3);
    // layer input h^l back from the global scratch into the dead EPQ region, behind the reduction buffer: one bulk
    // copy, in flight while the tensor-core g_h phase runs, so g_W's K loop reads h rows at shared-memory latency
    bool hin_smem = false;
    if constexpr (!BIG) {
      hin_smem = n <= HIN_NODES;
      if (tid == 0) {
        fence_proxy_async();
        if (hin_smem) {
          mbar_expect_tx(mbar + 3, (unsigned)n * 64u);
          bulk_g2s(smem + S_EPQ + KW * 512, hin, (unsigned)n * 64u, mbar + 3);
        }
        // after the last pull the candidate / pull-schedule / adjacency lists are dead: the node features the encoder backward
        // needs come back into that stretch now, two phases ahead of their use
        if (l == 0 && n <= XEARLY_NODES) {
          mbar_expect_tx(mbar + 2, (unsigned)n * (FS * 4u));
          bulk_g2s(smem + S_Z, g.x, (unsigned)n * (FS * 4u), mbar + 2);
        }
      }
    }
    if (tid < 16) gacc(gp, (l == 0 ? P_GCN0_B : P_GCN1_B) + tid, sV[V_TMP16 + tid]);
    gh_phase_tc(g, Wpq, l == 1);     // g_h = g_h' + GPQ Wpq (residual), in place
    if (hin_smem) mbar_wait(mbar + 3, l == 1 ? 0u : 1u);     // two phases per graph: parity 0 then 1
    if (warp < KW) {   // g_W[o][c] = sum_i GPQ[i][o] h^l[i][c]: tensor-core tiles, K split over KW warps
      if (hin_smem) gw_partial<true>(g, smem + S_EPQ + KW * 512, n, smem + S_EPQ);
      else gw_partial<false>(g, hin, n, smem + S_EPQ);
    }
    __syncthreads();
    if (tid < 512) {
      const float* redbuf = smem + S_EPQ;
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < KW; ++w) s += redbuf[w * 512 + tid];
      const int o = tid >> 4, c = tid & 15;
      const int dst = o < 16 ? o * 32 + c : (o - 16) * 32 + 16 + c;
      gacc(gp, (l == 0 ? P_GCN0_W : P_GCN1_W) + dst, s);
    }
    __syncthreads();
    UPB_STAMP(16+(1-l)*3);
  }

  // ---- node encoder backward: g_We = g_h0^T X + g_hc x_cur^T, g_be = sum g_h0 + g_hc
  {
    float* redbuf = smem + S_GPQ;                // [NW][384]  (GPQ is dead after the last g_h)
    const float* xsrc = g.x;
    if constexpr (!BIG) {                        // features: already on their way into the dead list stretch (above), or,
      if (n <= XEARLY_NODES) {                   // for graphs too large for it, into the dead EPQ region now
        xsrc = smem + S_Z;
      } else {
        if (tid == 0) {
          fence_proxy_async();
          mbar_expect_tx(mbar + 2, (unsigned)n * (FS * 4u));
          bulk_g2s(smem + S_EPQ, g.x, (unsigned)n * (FS * 4u), mbar + 2);
        }
        xsrc = smem + S_EPQ;
      }
    }
    float4 hs = f4(0.f);
    for (int task = tid; task < n * 4; task += NT) hs = hs + ld4(g.H + (task >> 2) * 16 + q * 4);
    if constexpr (!BIG) { mbar_wait(mbar + 2, mpar); __syncthreads(); }
    // partial g_We of this warp on the tensor cores: A = g_h0^T (16 x K: one m-tile) times B = X (K x 24: three n-tiles),
    // 3xTF32 (mma_3x), k-steps of 8 consecutive nodes as in gw_partial.  A row 8 j + g is channel c = 2 g + j (one
    // 64-bit load of g_h0[node][2g, 2g+1]); B keeps feature order and is loaded by scalars: the four nodes of a tile
    // column sit 24 floats apart, banks 0, 24, 16, 8 (mod 32) from each other, so a warp's 8 x 4 loads hit 32 banks.
    {
      const int gq = lane >> 2, t = lane & 3;
      float acc[3][4];   // [n-tile][fragment]: c = 2 gq + (q >> 1), f = 8 nt + 2 t + (q & 1)
#pragma unroll
      for (int nt = 0; nt < 3; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[nt][q] = 0.f;
      for (int kc = warp; kc * 8 < n; kc += 2 * NW) {   // two k-steps per trip
        float2 ha[2][2];    // [k-step][tile column t, t + 4]
        float xb[2][2][3];  // [k-step][tile row t, t + 4][n-tile]
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int s = 0; s < 2; ++s) {
            const int i = (kc + u * NW) * 8 + s * 4 + t;
            const bool ok = i < n;
            ha[u][s] = ok ? *reinterpret_cast<const float2*>(g.H + i * 16 + 2 * gq) : make_float2(0.f, 0.f);
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
              if constexpr (BIG) xb[u][s][nt] = ok ? __ldg(xsrc + (size_t)i * FS + nt * 8 + gq) : 0.f;
              else xb[u][s][nt] = ok ? xsrc[i * FS + nt * 8 + gq] : 0.f;
            }
          }
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int nt = 0; nt < 3; ++nt) {
            uint32_t bh0, bl0, bh1, bl1;
            tf32_split(xb[u][0][nt], bh0, bl0);
            tf32_split(xb[u][1][nt], bh1, bl1);
            mma_3x(acc[nt], ha[u][0].x, ha[u][0].y, ha[u][1].x, ha[u][1].y, bh0, bh1, bl0, bl1);
          }
      }
#pragma unroll
      for (int nt = 0; nt < 3; ++nt) {
        *reinterpret_cast<float2*>(redbuf + warp * 384 + (2 * gq) * 24 + nt * 8 + 2 * t) = make_float2(acc[nt][0], acc[nt][1]);
        *reinterpret_cast<float2*>(redbuf + warp * 384 + (2 * gq + 1) * 24 + nt * 8 + 2 * t) = make_float2(acc[nt][2], acc[nt][3]);
      }
    }
    block_sum_q4(hs, sRed, sV + V_TMP16);        // barriers inside publish redbuf
    if (tid < 384) {
      const int c = tid / 24, f = tid % 24;
      if (f < F) {
        float s = sV[V_GHC + c] * sV[V_XCUR + f];
#pragma unroll
        for (int w = 0; w < NW; ++w) s += redbuf[w * 384 + tid];
        gacc(gp, P_ENC_W + c * F + f, s);
      }
    }
    if (tid < 16) gacc(gp, P_ENC_B + tid, sV[V_TMP16 + tid] + sV[V_GHC + tid]);
  }
  __syncthreads();
  UPB_STAMP(21);
}


// ---- fused tail: gradient reduction, (cross-GPU) exchange, attention chain, Adam (see upb_ppo_step) ----------------------
// One code path for one GPU and for data-parallel ranks (one process per GPU, peers opened with CUDA IPC over NVLink /
// NVSwitch).  The flat gradient row is cut into NSLICE slices of 128 columns; slice s is owned by CTA s % gridDim.x of
// every rank.
//   grid barrier (local)  : all graphs of all CTAs are done, the per-CTA partial rows are complete
//   PUSH                  : the owner sums its slice over the local CTAs (fixed order) and STORES the 128 sums into
//                           region [parity][src = this rank] of EVERY rank's exchange buffer (remote stores over NVLink,
//                           fire and forget), then releases one flag per (destination rank, slice) carrying the step
//                           sequence number and this rank's stage bits
//   REDUCE + ADAM         : the owner polls the flags of ITS slice in its own (local) buffer until every rank has
//                           delivered, adds the world contributions in rank order (local loads) and applies Adam to its
//                           columns -- no second grid barrier, no serial publish, no remote loads, and a slice proceeds as
//                           soon as it alone has arrived
//   ATTENTION CHAIN       : the last CTA waits for the seven slices that hold the 816 "virtual" gradients of the composed
//                           attention projections, chains them to the six real tensors and applies their Adam.
// Same summation order on every rank -> bit-identical parameters everywhere without a broadcast.  Regions and flags are
// double-buffered by step parity: a rank can be at most one step ahead of the slowest one (it needs that rank's flags of
// the current step before its kernel can finish), so parity p is never rewritten while it is being read.
constexpr int MAX_PEERS = 16;
constexpr int NSLICE = SgnnRow::nslice;          // 114
static_assert(G_ROW % SLICE == 0, "slices tile the gradient row");
constexpr int CHAIN_S0 = G_QC / SLICE;           // first / last slice holding virtual attention gradients
constexpr int CHAIN_S1 = (G_STATS - 1) / SLICE;
constexpr int FLAG_STRIDE = 128;                 // flag words per (parity, source rank)
constexpr size_t XCHG_FLAGS = (size_t)2 * MAX_PEERS * G_ROW;                       // float offset of the flag words
// rank-local words of the global clip (tail_gclip): float64 partials [2 parities][FLAG_STRIDE], then u32 flags
// [2][FLAG_STRIDE] = (sequence << 1) | 1 if the publishing CTA gave up on a peer
constexpr size_t XCHG_GCLIP = XCHG_FLAGS + (size_t)2 * MAX_PEERS * FLAG_STRIDE;
constexpr size_t XCHG_GCLIP_FLAGS = XCHG_GCLIP + (size_t)2 * 2 * FLAG_STRIDE;
constexpr size_t XCHG_FLOATS = XCHG_GCLIP_FLAGS + (size_t)2 * FLAG_STRIDE;              // whole buffer
static_assert(XCHG_GCLIP % 2 == 0, "float64 partials are 8-byte aligned");
static_assert(NSLICE + 1 <= FLAG_STRIDE, "one flag word per slice, one for the global clip's chain partial");
static_assert(NSLICE == 114 && CHAIN_S0 == 107 && CHAIN_S1 == 113,
              "tests/test_gpu_shapes.py runs the fused tail at grids of 113 / 114 / 115 CTAs around NSLICE: move them");
constexpr unsigned PEER_SPIN_LIMIT = 1u << 24;   // polls before a CTA gives up on a peer (seconds): the step's Adam update
                                                 // is then SKIPPED by that CTA and the sticky counter gridbar[6] is bumped

__device__ __forceinline__ float ld_relaxed(const float* p, bool sys) {
  float v;
  if (sys) asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
  else asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_relaxed(float* p, float v, bool sys) {
  if (sys) asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
  else asm volatile("st.relaxed.gpu.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p, bool sys) {
  unsigned v;
  if (sys) asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  else asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v, bool sys) {
  if (sys) asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  else asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ void grid_arrive(unsigned int* ctr) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
  }
}
// the counter is never reset: the host passes the cumulative arrival count this launch ends at (wrap-safe compare)
__device__ __forceinline__ void grid_wait(unsigned int* ctr, unsigned int target) {
  if (threadIdx.x == 0) {
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    } while ((int)(v - target) < 0);
    __threadfence();
  }
  __syncthreads();
}

// torch.optim.Adam on one element with torch's operation order (same arithmetic as k_apply; no clipping here).
// m, v, p are the element's current moments / value (loaded early by the caller so the latency overlaps); p must be
// the value from before this step's update, because the weight-decay term is taken from it.
__device__ __forceinline__ void adam_elem(const StepArgs& a, int i, float g, float m, float v, float p, float step_size,
                                          float bc2_sqrt) {
  const float w1 = 1.f - a.beta1, w2 = 1.f - a.beta2;
  if (a.weight_decay != 0.f) g = __fmaf_rn(a.weight_decay, p, g);     // grad.add(param, alpha=weight_decay), as k_apply
  m = __fadd_rn(m, __fmul_rn(w1, __fsub_rn(g, m)));
  v = __fadd_rn(__fmul_rn(v, a.beta2), __fmul_rn(__fmul_rn(w2, g), g));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), a.adam_eps);
  p = __fadd_rn(p, __fmul_rn(-step_size, __fdiv_rn(m, denom)));
  a.params_rw[i] = p;
  a.adam_m[i] = m;
  a.adam_v[i] = v;
  if (a.prox_params != nullptr) prox_ewma_elem(a.prox_params, a.prox_beta, i, p);
}
// The EWMA of an element a step that applied Adam leaves unchanged (its head absent, its tensor frozen): theta_prox
// converges to it
__device__ __forceinline__ void prox_keep(const StepArgs& a, int i) {
  if (a.prox_params != nullptr) prox_ewma_elem(a.prox_params, a.prox_beta, i, a.params_rw[i]);
}

// ---- parameter groups in the fused tails (a.pg != NULL; k_sgnn_pg / k_mlp_pg).  Before the grid barrier every CTA stages
// each tensor's Adam values in free dynamic shared memory, pgs = float[4][PG_MAX_TENSORS]: the step size
// (float)(lr / bias_correction1) and sqrt(bias_correction2) at the tensor's count + 1 (k_apply's arithmetic: with every
// tensor trained at the context's lr, the per-segment values bit for bit), its decoupled factor pg->decay (row 2; the
// KL-adaptive lr re-forms rows 0 and 2 in tail_kl_gate) and its trained flag (row 3).  The bias corrections take the
// tensor's own betas; its other Adam settings are read from the table by pg_adam_step.
__device__ __forceinline__ void pg_stage(const StepArgs& a, float* pgs) {
  const int t = threadIdx.x;
  if (t < a.pg->n) {
    const long long stp = a.tsteps_in[t] + 1;
    const double bc1 = 1.0 - ipow((double)a.pg->beta1[t], stp);
    const double bc2 = 1.0 - ipow((double)a.pg->beta2[t], stp);
    pgs[t] = (float)(a.pg->lr[t] / bc1);
    pgs[PG_MAX_TENSORS + t] = (float)sqrt(bc2);
    pgs[2 * PG_MAX_TENSORS + t] = a.pg->decay[t];
    pgs[3 * PG_MAX_TENSORS + t] = a.pg->trained[t] ? 1.f : 0.f;
  }
}
__device__ __forceinline__ bool pg_trained(const StepArgs& a, const float* pgs, int col) {
  return pgs[3 * PG_MAX_TENSORS + a.pg->tensor_of[col]] != 0.f;
}
// Adam on column col with its tensor's values; nothing for a frozen tensor
__device__ __forceinline__ void pg_adam_elem(const StepArgs& a, const float* pgs, int col, float g) {
  const int k = a.pg->tensor_of[col];
  if (pgs[3 * PG_MAX_TENSORS + k] == 0.f) {
    prox_keep(a, col);
    return;
  }
  const float p = pg_adam_step(a.pg, k, col, g, pgs[k], pgs[PG_MAX_TENSORS + k], pgs[2 * PG_MAX_TENSORS + k],
                               a.params_rw, a.adam_m, a.adam_v);
  if (a.prox_params != nullptr) prox_ewma_elem(a.prox_params, a.prox_beta, col, p);
}

// ---- the exchange protocol both fused tails (fused_tail here, mlp_fused_tail in mlp_kernel.cuh) run on their row
// layout L; only the local column sums, the attention chain and which CTA writes the step counters differ.
struct TailShared {
  float adam[12];                 // [seg][live ? 1 : 0][step_size, sqrt(bc2)]
  long long steps[6];
  unsigned bits;                  // OR of the ranks' stage bits (carried by the flags)
  int timeout;
  int stop;                       // no Adam, counters unchanged: this step passes the KL criterion (tail_kl_gate) or,
                                  // once tail_gclip has decided, is not finite (upb_set_nonfinite_guard)
  int lr_dec;                     // the KL-adaptive lr's decision (tail_kl_gate; 0 on a stopping step)
  float* push[MAX_PEERS];         // region [par][src = me] of every rank's buffer
};

// Before the grid barrier: push pointers, this CTA's stage bits into the launch's word (which policy heads its graphs
// used), the NEXT launch's word cleared (the previous launch, which used it, has completed), and the Adam bias
// corrections of the three segments for "head live" and "head skipped" (as k_apply).
__device__ __forceinline__ void tail_prologue(const StepArgs& a, TailShared& sh, unsigned stage_bits) {
  const int tid = threadIdx.x;
  const unsigned par = a.seq & 1u;
  if (tid < a.world) sh.push[tid] = a.peers[tid] + ((size_t)par * MAX_PEERS + a.rank) * G_ROW;
  if (tid == 32) { sh.timeout = 0; sh.bits = 0u; sh.stop = 0; }
  if (tid == 0 && stage_bits) atomicOr(a.gridbar + 2 + par, stage_bits);
  if (tid == 1 && blockIdx.x == 0) a.gridbar[2 + (par ^ 1u)] = 0u;
  if (tid < 6) {
    const int seg = tid >> 1, live = tid & 1;
    const long long stp = a.steps_in[1 + seg] + live;
    const double bc1 = 1.0 - ipow((double)a.beta1, stp > 0 ? stp : 1);
    const double bc2 = 1.0 - ipow((double)a.beta2, stp > 0 ? stp : 1);
    sh.adam[tid * 2 + 0] = (float)(a.lr / bc1);
    sh.adam[tid * 2 + 1] = (float)sqrt(bc2);
    sh.steps[tid] = stp;
  }
}

// The grid barrier (all graphs of all CTAs are done, the gpart rows are complete); returns the flag word of this
// rank's slices: the step sequence and the stage bits of all its CTAs.
__device__ __forceinline__ unsigned tail_barrier(const StepArgs& a) {
  grid_arrive(a.gridbar);
  grid_wait(a.gridbar, a.bar_target);
  unsigned mybits;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(mybits) : "l"(a.gridbar + 2 + (a.seq & 1u)) : "memory");
  return (a.seq << 2) | (mybits & 3u);
}

// After this CTA's pushes: one released flag per (destination rank, owned slice)
template <class L>
__device__ __forceinline__ void tail_release(const StepArgs& a, unsigned flagword, int nthreads, bool sys) {
  __syncthreads();                // this CTA's pushes are issued (ordered before the releases below)
  const unsigned par = a.seq & 1u;
  const int nown = (L::nslice - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  for (int idx = threadIdx.x; idx < a.world * nown; idx += nthreads) {
    const int r = idx % a.world, sl = blockIdx.x + (idx / a.world) * gridDim.x;
    unsigned* f = reinterpret_cast<unsigned*>(a.peers[r] + XCHG_FLAGS) + ((size_t)par * MAX_PEERS + a.rank) * FLAG_STRIDE + sl;
    if (sys) __threadfence_system(); else __threadfence();
    st_release(f, flagword, sys);
  }
}

// Waits until rank r has delivered slice sl (or gives up after PEER_SPIN_LIMIT polls: sh.timeout) and collects its
// stage bits
__device__ __forceinline__ void tail_poll(const StepArgs& a, TailShared& sh, const unsigned* myflags, int r, int sl,
                                          bool sys) {
  unsigned polls = 0, f;
  while ((int)(((f = ld_acquire(myflags + (size_t)r * FLAG_STRIDE + sl, sys)) >> 2) - a.seq) < 0) {
    if (++polls >= PEER_SPIN_LIMIT) { sh.timeout = 1; break; }
  }
  if (f & 3u) atomicOr(&sh.bits, f & 3u);
}

// every rank's contribution to column col, added in rank order (identical on every rank)
__device__ __forceinline__ float rank_sum(const float* pull, int world, int col, bool sys) {
  float v[MAX_PEERS];
#pragma unroll
  for (int p = 0; p < MAX_PEERS; ++p) v[p] = p < world ? ld_relaxed(pull + (size_t)p * G_ROW + col, sys) : 0.f;
  float s = v[0];
#pragma unroll
  for (int p = 1; p < MAX_PEERS; ++p) if (p < world) s += v[p];
  return s;
}

// REDUCE + ADAM of the owned slices: every rank's contribution to column sl * SLICE + c (rank_sum), written by
// write_grad_col, and a parameter's Adam step unless its policy head is not live or a peer timed out.  Threads with
// `active` own a column; col0 is the column of the first owned slice, whose moments and parameter the caller loaded
// into pm, pv, pp before the grid barrier.
template <class L>
__device__ __forceinline__ void tail_reduce_adam(const StepArgs& a, TailShared& sh, const float* pull,
                                                 const unsigned* myflags, bool sys, int c, bool active, int col0,
                                                 float pm, float pv, float pp) {
  const int world = a.world;
  for (int sl = blockIdx.x; sl < L::nslice; sl += gridDim.x) {
    if ((int)threadIdx.x < world) tail_poll(a, sh, myflags, threadIdx.x, sl, sys);
    __syncthreads();
    const bool live_lu = sh.bits & 1u, live_rd = sh.bits & 2u;
    const bool dead = sh.timeout != 0 || sh.stop;
    const int col = sl * SLICE + c;
    if (active && (L::row % SLICE == 0 || col < L::row)) {
      const float s = rank_sum(pull, world, col, sys);
      if (write_grad_col<L>(a.grad_out, col, s)) {
        int seg = 0;
        bool live = true;
        if (col >= L::lu_begin && col < L::rd_begin) { seg = 1; live = live_lu; }
        else if (col >= L::rd_begin && col < L::policy_end) { seg = 2; live = live_rd; }
        if (live && !dead) {
          if (col != col0) { pm = a.adam_m[col]; pv = a.adam_v[col]; pp = a.params_rw[col]; }    // later slices (small grids)
          adam_elem(a, col, s, pm, pv, pp, sh.adam[(seg * 2 + 1) * 2], sh.adam[(seg * 2 + 1) * 2 + 1]);
        } else if (!dead) {
          prox_keep(a, col);
        }
      } else if (sh.stop && col == L::stats + KL_STOP_SLOT) {     // after write_grad_col's zero, same thread
        a.grad_out[L::stat_offset + KL_STOP_SLOT] = 1.f;
        *a.kl_stop = 1u;
      }
    }
    __syncthreads();              // sh.bits / sh.timeout are read before the next slice's polls
  }
}

// step counters ([0] global, [1] encoder+value, [2] land-use head, [3] road head), thread tid < 4 of the CTA whose
// flags carried the stage bits of every rank; unchanged when a peer timed out or the step stops on the KL criterion
__device__ __forceinline__ void tail_write_steps(const StepArgs& a, const TailShared& sh) {
  const int tid = threadIdx.x;
  const bool live_lu = sh.bits & 1u, live_rd = sh.bits & 2u;
  if (sh.timeout == 0 && !sh.stop)
    a.steps_out[tid] = tid == 0 ? a.steps_in[0] + 1
                                : sh.steps[(tid - 1) * 2 + (tid == 1 ? 1 : (tid == 2 ? (live_lu ? 1 : 0) : (live_rd ? 1 : 0)))];
  else
    a.steps_out[tid] = a.steps_in[tid];
}

// per-tensor counts (parameter groups), thread tid < a.pg->n of the CTA that calls tail_write_steps: a tensor's count
// advances when the step applied Adam, the tensor is trained and its segment is live
__device__ __forceinline__ void tail_write_tensor_steps(const StepArgs& a, const TailShared& sh) {
  const int t = threadIdx.x;
  const int s = a.pg->seg[t];
  const bool seg_live = s == 0 || (s == 1 ? (sh.bits & 1u) != 0 : (sh.bits & 2u) != 0);
  const bool step = sh.timeout == 0 && !sh.stop && a.pg->trained[t] && seg_live;
  a.tsteps_out[t] = a.tsteps_in[t] + (step ? 1 : 0);
}

// the sticky peer-timeout count (upb_peer_timeouts)
__device__ __forceinline__ void tail_count_timeout(const StepArgs& a, const TailShared& sh) {
  if (threadIdx.x == 0 && sh.timeout) atomicAdd(a.gridbar + 6, 1u);
}

// KL stop and KL-adaptive lr (a.kl_stop != NULL, which the host also passes for the adaptive lr alone), after this CTA's
// pushes and before its first Adam write: every CTA waits for the statistics slice of every rank and sums slots 4 and 8
// in rank order, as the slice's owner does in tail_reduce_adam, so all CTAs (and all ranks) take the same decisions,
// sh.stop and then sh.lr_dec, from the values written to the gradient buffer.  With the adaptive lr on, every CTA then
// replaces the step sizes tail_prologue staged (sh.adam) and, with parameter groups (PGS: the offset of pg_stage's
// values in the dynamic shared memory, < 0 = none), each tensor's step size and decoupled factor by those of the new lr.
// The values of all three decisions are formed before the wait, so only a selection follows it: warp 0's lanes
// 6 (d + 1) + s form segment slot s's step size for decision d in parallel, and a shuffle picks them.
struct LrCandidates {
  float step[3];                  // (float)(lr' / bc1) for the decisions -1, 0, +1
  float decay[3];                 // the decoupled factor at lr' (parameter groups)
};
__device__ __forceinline__ LrCandidates lr_candidates(const AdaptiveLr& al, double lr, double bc1,
                                                      const ParamGroups* pg, int k) {
  LrCandidates c;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double x = lr_adapt(lr, d - 1, al.lo, al.hi);
    c.step[d] = (float)(x / bc1);
    c.decay[d] = pg ? lr_decay(pg, k, x) : 1.f;
  }
  return c;
}
__device__ __forceinline__ float lr_pick(const float* v, int dec) { return dec < 0 ? v[0] : (dec > 0 ? v[2] : v[1]); }

template <class L, int PGS = -1>
__device__ __noinline__ void tail_kl_gate(const StepArgs& a, TailShared& sh, const float* pull, const unsigned* myflags,
                                          bool sys) {
  const int t = threadIdx.x;
  LrCandidates ten{};
  float seg = 0.f;
  if (a.alr.in) {
    if (t < 18) {     // slot t % 6 = [seg][live] at the count tail_prologue staged, decision t / 6 - 1
      const long long stp = sh.steps[t % 6];
      seg = (float)(lr_adapt(a.alr.in[0], t / 6 - 1, a.alr.lo, a.alr.hi) /
                    (1.0 - ipow((double)a.beta1, stp > 0 ? stp : 1)));
    }
    if constexpr (PGS >= 0) {
      if (t < a.pg->n)
        ten = lr_candidates(a.alr, a.alr.in[t], 1.0 - ipow((double)a.pg->beta1[t], a.tsteps_in[t] + 1), a.pg, t);
    }
  }
  if (t < a.world) tail_poll(a, sh, myflags, t, L::stats / SLICE, sys);
  __syncthreads();
  if (t == 0) {
    float s4 = ld_relaxed(pull + L::stats + 4, sys), s8 = ld_relaxed(pull + L::stats + 8, sys);
    for (int p = 1; p < a.world; ++p) {
      s4 += ld_relaxed(pull + (size_t)p * G_ROW + L::stats + 4, sys);
      s8 += ld_relaxed(pull + (size_t)p * G_ROW + L::stats + 8, sys);
    }
    sh.stop = sh.timeout == 0 && kl_exceeds(s8, s4, a.kl_limit);
    sh.lr_dec = a.alr.in && !sh.stop ? lr_decision(s8, s4, a.alr.up, a.alr.down) : 0;
  }
  __syncthreads();
  if (!a.alr.in) return;
  const int dec = sh.lr_dec;
  if (t < 32) {
    const float v = __shfl_sync(0xffffffffu, seg, 6 * (dec + 1) + t % 6);
    if (t < 6) sh.adam[t * 2] = v;
  }
  if constexpr (PGS >= 0) {
    extern __shared__ __align__(16) float smem[];
    float* const pgs = smem + PGS;
    if (t < a.pg->n) {
      pgs[t] = lr_pick(ten.step, dec);
      pgs[2 * PG_MAX_TENSORS + t] = lr_pick(ten.decay, dec);
    }
  }
  __syncthreads();
}

// KL-adaptive lr (a.alr.in != NULL): the model's next lr state and the decision slot, written by the CTA that owns the
// statistics slice, after its reduction has written that slice (write_grad_col's zero in slot 22 comes first, in the
// same CTA).  Nothing moves on a step that applied nothing (a KL stop, a non-finite step, a peer give-up of this CTA).
// A peer give-up is decided per CTA, like every other effect of one: tail_write_steps takes the counters CTA's view (the
// chain CTA, rl-mlp CTA 0), this function the statistics owner's, so after a give-up seen by only one of them the lr
// state and the step counters may disagree about whether the step applied, as the parameters of different slices
// already may.  Such a step leaves the ranks out of sync as a whole: upb_peer_timeouts counts it and the host discards
// the update (PPOUpdater raises UpbError; the run restores its last checkpoint), so neither value is used.  Writing both
// from one CTA would move the counters' writer, which the option-off kernels keep where it is, or order two CTAs' writes
// of slot 22, which would cost a wait on every step.
template <class L>
__device__ __noinline__ void tail_write_lr(const StepArgs& a, const TailShared& sh) {
  static_assert((L::stats + LR_DECISION_SLOT) / SLICE == L::stats / SLICE, "the decision slot is in the statistics slice");
  if (blockIdx.x != (unsigned)((L::stats / SLICE) % gridDim.x)) return;
  const bool applied = sh.timeout == 0 && !sh.stop;
  const int dec = applied ? sh.lr_dec : 0;
  lr_write(a.alr, a.pg, threadIdx.x, dec, applied);
  if (threadIdx.x == 0) a.grad_out[L::stat_offset + LR_DECISION_SLOT] = (float)dec;
}


// The chain CTA's attention chain: waits for the slices that hold every rank's virtual attention gradients, adds them in
// rank order and chains them to the six real tensors; STEPS: threads 0-3 write the step counters after the polls.  chain = fused_tail's shared block: sG [816] | sWin [768] | sW3
// [768] | sB [48] (the parameters, prefetched) | sOut [CHAIN_ELEMS] (the result, in the chain's element order).
template <bool STEPS>
__device__ __forceinline__ void tail_chain_grads(const StepArgs& a, TailShared& sh, const float* pull,
                                                 const unsigned* myflags, bool sys, float* chain) {
  float* sG = chain;
  float* sWin = sG + 816;
  float* sW3 = sWin + 768;
  float* sB = sW3 + 768;
  float* sOut = sB + 48;
  const int tid = threadIdx.x, world = a.world;
  {
    constexpr int NCH = CHAIN_S1 - CHAIN_S0 + 1;
    if (tid < world * NCH) tail_poll(a, sh, myflags, tid % world, CHAIN_S0 + tid / world, sys);
    __syncthreads();
  }
  if constexpr (STEPS) {
    if (tid < 4) tail_write_steps(a, sh);
  }
  {   // all loads of a thread are issued before the first use
    float v0[MAX_PEERS], v1[MAX_PEERS];
#pragma unroll
    for (int p = 0; p < MAX_PEERS; ++p) {
      v0[p] = 0.f; v1[p] = 0.f;
      if (p < world) {
        v0[p] = ld_relaxed(pull + (size_t)p * G_ROW + G_QC + tid, sys);
        if (tid + NT < 816) v1[p] = ld_relaxed(pull + (size_t)p * G_ROW + G_QC + tid + NT, sys);
      }
    }
    float s0 = v0[0], s1 = v1[0];
#pragma unroll
    for (int p = 1; p < MAX_PEERS; ++p) if (p < world) { s0 += v0[p]; s1 += v1[p]; }
    sG[tid] = s0;
    if (tid + NT < 816) sG[tid + NT] = s1;
  }
  __syncthreads();
  if (tid < 256) attention_chain(tid, sG, sWin, sW3, sB, sOut, 256, sOut + 768, sOut + 1536, 16, sOut + 1584);
  __syncthreads();
}

// Global gradient-norm clip of the fused tails (a.max_norm > 0, upb_set_max_grad_norm), after this CTA's pushes and the
// KL gate.  On a step that does not stop (sh.stop, tail_kl_gate), in turn:
//   1. the owned slices are reduced as tail_reduce_adam does, without Adam, and each slice's partial of the norm
//      (gclip_slice_tree) is published in this rank's own buffer with a flag carrying the step sequence: every rank
//      holds every rank's contributions, so the ranks form the same partials without another message;
//   2. the chain CTA (chain != NULL) runs the attention chain and publishes its partial;
//   3. every CTA waits for all partials (bounded like the peer polls; a flag marked by a CTA that gave up counts as a
//      give-up here too), forms the norm and coef (gclip_norm / gclip_coef);
//   4. Adam on coef * g for the owned columns (reloaded from grad_out, which the same thread wrote) and the chain's.
// Each CTA publishes everything it owns before it waits, so no grid size deadlocks.  A stopping step only reduces (and
// marks slot 13, as tail_reduce_adam does) and runs the chain.
// The non-finite guard (a.nonfinite_guard, upb_set_nonfinite_guard) is a decision on the same norm, with a.max_norm == 0
// when the clip itself is off (coef is then 1).  The owner of the statistics slice, which holds no parameter, publishes
// NaN as that slice's partial when the reduced slot 7 is not 0, so the norm every CTA and rank forms in step 3 is finite
// exactly on a good step, without a second poll of the statistics slice.  A bad step skips step 4, marks slot 19 and
// keeps the step counters (sh.stop); slot 17 stays 0.  sq: free dynamic shared memory,
// float64[SLICE + FLAG_STRIDE + 1] (the step kernel's static shared memory has no room for it).
// PG: the parameter groups are on (a.pg, k_sgnn_pg / k_mlp_pg; pgs: pg_stage's values).  A frozen tensor's reduced
// columns, the chain's included, are written and enter the norm as 0 (the sums the chain reads are not masked), and each
// trained column steps with its tensor's values.  These kernels take this tail whether or not the clip or the guard is
// on: with max_norm == 0 and the guard off, coef is 1 and the step is the plain fused step's, bit for bit.
template <class L, bool PG = false>
__device__ __forceinline__ void tail_gclip(const StepArgs& a, TailShared& sh, const float* pull,
                                           const unsigned* myflags, bool sys, int c, bool active, double* sq,
                                           float* chain, const float* pgs = nullptr) {
  constexpr bool CHAIN = L::chain0_end > L::chain0_begin;
  constexpr int NPARTS = L::nslice + (CHAIN ? 1 : 0);
  static_assert(NPARTS <= FLAG_STRIDE, "a flag word per partial");
  double* const sparts = sq + SLICE;
  float& snorm = *reinterpret_cast<float*>(sparts + FLAG_STRIDE);
  float& scoef = *(&snorm + 1);
  const int tid = threadIdx.x, world = a.world;
  const unsigned par = a.seq & 1u;
  float* const mine = a.peers[a.rank];
  double* const parts = reinterpret_cast<double*>(mine + XCHG_GCLIP) + (size_t)par * FLAG_STRIDE;
  unsigned* const pflags = reinterpret_cast<unsigned*>(mine + XCHG_GCLIP_FLAGS) + (size_t)par * FLAG_STRIDE;
  const bool stop = sh.stop;      // uniform: after tail_kl_gate's barrier

  for (int sl = blockIdx.x; sl < L::nslice; sl += gridDim.x) {
    if (tid < world) tail_poll(a, sh, myflags, tid, sl, sys);
    __syncthreads();
    const int col = sl * SLICE + c;
    if (active) {
      double x = 0.0;
      if (L::row % SLICE == 0 || col < L::row) {
        float s = rank_sum(pull, world, col, sys);
        if constexpr (PG) {
          if (col < L::num_params && !pg_trained(a, pgs, col)) s = 0.f;
        }
        if (write_grad_col<L>(a.grad_out, col, s)) x = (double)s * (double)s;
        else if (stop && col == L::stats + KL_STOP_SLOT) {     // after write_grad_col's zero, same thread
          a.grad_out[L::stat_offset + KL_STOP_SLOT] = 1.f;
          *a.kl_stop = 1u;
        } else if (a.nonfinite_guard && col == L::stats + NONFINITE_COUNT_SLOT && !(s == 0.f)) {
          x = CUDART_NAN;         // the guard's slot-7 condition travels in this slice's partial: the norm is then NaN
        }
      }
      sq[c] = x;
    }
    __syncthreads();
    if (tid < 32 && !stop) {               // warp 0 reads sq before it reaches the next slice's barrier, after which sq is rewritten
      const double p = gclip_slice_tree(sq[tid], sq[tid + 32], sq[tid + 64], sq[tid + 96]);
      if (tid == 0) {
        parts[sl] = p;
        st_release(pflags + sl, (a.seq << 1) | (sh.timeout ? 1u : 0u), false);
      }
    }
  }
  if constexpr (CHAIN) {
    if (chain != nullptr) {
      tail_chain_grads<false>(a, sh, pull, myflags, sys, chain);
      const float* sOut = chain + 2400;
      if constexpr (PG) {
        for (int i = tid; i < CHAIN_ELEMS; i += blockDim.x)
          if (!pg_trained(a, pgs, chain_dst(i))) chain[2400 + i] = 0.f;
        __syncthreads();
      }
      if (stop) {
        for (int i = tid; i < CHAIN_ELEMS; i += blockDim.x) a.grad_out[chain_dst(i)] = sOut[i];
        return;
      }
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = tid + j * GCLIP_BLOCK;
        if (i < CHAIN_ELEMS) {
          const float g = sOut[i];
          a.grad_out[chain_dst(i)] = g;
          s += (double)g * (double)g;
        }
      }
      s = gclip_block_tree(s, sq);
      if (tid == 0) {
        parts[L::nslice] = s;
        st_release(pflags + L::nslice, (a.seq << 1) | (sh.timeout ? 1u : 0u), false);
      }
    }
  }
  if (stop) return;

  for (int i = tid; i < NPARTS; i += blockDim.x) {
    unsigned polls = 0, f;
    while ((int)(((f = ld_acquire(pflags + i, false)) & ~1u) - (a.seq << 1)) < 0) {
      if (++polls >= PEER_SPIN_LIMIT) { sh.timeout = 1; break; }
    }
    if (f & 1u) sh.timeout = 1;
    double p;
    asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(p) : "l"(parts + i) : "memory");
    sparts[i] = p;
  }
  __syncthreads();
  if (tid == 0) {
    snorm = gclip_norm(sparts, NPARTS);
    scoef = a.max_norm > 0.f ? gclip_coef(snorm, a.max_norm) : 1.f;      // the guard alone: g * 1 is g, bit for bit
    if (a.nonfinite_guard && !isfinite(snorm)) sh.stop = 1;              // tail_write_steps keeps the counters
  }
  __syncthreads();

  const float norm = snorm, coef = scoef;
  const bool bad = a.nonfinite_guard && !isfinite(norm);                 // the same float on every CTA and rank
  const bool dead = sh.timeout != 0 || bad;
  const bool live_lu = sh.bits & 1u, live_rd = sh.bits & 2u;
  if (active) {
    for (int sl = blockIdx.x; sl < L::nslice; sl += gridDim.x) {
      const int col = sl * SLICE + c;
      if (col < L::num_params && !chain_owns<L>(col)) {
        int seg = 0;
        bool live = true;
        if (col >= L::lu_begin && col < L::rd_begin) { seg = 1; live = live_lu; }
        else if (col >= L::rd_begin && col < L::policy_end) { seg = 2; live = live_rd; }
        if (live && !dead) {
          if constexpr (PG)
            pg_adam_elem(a, pgs, col, __fmul_rn(a.grad_out[col], coef));
          else
            adam_elem(a, col, __fmul_rn(a.grad_out[col], coef), a.adam_m[col], a.adam_v[col], a.params_rw[col],
                      sh.adam[(seg * 2 + 1) * 2], sh.adam[(seg * 2 + 1) * 2 + 1]);
        } else if (!dead) {
          prox_keep(a, col);
        }
      } else if (col == L::stats + GCLIP_NORM_SLOT && !dead && a.max_norm > 0.f) {
        a.grad_out[L::stat_offset + GCLIP_NORM_SLOT] = norm;      // after write_grad_col's zero, same thread
      } else if (col == L::stats + NONFINITE_SLOT && bad && sh.timeout == 0) {
        a.grad_out[L::stat_offset + NONFINITE_SLOT] = 1.f;        // likewise
      }
    }
  }
  if constexpr (CHAIN) {
    if (chain != nullptr && !dead) {
      const float* sOut = chain + 2400;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = tid + j * GCLIP_BLOCK;
        if (i < CHAIN_ELEMS) {
          const int dst = chain_dst(i);
          if constexpr (PG)
            pg_adam_elem(a, pgs, dst, __fmul_rn(sOut[i], coef));
          else
            adam_elem(a, dst, __fmul_rn(sOut[i], coef), a.adam_m[dst], a.adam_v[dst], a.params_rw[dst], sh.adam[2],
                      sh.adam[3]);      // segment 0 (encoder), live
        }
      }
    }
  }
}

// A training launch while the stop word is set: no graph, no partial row, no exchange.  The fused step writes the
// skipped row (zeros, KL_SKIP_SLOT = 1) and unchanged step counters, clears the next launch's stage word as
// tail_prologue does, and arrives at the cumulative grid counter, which the host advances by this launch's grid.
template <class L>
__device__ __noinline__ void skip_step(const StepArgs& a) {
  if (!a.fuse_tail) return;       // the two-call path: the reduction kernel writes the skipped row
  const int tid = threadIdx.x;
  for (int i = blockIdx.x * blockDim.x + tid; i < L::stat_offset + UPB_STAT_COUNT; i += gridDim.x * blockDim.x)
    write_skip_elem(a.grad_out, L::stat_offset, i);
  if (blockIdx.x == 0) {
    if (tid < 4) a.steps_out[tid] = a.steps_in[tid];
    if (tid == 4) a.gridbar[2 + ((a.seq & 1u) ^ 1u)] = 0u;
    if (a.pg) pg_keep_steps(a.pg, a.tsteps_in, a.tsteps_out, tid);
    if (a.alr.in) lr_write(a.alr, a.pg, tid, 0, false);
  }
  grid_arrive(a.gridbar);
}

// Everything that does not depend on other CTAs' results is fetched or computed BEFORE the barrier it would otherwise
// follow, so the serial part after the barrier is short.  GCLIP: the global clip is on (a.max_norm > 0; tail_gclip).
// PG (with GCLIP): the parameter groups are on (k_sgnn_pg).
// pg_stage's values sit above the chain CTA's block [0, 4032), sPart [4096, 4608) and tail_gclip's sq [4608, 5122)
constexpr int PG_SMEM = 5632;
static_assert(PG_SMEM + 4 * PG_MAX_TENSORS <= (int)(SMEM_BYTES / 4), "pg_stage's values fit the dynamic shared memory");
template <bool GCLIP, bool PG = false>
__device__ __forceinline__ void fused_tail(const StepArgs& a, float* smem, unsigned stage_bits) {
  static_assert(GCLIP || !PG, "the parameter groups take the clip's tail");
  const int tid = threadIdx.x;
  const int nparts = gridDim.x;
  const int world = a.world, me = a.rank;
  const bool sys = world > 1;                       // flag / data scope: peers over NVLink need system scope
  const unsigned par = a.seq & 1u;
  const bool chain_cta = blockIdx.x == gridDim.x - 1;
  __shared__ TailShared sh;
#define UPB_TSTAMP(ID) do { if (a.stamps != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.stamps[ID] = clock64(); } while (0)
  UPB_TSTAMP(40);
  float* const mine = a.peers[me];
  const float* const pull = mine + (size_t)par * MAX_PEERS * G_ROW;        // [src][G_ROW] contributions delivered to me
  const unsigned* const myflags = reinterpret_cast<const unsigned*>(mine + XCHG_FLAGS) + (size_t)par * MAX_PEERS * FLAG_STRIDE;
  tail_prologue(a, sh, stage_bits);
  if constexpr (PG) pg_stage(a, smem + PG_SMEM);
  // this thread's column of the first owned slice: its moments / parameter do not depend on the reduction
  const int col0 = blockIdx.x * SLICE + (tid >> 2), part = tid & 3;
  float pm = 0.f, pv = 0.f, pp = 0.f;
  if (!GCLIP && part == 0 && col0 < NUM_PARAMS && !chain_owns<SgnnRow>(col0)) {
    pm = a.adam_m[col0]; pv = a.adam_v[col0]; pp = a.params_rw[col0];
  }
  // the chain CTA also prefetches what the attention chain needs from the (still old) parameters
  float* sG = smem;                 // Qc | qbc | Kc | Vc | vbc gradients [816]
  float* sWin = sG + 816;           // in_proj_weight [768]
  float* sW3 = sWin + 768;          // Wq | Wk | Wv [768]
  float* sB = sW3 + 768;            // bq | bk | bv [48]
  float* sOut = sB + 48;            // new gradients: Wq,Wk,Wv [768] | Win [768] | bq,bk,bv [48] | bin [48]
  const int pW[3] = {P_ATT_Q_W, P_ATT_K_W, P_ATT_V_W};
  const int pB[3] = {P_ATT_Q_B, P_ATT_K_B, P_ATT_V_B};
  float cm[4], cv[4], cp[4];
  int cdst[4];
  if (chain_cta) {
    const float* P = a.params_rw;
    for (int i = tid; i < 768; i += NT) sWin[i] = P[P_MHA_IN_W + i];
    if (tid < 256) { sW3[tid] = P[P_ATT_Q_W + tid]; sW3[256 + tid] = P[P_ATT_K_W + tid]; sW3[512 + tid] = P[P_ATT_V_W + tid]; }
    if (tid < 16) { sB[tid] = P[P_ATT_Q_B + tid]; sB[16 + tid] = P[P_ATT_K_B + tid]; sB[32 + tid] = P[P_ATT_V_B + tid]; }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = tid + j * NT;
      int dst = 0;
      if (i < 768) dst = pW[i >> 8] + (i & 255);
      else if (i < 1536) dst = P_MHA_IN_W + (i - 768);
      else if (i < 1584) dst = pB[(i - 1536) >> 4] + ((i - 1536) & 15);
      else if (i < 1632) dst = P_MHA_IN_B + (i - 1584);
      cdst[j] = dst;
      if (!GCLIP && i < 1632) { cm[j] = a.adam_m[dst]; cv[j] = a.adam_v[dst]; cp[j] = P[dst]; }
    }
  }
  const unsigned flagword = tail_barrier(a);
  UPB_TSTAMP(41);

  // ---- PUSH: local column sums of the owned slices -> every rank's buffer.  Coalesced: a warp reads 32 consecutive
  // columns of ONE partial row per load (one 128-byte line; four-row gathers cost four L1 wavefronts each); warp w owns
  // column group w & 3 and the rows r = (w >> 2) mod 4; the four row groups are combined through shared memory in the
  // order ((g0 + g1) + (g2 + g3)).
  float* sPart = smem + 4096;                        // [4 row groups][SLICE] (the chain CTA's prefetch sits below 4096)
  for (int sl = blockIdx.x; sl < NSLICE; sl += gridDim.x) {
    const int lane = tid & 31, warp = tid >> 5, cg = warp & 3, rg = warp >> 2;
    const float* src = a.gpart + sl * SLICE + cg * 32 + lane;
    float s = 0.f;
    for (int r0 = rg; r0 < nparts; r0 += 160) {      // all loads of a chunk of 160 rows in flight together, fixed order
      float t[40];
#pragma unroll
      for (int j = 0; j < 40; ++j) t[j] = r0 + 4 * j < nparts ? __ldcg(src + (size_t)(r0 + 4 * j) * G_ROW) : 0.f;
#pragma unroll
      for (int w = 1; w < 40; w <<= 1)
#pragma unroll
        for (int j = 0; j + w < 40; j += 2 * w) t[j] += t[j + w];
      s += t[0];
    }
    __syncthreads();                                 // the previous slice's partials have been consumed
    sPart[rg * SLICE + cg * 32 + lane] = s;
    __syncthreads();
    if (tid < SLICE) {
      const float v = (sPart[tid] + sPart[SLICE + tid]) + (sPart[2 * SLICE + tid] + sPart[3 * SLICE + tid]);
      const int col = sl * SLICE + tid;
      for (int r = 0; r < world; ++r) st_relaxed(sh.push[r] + col, v, sys);
    }
  }
  tail_release<SgnnRow>(a, flagword, NT, sys);
  if (a.kl_stop) tail_kl_gate<SgnnRow, PG ? PG_SMEM : -1>(a, sh, pull, myflags, sys);
  UPB_TSTAMP(42);
  if constexpr (GCLIP) {
    tail_gclip<SgnnRow, PG>(a, sh, pull, myflags, sys, tid >> 2, part == 0,
                            reinterpret_cast<double*>(sPart + 4 * SLICE), chain_cta ? smem : nullptr,
                            PG ? smem + PG_SMEM : nullptr);
    if (a.alr.in) tail_write_lr<SgnnRow>(a, sh);
    if (chain_cta && tid < 4) tail_write_steps(a, sh);
    if constexpr (PG) {
      if (chain_cta && tid < a.pg->n) tail_write_tensor_steps(a, sh);
    }
    tail_count_timeout(a, sh);
    return;
  }

  tail_reduce_adam<SgnnRow>(a, sh, pull, myflags, sys, tid >> 2, part == 0, col0, pm, pv, pp);
  if (a.alr.in) tail_write_lr<SgnnRow>(a, sh);
  UPB_TSTAMP(43);
  if (!chain_cta) {
    tail_count_timeout(a, sh);
    return;
  }

  // ---- ATTENTION CHAIN (last CTA): the virtual gradients of all ranks, chained to the six attention tensors, Adam
  tail_chain_grads<true>(a, sh, pull, myflags, sys, sG);
  const bool dead = sh.timeout != 0 || sh.stop;
#pragma unroll
  for (int j = 0; j < 4; ++j) {       // 1632 = 3.2 x 512 elements
    const int i = tid + j * NT;
    if (i < 1632) {
      const float g = sOut[i];
      a.grad_out[cdst[j]] = g;
      if (!dead) adam_elem(a, cdst[j], g, cm[j], cv[j], cp[j], sh.adam[2], sh.adam[3]);     // segment 0 (encoder), live
    }
  }
  tail_count_timeout(a, sh);
  UPB_TSTAMP(44);
}

// The step kernel's body; GCLIP: the fused step of the global clip (k_sgnn_gclip); PG: of the parameter groups
// (k_sgnn_pg); VALUES: the value-only sweep (k_sgnn_values).
template <bool TRAIN, bool GCLIP, bool PG = false, bool VALUES = false>
__device__ __forceinline__ void sgnn_step(const StepArgs& a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ __align__(8) uint64_t s_mbar[4];   // bulk-copy completion: [0] graph staging, [1] EPQ reload, [2] feature reload, [3] h rows for g_W
  if constexpr (TRAIN) {
    if (a.kl_stop && kl_stop_set(a.kl_stop)) {       // set only by a finished launch: the same value in every CTA
      skip_step<SgnnRow>(a);
      return;
    }
  } else {
    if (a.kl_stop && kl_stop_set(a.kl_stop)) return;   // the proximal forward of a skipped step (StepArgs::prox_lp)
  }
  const long long t_cta0 = a.stamps ? clock64() : 0;
  if (a.stamps && threadIdx.x == 0 && blockIdx.x == 0) {      // clock64 vs globaltimer (ns): the SM clock actually running
    unsigned long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    a.stamps[30] = t_cta0; a.stamps[32] = (long long)gt;
  }
  if (threadIdx.x == 0) {
    mbar_init(s_mbar + 0, 1); mbar_init(s_mbar + 1, 1); mbar_init(s_mbar + 2, 1); mbar_init(s_mbar + 3, 1);
    fence_mbar_init();
  }
  unsigned nstaged = 0;                         // graphs staged by bulk copies so far: phase parity of the mbarriers
  load_weights(a.params, smem);
  float* gp = nullptr;
  if constexpr (TRAIN) {
    gp = a.gpart + (size_t)blockIdx.x * G_ROW;
    for (int i = threadIdx.x; i < G_ROW / 4; i += NT) reinterpret_cast<float4*>(gp)[i] = f4(0.f);
  }
  __syncthreads();
  if (a.stamps && threadIdx.x == 0 && blockIdx.x < 160) a.stamps[64 + 160 + blockIdx.x] = clock64() - t_cta0;   // launch prologue
  const BlobHeader& hd = *reinterpret_cast<const BlobHeader*>(a.blob);
  const GraphDesc* descs = reinterpret_cast<const GraphDesc*>(a.blob + hd.off_desc);
  float* scr = a.scratch + (size_t)blockIdx.x * a.scratch_stride;
  unsigned stage_bits = 0;     // bit 0: a land-use graph, bit 1: a road graph was walked by this CTA
  for (int item = blockIdx.x; item < a.count; item += gridDim.x) {
    const int gid = a.ids ? a.ids[item] : item;
    const GraphDesc d = descs[gid];
    stage_bits |= 1u << (d.stage & 1);
    if (d.n > a.n_cap || d.e > a.e_cap || d.n < 1) {   // larger than the context was sized for: skip, flag
      if (threadIdx.x == 0) {
        if constexpr (TRAIN) gacc(gp, G_STATS + 7, 1.f);
        if (a.out_value) a.out_value[gid] = CUDART_NAN_F;
        if (a.out_logp) a.out_logp[gid] = CUDART_NAN_F;
        if (a.out_entropy) a.out_entropy[gid] = CUDART_NAN_F;
      }
      if constexpr (!TRAIN && !VALUES) { write_skipped_logit_row<NT>(a, gid, d.stage); write_skipped_cand_logp<NT>(a, d); }
      continue;
    }
    if (item + (int)gridDim.x < a.count) prefetch_next_graph<TRAIN>(a, item + gridDim.x);
    const bool big = d.n > NS || 2 * d.e > AS || d.k > KS || d.ord_rounds > ORD_ROUNDS;
    // stamps: the SECOND graph of CTA 0 (steady state)
    if (big) graph_body<TRAIN, true, VALUES>(a, hd, d, gid, item, smem, gp, scr, item == (int)(blockIdx.x + gridDim.x), s_mbar, 0u);
    else { graph_body<TRAIN, false, VALUES>(a, hd, d, gid, item, smem, gp, scr, item == (int)(blockIdx.x + gridDim.x), s_mbar, nstaged & 1u); ++nstaged; }
    __syncthreads();
  }
  if (a.stamps && threadIdx.x == 0 && blockIdx.x < 160) a.stamps[64 + blockIdx.x] = clock64() - t_cta0;           // CTA busy time
  if (a.stamps && threadIdx.x == 0 && blockIdx.x == 0) {
    unsigned long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    a.stamps[31] = clock64(); a.stamps[33] = (long long)gt;
  }
  if constexpr (TRAIN) {
    if (a.fuse_tail) fused_tail<GCLIP, PG>(a, smem, stage_bits);
  }
}

template <bool TRAIN>
__global__ void __launch_bounds__(NT, 1) k_sgnn(const __grid_constant__ StepArgs a) {
  sgnn_step<TRAIN, false>(a);
}
// The fused step with the global clip on (a.max_norm > 0): a kernel of its own, so that the clip's tail adds nothing to
// k_sgnn<true>'s registers (a device call from its tail costs the graph loop spills).
__global__ void __launch_bounds__(NT, 1) k_sgnn_gclip(const __grid_constant__ StepArgs a) {
  sgnn_step<true, true>(a);
}
// The fused step with parameter groups (a.pg != NULL, upb_set_param_groups), with or without the clip and the guard: a
// kernel of its own, so that the tables add nothing to the two kernels above.
__global__ void __launch_bounds__(NT, 1) k_sgnn_pg(const __grid_constant__ StepArgs a) {
  sgnn_step<true, true, true>(a);
}
// The value-only sweep (upb_values): the forward up to the value head, which writes a.out_value only.  Its values are
// k_sgnn<false>'s bit for bit: the same code computes them, and what it leaves out never feeds the value head.
__global__ void __launch_bounds__(NT, 1) k_sgnn_values(const __grid_constant__ StepArgs a) {
  sgnn_step<false, false, false, true>(a);
}

}  // namespace upb
