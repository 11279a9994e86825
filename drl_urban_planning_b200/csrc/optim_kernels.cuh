// Small kernels around the fused SGNN kernel: cross-CTA gradient reduction, attention chain rule,
// clip + Adam, GAE; and the column helpers the reductions share with the fused step tails.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/upb200.h"
#include "layout.h"

namespace upb {

// ---- helpers of the gradient reductions and the fused step tails (L: a row layout, layout.h) ------------------------
template <class L>
__device__ __forceinline__ bool chain_owns(int col) {
  return (col >= L::chain0_begin && col < L::chain0_end) || (col >= L::chain1_begin && col < L::chain1_end);
}

// Writes the reduced partial-row column `col` (value v) into the flat gradient buffer: a parameter's gradient (unless
// the attention chain writes it), a zero for the pad words, a statistic copied (the sums, stat_summed) or zeroed.
// Returns true where a parameter's gradient was written (its Adam step follows in the fused tails).
template <class L>
__device__ __forceinline__ bool write_grad_col(float* grad, int col, float v) {
  bool param = false;
  if (col < L::num_params && !chain_owns<L>(col)) { grad[col] = v; param = true; }
  else if (col >= L::num_params && col < L::stat_offset) grad[col] = 0.f;
  if (col >= L::stats && col < L::stats + UPB_STAT_COUNT)
    grad[L::stat_offset + (col - L::stats)] = stat_summed(col - L::stats) ? v : 0.f;
  return param;
}

// ---- per-tensor parameter groups (upb_set_param_groups): torch.optim.Adam over param_groups, with frozen tensors.  One
// table per model in device memory; NULL in the launch arguments means no table (every tensor trained with the
// context's lr and weight decay, the per-segment counters alone).
constexpr int PG_MAX_TENSORS = 32;        // the SGNN's 32 tensors; the rl-mlp has 18
struct ParamGroups {
  double lr[PG_MAX_TENSORS];              // a double per tensor, as upb_set_lr keeps it
  float weight_decay[PG_MAX_TENSORS];
  int trained[PG_MAX_TENSORS];            // 0: frozen -- no Adam step, a zero gradient column, the count kept
  int seg[PG_MAX_TENSORS];                // the tensor's segment: 0 encoder / value, 1 land-use head, 2 road head
  int n;                                  // tensors of the model
  uint8_t tensor_of[NUM_PARAMS];          // flat column -> tensor (upb_param_slot order)
  // Adam settings per tensor (upb_set_adam, upb_set_param_groups_adam), formed on the host.  A tensor at the context's
  // creation-time betas and eps, coupled and without AMSGrad, holds exactly the values of the untabled steps.
  float beta1[PG_MAX_TENSORS];            // fp32(beta1): the bias correction 1 - beta1^t is formed in double from it
  float beta2[PG_MAX_TENSORS];            // fp32(beta2): mul_(beta2), and the bias correction 2
  float w1[PG_MAX_TENSORS];               // 1.f - beta1: lerp_'s weight
  float w2[PG_MAX_TENSORS];               // 1.f - beta2: addcmul_'s value
  float eps[PG_MAX_TENSORS];
  float decay[PG_MAX_TENSORS];            // decoupled decay: fp32(1 - lr * weight_decay), 1 = none (weight_decay above is 0)
  int amsgrad[PG_MAX_TENSORS];            // 1: the denominator takes max_exp_avg_sq
  float* vmax;                            // max_exp_avg_sq [num_params] (NULL while no tensor has had amsgrad)
  double decoupled_wd[PG_MAX_TENSORS];    // the double weight decay of a decoupled tensor (0: none): the KL-adaptive lr
                                          // re-forms decay from it and the step's lr
};
__device__ __forceinline__ bool pg_frozen(const ParamGroups* pg, int col) { return !pg->trained[pg->tensor_of[col]]; }

// torch 2.11's _single_tensor_adam on element i of tensor k of a table, after the clip (g is the clipped gradient):
//   decoupled: p *= fp32(1 - lr * wd)   coupled: g += wd * p (fma, as the untabled steps)
//   m = m.lerp(g, w1); v = v * beta2 + (w2 * g) * g; amsgrad: vmax = max(vmax, v) (NaN propagates, as torch.maximum)
//   p += -step_size * (m / (sqrt(v or vmax) / sqrt(bc2) + eps))
// With a tensor at the default settings this is the untabled arithmetic, operation for operation.  Only called on a
// step that updates the tensor's moments, so a frozen tensor, an absent head and a skipped step neither decay nor touch
// vmax.  decay: the tensor's decoupled factor as the caller staged it (pg->decay[k], or the KL-adaptive lr's re-formed
// one, lr_decay).
__device__ __forceinline__ float pg_adam_step(const ParamGroups* pg, int k, int i, float g, float step_size,
                                              float bc2_sqrt, float decay, float* params, float* mm, float* vv) {
  float p = params[i];
  const float wd = pg->weight_decay[k];
  if (decay != 1.f) p = __fmul_rn(p, decay);
  if (wd != 0.f) g = __fmaf_rn(wd, p, g);
  float m = mm[i], v = vv[i];
  m = __fadd_rn(m, __fmul_rn(pg->w1[k], __fsub_rn(g, m)));
  v = __fadd_rn(__fmul_rn(v, pg->beta2[k]), __fmul_rn(__fmul_rn(pg->w2[k], g), g));
  float vd = v;
  if (pg->amsgrad[k]) {
    const float vm = pg->vmax[i];
    vd = (v > vm || v != v) ? v : vm;
    pg->vmax[i] = vd;
  }
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vd), bc2_sqrt), pg->eps[k]);
  p = __fadd_rn(p, __fmul_rn(-step_size, __fdiv_rn(m, denom)));
  params[i] = p;
  mm[i] = m;
  vv[i] = v;
  return p;
}

// PPO-EWMA's proximal parameters (upb_set_prox_ewma) on element i of a step that applied Adam, in the thread that wrote
// the element: theta_prox <- fma(beta, theta_prox - theta, theta), theta the value the step left (new, or unchanged for a
// frozen tensor or an absent head)
__device__ __forceinline__ void prox_ewma_elem(float* prox, float beta, int i, float theta) {
  prox[i] = __fmaf_rn(beta, __fsub_rn(prox[i], theta), theta);
}

// Per-tensor counts (double-buffered as the per-segment ones: in -> out) of a step that changes nothing: copied.
__device__ __forceinline__ void pg_keep_steps(const ParamGroups* pg, const long long* in, long long* out, int t) {
  if (t < pg->n) out[t] = in[t];
}

// ---- KL stop (upb_set_target_kl).  The criterion on a step's globally reduced statistics, slot 8 (sum of the approximate
// KL) and slot 4 (|ind|), with limit = fp32(1.5 * target_kl) (upb200.cu: kl_limit).  False for a NaN and for a minibatch
// without an exps != 0 graph.
constexpr int KL_STOP_SLOT = 13;      // 1 in the row of the step that stopped
constexpr int KL_SKIP_SLOT = 14;      // 1 in the row of a step skipped while the stop word is set (the rest is zeros)
static_assert(KL_SKIP_SLOT < UPB_STAT_COUNT && !stat_summed(KL_STOP_SLOT) && !stat_summed(KL_SKIP_SLOT),
              "the stop slots are not sums");
static_assert(VCLIP_COUNT_SLOT < UPB_STAT_COUNT && VCLIP_LOSS_SLOT > KL_SKIP_SLOT, "value-clip slots");

__device__ __forceinline__ bool kl_exceeds(float s8, float s4, float limit) {
  return s8 > __fmul_rn(limit, fmaxf(s4, 1.f));
}
__device__ __forceinline__ bool kl_stop_set(const unsigned int* word) {
  return *reinterpret_cast<const volatile unsigned int*>(word) != 0u;
}
// element i of a skipped step's gradient buffer (i < stat_offset + UPB_STAT_COUNT)
__device__ __forceinline__ void write_skip_elem(float* grad, int stat_offset, int i) {
  grad[i] = i == stat_offset + KL_SKIP_SLOT ? 1.f : 0.f;
}

// ---- KL-adaptive learning rate (upb_set_adaptive_lr): RSL-RL's schedule="adaptive" with desired_kl, decided on the same
// globally reduced slots 8 and 4 as the KL stop, in fp32 as kl_exceeds:
//   down (-1): s8 > fp32(2 desired_kl) max(s4, 1);   up (+1): s8 > 0 and s8 < fp32(desired_kl / 2) max(s4, 1);
//   otherwise 0 (a NaN, a minibatch without an exps != 0 graph).
// The new lr is formed in double: max(lr_min, lr / 1.5) or min(lr_max, lr * 1.5); 0 leaves lr as it is, even outside
// the bounds.  The model's lr state is double[2][PG_MAX_TENSORS] (one entry per tensor of a table, every entry equal
// without one), flipped with steps_cur: a step reads lr_in and writes every entry of lr_out, so no CTA or block reads an
// entry another one already advanced.  A step that applies nothing (a KL stop, a non-finite step, a peer give-up)
// copies lr_in and leaves the decision slot at 0; so does a frozen tensor's entry.
static_assert(!stat_summed(LR_DECISION_SLOT) && LR_DECISION_SLOT < UPB_STAT_COUNT, "the decision slot is not a sum");
struct AdaptiveLr {
  const double* in;           // NULL: the option is off
  double* out;
  float up, down;             // fp32(desired_kl / 2), fp32(2 desired_kl)
  double lo, hi;              // lr_min, lr_max
};
__device__ __forceinline__ int lr_decision(float s8, float s4, float up, float down) {
  if (kl_exceeds(s8, s4, down)) return -1;
  return s8 > 0.f && s8 < __fmul_rn(up, fmaxf(s4, 1.f)) ? 1 : 0;
}
__device__ __forceinline__ double lr_adapt(double lr, int dec, double lo, double hi) {
  if (dec < 0) return fmax(lo, __ddiv_rn(lr, 1.5));
  if (dec > 0) return fmin(hi, __dmul_rn(lr, 1.5));
  return lr;
}
// a decoupled tensor's factor fp32(1 - lr wd) at the step's lr, formed in double as fill_tensor (upb200.cu) forms it
__device__ __forceinline__ float lr_decay(const ParamGroups* pg, int k, double lr) {
  const double wd = pg->decoupled_wd[k];
  return wd != 0.0 ? (float)__dsub_rn(1.0, __dmul_rn(lr, wd)) : pg->decay[k];
}
// Entry t of the lr state after a step with decision dec that applied Adam (applied) or not; a frozen tensor keeps its lr
__device__ __forceinline__ void lr_write(const AdaptiveLr& al, const ParamGroups* pg, int t, int dec, bool applied) {
  if (t >= PG_MAX_TENSORS) return;
  const bool moves = applied && (pg == nullptr || t >= pg->n || pg->trained[t]);
  al.out[t] = moves ? lr_adapt(al.in[t], dec, al.lo, al.hi) : al.in[t];
}

// ---- global gradient-norm clip (upb_set_max_grad_norm): torch.nn.utils.clip_grad_norm_(parameters(), max_norm) with
// one norm, the same float on every CTA, every rank and both paths.  Its order, defined here once:
//   * a slice partial per 128-column slice of the model's row: the float64 squares of its real-parameter columns (pads,
//     statistics, virtual attention columns and chain-owned columns are 0), added by halving (x[c] += x[c + h] for
//     h = 64, 32, ..., 1): gclip_slice_tree, lane l of a warp holding columns l, l + 32, l + 64, l + 96;
//   * the SGNN: one more partial over the CHAIN_ELEMS attention gradients in the chain's element order i (flat column
//     chain_dst(i)): thread t of a 512-thread block adds i = t, t + 512, t + 1024, t + 1536 in turn, a warp halves its
//     lanes as above, the warps are added in order (gclip_block_tree);
//   * norm = fp32(sqrt(sum of the partials in slice order, the chain last)), in double (gclip_norm);
//   * coef = clamp(max_norm / (norm + 1e-6), max=1) as torch forms it in fp32: torch's scalar / tensor is
//     reciprocal(tensor) * scalar, and a NaN norm gives a NaN coef (gclip_coef).
// The fused tails publish their slice partials as they reduce (sgnn_kernel.cuh: tail_gclip); k_apply recomputes them
// from the flat buffer, where a real parameter's column is its flat index.
constexpr int GCLIP_NORM_SLOT = 17;       // the fp32 pre-clip norm of a step that applied Adam with the clip on
static_assert(!stat_summed(GCLIP_NORM_SLOT) && GCLIP_NORM_SLOT < UPB_STAT_COUNT, "the norm slot is not a sum");
static_assert(stat_summed(KLPEN_SLOT) && KLPEN_SLOT > GCLIP_NORM_SLOT && KLPEN_SLOT < UPB_STAT_COUNT,
              "the KL-penalty slot is a sum beyond the norm");
// ---- non-finite guard (upb_set_nonfinite_guard): a step is bad, and applies nothing, when its globally reduced slot 7
// is not 0 (a NaN there included) or the norm above is not finite.  k_apply evaluates step_nonfinite on the flat buffer;
// the fused tails fold the slot-7 condition into the statistics slice's partial (tail_gclip), so there the norm alone
// carries the same decision.
constexpr int NONFINITE_COUNT_SLOT = 7;   // the step kernels' count of non-finite per-graph results
constexpr int NONFINITE_SLOT = 19;        // 1 in the row of a step the guard skipped
static_assert(!stat_summed(NONFINITE_SLOT) && NONFINITE_SLOT < UPB_STAT_COUNT && stat_summed(NONFINITE_COUNT_SLOT),
              "the guard's slot is not a sum");
__device__ __forceinline__ bool step_nonfinite(float s7, float norm) { return !(s7 == 0.f) || !isfinite(norm); }

constexpr int CHAIN_ELEMS = 1632;         // Wq, Wk, Wv [768] | in_proj_weight [768] | bq, bk, bv [48] | in_proj_bias [48]
constexpr int GCLIP_BLOCK = 512;          // threads of the blocks that form the chain partial (the chain CTA, k_apply)

__device__ __forceinline__ int chain_dst(int i) {
  if (i < 768) return P_ATT_Q_W + (i >> 8) * (P_ATT_K_W - P_ATT_Q_W) + (i & 255);
  if (i < 1536) return P_MHA_IN_W + (i - 768);
  if (i < 1584) return P_ATT_Q_B + ((i - 1536) >> 4) * (P_ATT_K_B - P_ATT_Q_B) + ((i - 1536) & 15);
  return P_MHA_IN_B + (i - 1584);
}

__device__ __forceinline__ double gclip_slice_tree(double x0, double x32, double x64, double x96) {
  double s = (x0 + x64) + (x32 + x96);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);     // halving: the same value in every lane
  return s;
}

// s: this thread's sum of its chain elements; red: shared double[GCLIP_BLOCK / 32].  The partial, in thread 0.
__device__ __forceinline__ double gclip_block_tree(double s, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < GCLIP_BLOCK / 32; ++w) r += red[w];
  return r;
}

__device__ __forceinline__ float gclip_norm(const double* parts, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += parts[i];
  return (float)sqrt(s);
}

__device__ __forceinline__ float gclip_coef(float norm, float max_norm) {
  const float c = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm);
  return c > 1.f ? 1.f : c;                   // torch.clamp(max=1.0): NaN stays NaN
}

// Column `col` of the partial rows summed in the two-call path's fixed order: four accumulators over the rows 0, 1, 2,
// 3 (mod 4) of the first 4 floor(nparts / 4) rows, the remaining rows added to the first, (s0 + s1) + (s2 + s3).
// (mlp_fused_tail reproduces this order for the rl-mlp row: change both together.)
template <class L>
__device__ __forceinline__ float column_sum4(const float* __restrict__ gpart, int nparts, int col) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int c = 0;
  for (; c + 4 <= nparts; c += 4) {
    s0 += gpart[(size_t)(c + 0) * L::row + col];
    s1 += gpart[(size_t)(c + 1) * L::row + col];
    s2 += gpart[(size_t)(c + 2) * L::row + col];
    s3 += gpart[(size_t)(c + 3) * L::row + col];
  }
  for (; c < nparts; ++c) s0 += gpart[(size_t)c * L::row + col];
  return (s0 + s1) + (s2 + s3);
}

// Chain rule of the composed ("virtual") attention projections, thread t < 256 of a block (r = t / 16, c = t % 16):
//   q' = Win_q (Wq hc + bq) + bin_q = Qc hc + qbc   =>  g_Wq = Win_q^T g_Qc,  g_bq = Win_q^T g_qbc,
//   g_Win_q = g_Qc Wq^T + g_qbc bq^T,  g_bin_q = g_qbc;   same for V;  K has no bias gradient (softmax shift
//   invariance, SURVEY A.7).
// Inputs in shared memory: sG = Qc | qbc | Kc | Vc | vbc gradients [816], sWin = in_proj_weight [768], sW = Wq | Wk |
// Wv [768], sB = bq | bk | bv [48].  Projection s (q, k, v) writes gW[s * w_stride + t], gWin[s * 256 + t] and, for
// t < 16, gB[s * b_stride + t], gBin[s * 16 + t].  k_reduce_finish and fused_tail's chain CTA both call this.
__device__ __forceinline__ void attention_chain(int t, const float* sG, const float* sWin, const float* sW,
                                                const float* sB, float* gW, int w_stride, float* gWin, float* gB,
                                                int b_stride, float* gBin) {
  const int r = t >> 4, c = t & 15;
  const int gC[3] = {0, 272, 528};       // offsets inside sG: Qc, Kc, Vc
  const int gBo[3] = {256, -1, 784};     // qbc, -, vbc
#pragma unroll
  for (int s = 0; s < 3; ++s) {
    const float* Win = sWin + s * 256;
    const float* gc = sG + gC[s];
    const float* W = sW + s * 256;
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int rr = 0; rr < 16; ++rr) {
      a = fmaf(Win[rr * 16 + r], gc[rr * 16 + c], a);      // g_W[m=r][c]   = sum_rr Win[rr][m] gC[rr][c]
      b = fmaf(gc[r * 16 + rr], W[c * 16 + rr], b);        // g_Win[r][m=c] = sum_cc gC[r][cc] W[m][cc]
    }
    if (gBo[s] >= 0) b = fmaf(sG[gBo[s] + r], sB[s * 16 + c], b);
    gW[s * w_stride + t] = a;
    gWin[s * 256 + t] = b;
    if (t < 16) {
      float gb = 0.f, gbin = 0.f;
      if (gBo[s] >= 0) {
        for (int rr = 0; rr < 16; ++rr) gb = fmaf(Win[rr * 16 + t], sG[gBo[s] + rr], gb);
        gbin = sG[gBo[s] + t];
      }
      gB[s * b_stride + t] = gb;
      gBin[s * 16 + t] = gbin;
    }
  }
}

// Gradient tail of the SGNN's two-call path, one launch: every block sums its 256 columns of gpart over the CTAs
// (column_sum4: fixed order -> deterministic) and writes them into the flat gradient buffer (write_grad_col); the
// block that finishes last (ticket counter) chains the virtual attention gradients to the six real tensors
// (attention_chain).  grad = [13,729 gradients | 3 pad | 28 statistics] (upb200.h).
constexpr int RF_THREADS = 256;
constexpr int RF_BLOCKS = (G_ROW + RF_THREADS - 1) / RF_THREADS;
static_assert(P_ATT_K_W - P_ATT_Q_W == P_ATT_V_W - P_ATT_K_W && P_ATT_K_B - P_ATT_Q_B == P_ATT_V_B - P_ATT_K_B,
              "q / k / v projections at a fixed stride");

// kl_stop: the stop word (NULL = off); while it is set the step kernel wrote no partial rows, and grad becomes the
// skipped step's row.  pg: the parameter groups (NULL = none): a frozen tensor's columns of grad are 0 (gsum, which the
// chain reads, keeps the sums).
__global__ void __launch_bounds__(RF_THREADS) k_reduce_finish(const float* __restrict__ gpart, int nparts,
                                                              float* __restrict__ gsum, const float* __restrict__ P,
                                                              float* __restrict__ grad, unsigned int* ticket,
                                                              const unsigned int* kl_stop, const ParamGroups* pg) {
  __shared__ float sG[816];        // Qc | qbc | Kc | Vc | vbc gradients
  __shared__ float sWin[768];      // in_proj_weight
  __shared__ float sW[768];        // Wq | Wk | Wv
  __shared__ float sB[48];         // bq | bk | bv
  __shared__ bool is_last;
  const int t = threadIdx.x;
  const int idx = blockIdx.x * RF_THREADS + t;
  if (kl_stop && kl_stop_set(kl_stop)) {           // every block returns: the ticket is not touched
    if (idx < UPB_GRAD_STRIDE) write_skip_elem(grad, UPB_STAT_OFFSET, idx);
    return;
  }
  if (idx < G_ROW) {
    const float v = column_sum4<SgnnRow>(gpart, nparts, idx);
    gsum[idx] = v;
    write_grad_col<SgnnRow>(grad, idx, pg && idx < NUM_PARAMS && pg_frozen(pg, idx) ? 0.f : v);
  }
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (t == 0) *ticket = 0u;        // ready for the next launch
  for (int i = t; i < 816; i += RF_THREADS) sG[i] = __ldcg(gsum + G_QC + i);
  for (int i = t; i < 768; i += RF_THREADS) sWin[i] = P[P_MHA_IN_W + i];
  sW[t] = P[P_ATT_Q_W + t];
  sW[256 + t] = P[P_ATT_K_W + t];
  sW[512 + t] = P[P_ATT_V_W + t];
  if (t < 16) { sB[t] = P[P_ATT_Q_B + t]; sB[16 + t] = P[P_ATT_K_B + t]; sB[32 + t] = P[P_ATT_V_B + t]; }
  __syncthreads();
  attention_chain(t, sG, sWin, sW, sB, grad + P_ATT_Q_W, P_ATT_K_W - P_ATT_Q_W, grad + P_MHA_IN_W, grad + P_ATT_Q_B,
                  P_ATT_K_B - P_ATT_Q_B, grad + P_MHA_IN_B);
  if (pg) {
    __syncthreads();               // the chain's writes of this block are visible to it
    for (int i = t; i < CHAIN_ELEMS; i += RF_THREADS)
      if (pg_frozen(pg, chain_dst(i))) grad[chain_dst(i)] = 0.f;
  }
}

// ---- gradient noise scale (upb_ppo_grad_noise): McCandlish et al.'s two-batch estimator on one two-call gradient
// launch, whose per-CTA partial rows are the small batches and whose reduced row is the big one.  One block per partial
// row c forms |G_c|^2 over the trained real parameters (the SGNN's virtual attention columns chained to the six real
// tensors on the row itself, attention_chain), one more block |g|^2 over the same columns of the reduced flat buffer;
// float64 squares summed in a fixed order (per-thread strided sums, a fixed shuffle tree, the warps in order), and the
// block that finishes last (ticket counter) adds the row sums in row order.  Frozen tensors (pg), pads, statistics and
// virtual columns are never counted.  out = {A = sum_c |G_c|^2, S = |g|^2, Q = sum_c n_c^2, N = count}, where CTA c of
// the launch's nparts = min(count, grid) CTAs took the items c, c + nparts, ... (n_c = count / nparts, one more for
// c < count % nparts).  While the stop word is set the launch wrote no partial rows: out = {0, 0, 0, 0} (no sample).
// Deterministic.
constexpr int GNS_THREADS = 256;
static_assert(GNS_THREADS == RF_THREADS, "attention_chain runs on the reduction's 256 threads");

__device__ __forceinline__ double gns_block_sum(double s, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  double r = 0.0;
  for (int w = 0; w < GNS_THREADS / 32; ++w) r += red[w];
  return r;
}

// thread t's share of the squared chained attention gradients of the SGNN partial row `row`, over the trained chain
// elements (k_reduce_finish's chain, on one row instead of the column sums)
__device__ __forceinline__ double gns_row_chain(const float* __restrict__ row, const float* __restrict__ P,
                                                const ParamGroups* pg, int t) {
  __shared__ float sG[816];        // Qc | qbc | Kc | Vc | vbc gradients
  __shared__ float sWin[768];      // in_proj_weight
  __shared__ float sW[768];        // Wq | Wk | Wv
  __shared__ float sB[48];         // bq | bk | bv
  __shared__ float sC[CHAIN_ELEMS];  // the chained gradients in the chain's element order (chain_dst)
  for (int i = t; i < 816; i += GNS_THREADS) sG[i] = row[G_QC + i];
  for (int i = t; i < 768; i += GNS_THREADS) sWin[i] = P[P_MHA_IN_W + i];
  sW[t] = P[P_ATT_Q_W + t];
  sW[256 + t] = P[P_ATT_K_W + t];
  sW[512 + t] = P[P_ATT_V_W + t];
  if (t < 16) { sB[t] = P[P_ATT_Q_B + t]; sB[16 + t] = P[P_ATT_K_B + t]; sB[32 + t] = P[P_ATT_V_B + t]; }
  __syncthreads();
  attention_chain(t, sG, sWin, sW, sB, sC, 256, sC + 768, sC + 1536, 16, sC + 1584);
  __syncthreads();
  double s = 0.0;
  for (int i = t; i < CHAIN_ELEMS; i += GNS_THREADS)
    if (!(pg && pg_frozen(pg, chain_dst(i)))) { const double x = (double)sC[i]; s += x * x; }
  return s;
}

// gridDim.x = nparts + 1; part: double[nparts + 1] scratch; ticket: a counter at 0, left at 0
template <class L>
__global__ void __launch_bounds__(GNS_THREADS) k_grad_noise(const float* __restrict__ gpart, int nparts,
                                                            const float* __restrict__ grad, const float* __restrict__ P,
                                                            const unsigned int* kl_stop, const ParamGroups* pg,
                                                            int count, double* part, unsigned int* ticket,
                                                            double* __restrict__ out) {
  __shared__ double red[GNS_THREADS / 32];
  __shared__ bool is_last;
  const int t = threadIdx.x, b = blockIdx.x;
  if (kl_stop && kl_stop_set(kl_stop)) {           // every block returns: the ticket is not touched
    if (b == 0 && t < 4) out[t] = 0.0;
    return;
  }
  double s = 0.0;
  if (b < nparts) {
    const float* row = gpart + (size_t)b * L::row;
    for (int col = t; col < L::num_params; col += GNS_THREADS)
      if (!chain_owns<L>(col) && !(pg && pg_frozen(pg, col))) { const double x = (double)row[col]; s += x * x; }
    if constexpr (L::chain0_end > L::chain0_begin) s += gns_row_chain(row, P, pg, t);
  } else {                          // the reduced row: the chain already wrote its real attention columns
    for (int col = t; col < L::num_params; col += GNS_THREADS)
      if (!(pg && pg_frozen(pg, col))) { const double x = (double)grad[col]; s += x * x; }
  }
  s = gns_block_sum(s, red);
  if (t == 0) part[b] = s;
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last || t != 0) return;
  __threadfence();
  *ticket = 0u;                    // ready for the next launch
  double A = 0.0;
  for (int c = 0; c < nparts; ++c) A += __ldcg(part + c);
  double Q = 0.0;
  if (nparts > 0) {
    const double q = (double)(count / nparts), r = (double)(count % nparts);
    Q = r * (q + 1.0) * (q + 1.0) + ((double)nparts - r) * q * q;
  }
  out[0] = A;
  out[1] = __ldcg(part + nparts);
  out[2] = Q;
  out[3] = (double)count;
}

struct ApplyArgs {
  float* params;
  float* grad;                // [UPB_GRAD_STRIDE]; only the stop slot, the clip's norm slot and the guard's slot are written
  float* m;
  float* v;
  const long long* steps_in;  // [4] global, encoder+value, land-use head, road head
  long long* steps_out;       // [4] written by block 0 (ping-pong with steps_in across calls)
  double lr;                  // a double, as torch keeps it: the step size is (float)(lr / bias_correction1) (upb_set_lr)
  float beta1, beta2, eps;
  float weight_decay;         // Adam's coupled L2 term (upb_set_weight_decay); 0 = off
  int clip_now;               // 1: two-group clip on this step (decided on the host: mode + first-step latch)
  // flat layout of the model being updated (SGNN: layout.h; rl-mlp: mlp_kernel.cuh)
  int num_params, encoder_end, policy_end, lu_begin, rd_begin, stat_offset;
  unsigned int* kl_stop;      // the model's stop word (NULL: the KL stop is off)
  float kl_limit;
  float max_norm;             // global gradient-norm clip (upb_set_max_grad_norm); 0 = off
  int nslice;                 // the model's row in SLICE-column slices and its chain-owned columns (layout.h), for the
  int chain0_begin, chain0_end, chain1_begin, chain1_end;     // norm's order
  int nonfinite_guard;        // 1: a step that is not finite applies nothing (upb_set_nonfinite_guard)
  // parameter groups (upb_set_param_groups; NULL = none): each tensor's lr, weight decay and trained flag replace lr and
  // weight_decay above, and its own count (tsteps_in -> tsteps_out, written by block 0) its segment's in the bias
  // corrections
  const ParamGroups* pg;
  const long long* tsteps_in;
  long long* tsteps_out;
  // EWMA proximal parameters (upb_set_prox_ewma; NULL = off): every element after a step that applied Adam
  float* prox;
  float prox_beta;
};

constexpr int AP_THREADS = 512;
constexpr int AP_PER_THREAD = 2;
constexpr int AP_BLOCKS = (NUM_PARAMS + AP_THREADS * AP_PER_THREAD - 1) / (AP_THREADS * AP_PER_THREAD);

__device__ __forceinline__ float block_sum_ap(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < AP_THREADS / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

// The global clip's norm of the flat gradient buffer, in gclip_norm's order, computed by every block: warp w forms the
// partials of the slices w, w + 16, ..., the block the chain partial (the SGNN), thread 0 the sum.
static_assert(AP_THREADS == GCLIP_BLOCK, "k_apply forms the chain partial with the chain CTA's tree");
constexpr int GCLIP_MAX_PARTS = 128;
__device__ __noinline__ float apply_gclip_norm(const ApplyArgs& a) {
  __shared__ double parts[GCLIP_MAX_PARTS];
  __shared__ double red[GCLIP_BLOCK / 32];
  __shared__ float norm;
  const int t = threadIdx.x, lane = t & 31;
  for (int sl = t >> 5; sl < a.nslice; sl += AP_THREADS / 32) {
    double x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int col = sl * SLICE + lane + 32 * k;
      const bool real = col < a.num_params && !(col >= a.chain0_begin && col < a.chain0_end) &&
                        !(col >= a.chain1_begin && col < a.chain1_end);
      const double g = real ? (double)a.grad[col] : 0.0;
      x[k] = g * g;
    }
    const double p = gclip_slice_tree(x[0], x[1], x[2], x[3]);
    if (lane == 0) parts[sl] = p;
  }
  const bool chain = a.chain0_end > a.chain0_begin;
  int n = a.nslice;
  if (chain) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = t + j * AP_THREADS;
      if (i < CHAIN_ELEMS) { const double g = (double)a.grad[chain_dst(i)]; s += g * g; }
    }
    s = gclip_block_tree(s, red);           // barrier inside: the slice partials are in place too
    if (t == 0) parts[n] = s;
    ++n;
  }
  __syncthreads();
  if (t == 0) norm = gclip_norm(parts, n);
  __syncthreads();
  return norm;
}

// A step of k_apply that applies nothing, thread t of block 0: the lr state is copied and the decision slot cleared (a
// buffer applied a second time may carry an earlier decision)
__device__ __noinline__ void apply_keep_lr(const ApplyArgs& a, const AdaptiveLr& alr, int t) {
  lr_write(alr, a.pg, t, 0, false);
  if (t == 0) a.grad[a.stat_offset + LR_DECISION_SLOT] = 0.f;
}

// A step of k_apply that applies Adam with the KL-adaptive lr on: every block takes the same decision from the same
// slots, re-forms the step sizes (sh: [seg][step size, sqrt(bc2)]; pg_adam: [step size, sqrt(bc2), decay][tensor])
// k_apply staged from lr / pg->lr with the new lr, and block 0 writes the lr state and the decision slot.
__device__ __noinline__ void apply_adapt_lr(const ApplyArgs& a, const AdaptiveLr& alr, bool live_lu, bool live_rd,
                                            float* sh, float (*pg_adam)[PG_MAX_TENSORS]) {
  const int t = threadIdx.x;
  const float* st = a.grad + a.stat_offset;
  const int dec = lr_decision(st[8], st[4], alr.up, alr.down);
  if (t < 3) {
    const bool live = t == 0 ? true : (t == 1 ? live_lu : live_rd);
    const long long stp = a.steps_in[1 + t] + (live ? 1 : 0);
    const double bc1 = 1.0 - ipow((double)a.beta1, stp > 0 ? stp : 1);
    sh[t * 2 + 0] = (float)(lr_adapt(alr.in[0], dec, alr.lo, alr.hi) / bc1);
  }
  if (a.pg && t < a.pg->n) {
    const int s = a.pg->seg[t];
    const bool live = a.pg->trained[t] && (s == 0 || (s == 1 ? live_lu : live_rd));
    const long long stp = a.tsteps_in[t] + (live ? 1 : 0);
    const double bc1 = 1.0 - ipow((double)a.pg->beta1[t], stp > 0 ? stp : 1);
    const double lr = lr_adapt(alr.in[t], dec, alr.lo, alr.hi);
    pg_adam[0][t] = (float)(lr / bc1);
    pg_adam[2][t] = lr_decay(a.pg, t, lr);
  }
  if (blockIdx.x == 0) {
    lr_write(alr, a.pg, t, dec, true);
    if (t == 0) a.grad[a.stat_offset + LR_DECISION_SLOT] = (float)dec;    // no block reads this slot
  }
}

// clip_policy_grad (agent_ppo.py:43-46: clip_grad_norm_(policy params, 1) then clip_grad_norm_(value params, 1);
// the shared encoder is in both groups) followed by torch.optim.Adam.step (urban_planning_agent.py:145-149,337),
// weight decay included.
// Several blocks: each one recomputes the (rarely needed) clip norms itself, so there is no inter-block
// dependency; step counters are read from steps_in and written to steps_out.  ALR: the KL-adaptive lr is on
// (upb_set_adaptive_lr; alr.in != NULL), whose lr state replaces lr / pg->lr: an instantiation of its own, so that the
// option adds nothing to k_apply<false>.
template <bool ALR>
__global__ void __launch_bounds__(AP_THREADS) k_apply(const ApplyArgs a, const AdaptiveLr alr) {
  __shared__ float red[AP_THREADS / 32];
  __shared__ float sh[8];
  const int t = threadIdx.x;
  const float* st = a.grad + a.stat_offset;
  if (a.kl_stop) {
    // No parameter, moment or counter changes while the stop word is set, nor on the step whose statistics pass the
    // criterion; that step's block 0 sets the word and marks the row.  Every thread of a block has read the word
    // before block 0 writes it; another block may see block 0's write, which leads it to the same skip.
    __shared__ unsigned int word;
    if (t == 0) word = kl_stop_set(a.kl_stop) ? 1u : 0u;
    __syncthreads();
    const bool skip = word != 0u;
    if (skip || kl_exceeds(st[8], st[4], a.kl_limit)) {
      if (blockIdx.x == 0) {
        if (t < 4) a.steps_out[t] = a.steps_in[t];
        if (a.pg) pg_keep_steps(a.pg, a.tsteps_in, a.tsteps_out, t);
        if (t == 0 && !skip) { a.grad[a.stat_offset + KL_STOP_SLOT] = 1.f; *a.kl_stop = 1u; }
        if constexpr (ALR) apply_keep_lr(a, alr, t);
      }
      return;
    }
  }
  float gnorm = 0.f;
  if (a.nonfinite_guard) {
    // Every block forms the same norm and reads the same slot 7, so all take the same decision; it comes before either
    // clip's coefficients are used.  A bad step changes no parameter, moment or counter and marks the row.
    gnorm = apply_gclip_norm(a);
    if (step_nonfinite(st[NONFINITE_COUNT_SLOT], gnorm)) {
      if (blockIdx.x == 0) {
        if (t < 4) a.steps_out[t] = a.steps_in[t];
        if (a.pg) pg_keep_steps(a.pg, a.tsteps_in, a.tsteps_out, t);
        if (t == 0) a.grad[a.stat_offset + NONFINITE_SLOT] = 1.f;      // no block reads this slot
        if constexpr (ALR) apply_keep_lr(a, alr, t);
      }
      return;
    }
    // a buffer applied a second time may still carry an earlier decision's mark
    if (blockIdx.x == 0 && t == 0) a.grad[a.stat_offset + NONFINITE_SLOT] = 0.f;
  }
  const bool live_lu = st[5] > 0.f, live_rd = st[6] > 0.f;
  const long long gstep = a.steps_in[0];
  const bool do_clip = a.clip_now != 0;
  float c_enc = 1.f, c_pol = 1.f, c_val = 1.f;
  if (do_clip) {
    float se = 0.f, sp = 0.f, sv = 0.f;
    for (int i = t; i < a.num_params; i += AP_THREADS) {
      const float g = a.grad[i];
      if (i < a.encoder_end) se += g * g;
      else if (i < a.policy_end) sp += g * g;
      else sv += g * g;
    }
    se = block_sum_ap(se, red);
    sp = block_sum_ap(sp, red);
    sv = block_sum_ap(sv, red);
    const float n1 = sqrtf(se + sp);
    const float k1 = fminf(1.f / (n1 + 1e-6f), 1.f);               // policy group
    const float n2 = sqrtf(k1 * k1 * se + sv);
    const float k2 = fminf(1.f / (n2 + 1e-6f), 1.f);               // value group, encoder already scaled
    c_enc = k1 * k2; c_pol = k1; c_val = k2;
  }
  if (a.max_norm > 0.f) {         // one group (the host keeps it exclusive with the two-group clip above)
    const float norm = a.nonfinite_guard ? gnorm : apply_gclip_norm(a);
    c_enc = c_pol = c_val = gclip_coef(norm, a.max_norm);
    if (blockIdx.x == 0 && t == 0) a.grad[a.stat_offset + GCLIP_NORM_SLOT] = norm;   // no block reads this slot
  }
  if (t < 3) {
    // per-segment Adam step counts: a head whose stage is absent has grad None and is skipped entirely
    const bool live = t == 0 ? true : (t == 1 ? live_lu : live_rd);
    const long long stp = a.steps_in[1 + t] + (live ? 1 : 0);
    const double bc1 = 1.0 - ipow((double)a.beta1, stp > 0 ? stp : 1);
    const double bc2 = 1.0 - ipow((double)a.beta2, stp > 0 ? stp : 1);
    sh[t * 2 + 0] = (float)(a.lr / bc1);
    sh[t * 2 + 1] = (float)sqrt(bc2);
    if (blockIdx.x == 0) a.steps_out[1 + t] = stp;
  }
  if (blockIdx.x == 0 && t == 3) a.steps_out[0] = gstep + 1;
  // per-tensor step sizes with a table: a tensor steps when it is trained and its segment is live
  __shared__ float pg_adam[3][PG_MAX_TENSORS];     // step size, sqrt(bias_correction2) at the tensor's betas, decay
  __shared__ int pg_live[PG_MAX_TENSORS];
  if (a.pg && t < a.pg->n) {
    const int s = a.pg->seg[t];
    const bool live = a.pg->trained[t] && (s == 0 || (s == 1 ? live_lu : live_rd));
    const long long stp = a.tsteps_in[t] + (live ? 1 : 0);
    const double bc1 = 1.0 - ipow((double)a.pg->beta1[t], stp > 0 ? stp : 1);
    const double bc2 = 1.0 - ipow((double)a.pg->beta2[t], stp > 0 ? stp : 1);
    pg_adam[0][t] = (float)(a.pg->lr[t] / bc1);
    pg_adam[1][t] = (float)sqrt(bc2);
    pg_adam[2][t] = a.pg->decay[t];
    pg_live[t] = live;
    if (blockIdx.x == 0) a.tsteps_out[t] = stp;
  }
  if constexpr (ALR) apply_adapt_lr(a, alr, live_lu, live_rd, sh, pg_adam);
  __syncthreads();
  const float w1 = 1.f - a.beta1, w2 = 1.f - a.beta2;
#pragma unroll
  for (int j = 0; j < AP_PER_THREAD; ++j) {
    const int i = (blockIdx.x * AP_PER_THREAD + j) * AP_THREADS + t;
    if (i >= a.num_params) break;
    int seg = 0;
    bool live = true;
    const float coef = i < a.encoder_end ? c_enc : (i < a.policy_end ? c_pol : c_val);
    if (i >= a.lu_begin && i < a.rd_begin) { seg = 1; live = live_lu; }
    else if (i >= a.rd_begin && i < a.policy_end) { seg = 2; live = live_rd; }
    if (a.pg) {
      const int k = a.pg->tensor_of[i];
      if (pg_live[k]) {
        const float p = pg_adam_step(a.pg, k, i, __fmul_rn(a.grad[i], coef), pg_adam[0][k], pg_adam[1][k],
                                     pg_adam[2][k], a.params, a.m, a.v);
        if (a.prox) prox_ewma_elem(a.prox, a.prox_beta, i, p);
      } else if (a.prox) {
        prox_ewma_elem(a.prox, a.prox_beta, i, a.params[i]);
      }
      continue;
    }
    const float step_size = sh[seg * 2 + 0], bc2_sqrt = sh[seg * 2 + 1], wd = a.weight_decay;
    if (!live) {
      if (a.prox) prox_ewma_elem(a.prox, a.prox_beta, i, a.params[i]);
      continue;
    }
    const float p = a.params[i];
    float g = __fmul_rn(a.grad[i], coef);
    // grad.add(param, alpha=weight_decay) inside Adam.step, after the clip: the clip norms never see the decay term.
    // Skipped at 0 so that -0 gradients and non-finite parameters keep the undecayed arithmetic.
    if (wd != 0.f) g = __fmaf_rn(wd, p, g);
    float m = a.m[i], v = a.v[i];
    m = __fadd_rn(m, __fmul_rn(w1, __fsub_rn(g, m)));                           // lerp_(grad, 1-beta1)
    v = __fadd_rn(__fmul_rn(v, a.beta2), __fmul_rn(__fmul_rn(w2, g), g));       // mul_(beta2).addcmul_(g, g, 1-beta2)
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), a.eps);
    const float pn = __fadd_rn(p, __fmul_rn(-step_size, __fdiv_rn(m, denom)));
    a.params[i] = pn;
    a.m[i] = m;
    a.v[i] = v;
    if (a.prox) prox_ewma_elem(a.prox, a.prox_beta, i, pn);
  }
}

// Squared L2 norms of whole gradient-buffer rows over the three groups k_apply clips by: out[row] = sums of g^2 over the
// shared encoder [0, encoder_end), the policy heads [encoder_end, policy_end) and the value head [policy_end, num_params).
// One block per row; float64 sums in a fixed order (per-thread strided sums, then a fixed shuffle tree and the warps in
// order), so the result is deterministic.
constexpr int GN_THREADS = 256;
static_assert(STATS_USED <= UPB_STAT_COUNT && G_STATS + UPB_STAT_COUNT <= G_ROW, "statistics fit the rows");

__global__ void __launch_bounds__(GN_THREADS) k_grad_norms(const float* __restrict__ rows, int stride, int num_params,
                                                           int encoder_end, int policy_end, float* __restrict__ out) {
  __shared__ double red[3][GN_THREADS / 32];
  const float* g = rows + (size_t)blockIdx.x * stride;
  const int t = threadIdx.x;
  double se = 0.0, sp = 0.0, sv = 0.0;
  for (int i = t; i < num_params; i += GN_THREADS) {
    const double x = (double)g[i];
    if (i < encoder_end) se = fma(x, x, se);
    else if (i < policy_end) sp = fma(x, x, sp);
    else sv = fma(x, x, sv);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sp += __shfl_xor_sync(0xffffffffu, sp, o);
    sv += __shfl_xor_sync(0xffffffffu, sv, o);
  }
  if ((t & 31) == 0) { red[0][t >> 5] = se; red[1][t >> 5] = sp; red[2][t >> 5] = sv; }
  __syncthreads();
  if (t < 3) {
    double s = 0.0;
    for (int w = 0; w < GN_THREADS / 32; ++w) s += red[t][w];
    out[(size_t)blockIdx.x * 3 + t] = (float)s;
  }
}

// Per-minibatch advantage normalisation (Stable-Baselines3's normalize_advantage, CleanRL's norm_adv), one block per
// minibatch b = order[b B, (b + 1) B) of an epoch: the mean and the unbiased standard deviation of the advantages of its
// graphs with exps != 0, accumulated in float64 in a fixed order (per-thread strided sums, a fixed shuffle tree, the
// warps in order; two passes) and each rounded once to fp32, then out = (A - mean) / (std + 1e-8) in fp32 for every
// graph of the minibatch.  Fewer than two such graphs: the advantages are copied unchanged.  Deterministic.
constexpr int AN_THREADS = 256;

__device__ __forceinline__ double block_sum_an(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < AN_THREADS / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(AN_THREADS) k_adv_norm(const float* __restrict__ adv_in, const float* __restrict__ exps,
                                                         const int* __restrict__ order, int B,
                                                         float* __restrict__ adv_out) {
  __shared__ double red[AN_THREADS / 32];
  const int* ids = order + (size_t)blockIdx.x * B;
  const int t = threadIdx.x;
  double s = 0.0, n = 0.0;
  for (int i = t; i < B; i += AN_THREADS) {
    const int g = ids[i];
    if (exps[g] != 0.f) { s += (double)adv_in[g]; n += 1.0; }
  }
  s = block_sum_an(s, red);
  n = block_sum_an(n, red);
  float mean = 0.f, den = 1.f;
  const bool norm = n >= 2.0;
  if (norm) {
    const double mu = s / n;
    double q = 0.0;
    for (int i = t; i < B; i += AN_THREADS) {
      const int g = ids[i];
      if (exps[g] != 0.f) { const double d = (double)adv_in[g] - mu; q = fma(d, d, q); }
    }
    q = block_sum_an(q, red);
    mean = (float)mu;
    den = __fadd_rn((float)sqrt(q / (n - 1.0)), 1e-8f);
  }
  for (int i = t; i < B; i += AN_THREADS) {
    const int g = ids[i];
    const float A = adv_in[g];
    adv_out[g] = norm ? __fdiv_rn(__fsub_rn(A, mean), den) : A;
  }
}

// ---- value-target normalisation (upb_set_value_norm): MAPPO's ValueNorm (per_element_update=False) with PopArt's
// output-preserving rescale of the value head's last layer.  The running state is three doubles {m1, m2, d} per model.
// Every product and sum below is an explicit round-to-nearest double operation (no contraction into fma), so a float64
// host replay in the same order gives the same bits.
struct VnStats {
  double mean, std;
};

__device__ __forceinline__ VnStats vnorm_stats(double m1, double m2, double d) {
  if (d == 0.0) return {0.0, 1.0};
  const double dd = fmax(d, 1e-5);
  const double mu = __ddiv_rn(m1, dd);
  const double var = __dsub_rn(__ddiv_rn(m2, dd), __dmul_rn(mu, mu));
  return {mu, __dsqrt_rn(fmax(var, 1e-2))};
}

// out[i] = fmaf(fp32(std), n[i], fp32(mean)) with the statistics of `state`; with d == 0 (identity) out[i] = n[i].
__global__ void __launch_bounds__(256) k_value_denorm(const float* __restrict__ n, int T, const double* __restrict__ state,
                                                      float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T) return;
  const double d = state[2];
  const VnStats s = vnorm_stats(state[0], state[1], d);
  out[i] = d == 0.0 ? n[i] : __fmaf_rn((float)s.std, n[i], (float)s.mean);
}

// One block of AN_THREADS over all T returns: b1 = sum R / T and b2 = sum R^2 / T in float64 in block_sum_an's fixed
// order; if every R is finite, the state moves to beta * state + (1 - beta) * (b1, b2, 1), else it is kept.  With the old
// statistics (mo, so) and the new ones (mn, sn), and only when the state moved, the value head's last layer is rescaled
// in place: w2 <- fp32((w2 * so) / sn), b2 <- fp32(((so * b2 + mo) - mn) / sn), in double from the fp32 values.  Then
// R' = (R - fp32(mn)) / fp32(sn) in fp32, and V' likewise when V is not NULL.  mean_std (may be NULL) receives (mn, sn).
// Deterministic: one block, a fixed order.
__global__ void __launch_bounds__(AN_THREADS) k_value_norm(const float* __restrict__ R, const float* __restrict__ V,
                                                           int T, double* state, double beta, float* params, int w2,
                                                           int b2, float* __restrict__ R_out, float* __restrict__ V_out,
                                                           double* mean_std) {
  __shared__ double red[AN_THREADS / 32];
  const int t = threadIdx.x;
  double s1 = 0.0, s2 = 0.0;
  bool bad = false;
  for (int i = t; i < T; i += AN_THREADS) {
    const double r = (double)R[i];
    bad |= !isfinite(r);
    s1 = __dadd_rn(s1, r);
    s2 = __dadd_rn(s2, __dmul_rn(r, r));
  }
  s1 = block_sum_an(s1, red);
  s2 = block_sum_an(s2, red);
  const bool moved = !__syncthreads_or(bad);        // the barrier also orders every thread's state read before the write
  const double m1 = state[0], m2 = state[1], d = state[2];
  const VnStats so = vnorm_stats(m1, m2, d);
  VnStats sn = so;
  if (moved) {
    const double b1 = __ddiv_rn(s1, (double)T), bq = __ddiv_rn(s2, (double)T), w = __dsub_rn(1.0, beta);
    const double n1 = __dadd_rn(__dmul_rn(beta, m1), __dmul_rn(w, b1));
    const double n2 = __dadd_rn(__dmul_rn(beta, m2), __dmul_rn(w, bq));
    const double nd = __dadd_rn(__dmul_rn(beta, d), w);
    sn = vnorm_stats(n1, n2, nd);
    __syncthreads();
    if (t == 0) { state[0] = n1; state[1] = n2; state[2] = nd; }
    if (t < 32) params[w2 + t] = (float)__ddiv_rn(__dmul_rn((double)params[w2 + t], so.std), sn.std);
    if (t == 32)
      params[b2] = (float)__ddiv_rn(__dsub_rn(__dadd_rn(__dmul_rn(so.std, (double)params[b2]), so.mean), sn.mean), sn.std);
  }
  if (t == 0 && mean_std) { mean_std[0] = sn.mean; mean_std[1] = sn.std; }
  const float mu = (float)sn.mean, sd = (float)sn.std;
  for (int i = t; i < T; i += AN_THREADS) {
    R_out[i] = __fdiv_rn(__fsub_rn(R[i], mu), sd);
    if (V) V_out[i] = __fdiv_rn(__fsub_rn(V[i], mu), sd);
  }
}

// estimate_advantages (khrylib/rl/core/common.py:5-26).  The recurrence only chains inside an episode
// (masks[i] == 0 at its last step), so one thread walks one episode backwards with the reference's exact fp32
// operation order; episodes run in parallel.  That order is exact for finite inputs only: a non-finite advantage stays
// in its episode here, where the reference's whole-buffer scan forms prev_advantage * 0 = NaN at the boundary and
// carries it to every earlier sample (the non-finite guard relies on this containment).
__global__ void __launch_bounds__(256) k_gae(const float* __restrict__ rewards, const float* __restrict__ masks,
                                             const float* __restrict__ values, int T, float gamma, float gamma_tau,
                                             float* __restrict__ adv, float* __restrict__ ret) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T) return;
  if (!(i == T - 1 || masks[i] == 0.f)) return;       // not the last step of a segment
  float prev_v = 0.f, prev_a = 0.f;
  if (masks[i] != 0.f) { prev_v = 0.f; prev_a = 0.f; } // i == T-1: the scan starts from zeros
  for (int j = i; j >= 0; --j) {
    const float mk = masks[j];
    if (j != i && mk == 0.f) break;                    // previous segment
    const float vj = values[j];
    float d = __fmul_rn(__fmul_rn(gamma, prev_v), mk);
    d = __fsub_rn(__fadd_rn(rewards[j], d), vj);
    const float aj = __fadd_rn(d, __fmul_rn(__fmul_rn(gamma_tau, prev_a), mk));
    adv[j] = aj;
    ret[j] = __fadd_rn(vj, aj);
    prev_v = vj;
    prev_a = aj;
  }
}

// The targets of one more epoch from the value head's raw outputs `head` (upb_gae_targets): k_gae's walk and arithmetic
// on the values V, writing the advantages adv (reward units), the returns ret the steps train on and the value-clip
// anchor (= head).  state NULL (value normalisation off): V = head and ret = R, k_gae exactly.  Otherwise, with the
// model's current statistics (mean, std) of `state`, which this kernel does not move: V = fmaf(fp32 std, head, fp32 mean)
// as k_value_denorm forms it (V = head while d == 0), and ret = (R - fp32 mean) / fp32 std as k_value_norm forms it.
__global__ void __launch_bounds__(256) k_gae_targets(const float* __restrict__ rewards, const float* __restrict__ masks,
                                                     const float* __restrict__ head, int T, float gamma, float gamma_tau,
                                                     const double* __restrict__ state, float* __restrict__ adv,
                                                     float* __restrict__ ret, float* __restrict__ anchor) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T) return;
  if (!(i == T - 1 || masks[i] == 0.f)) return;       // not the last step of a segment
  float mu = 0.f, sd = 1.f;
  bool denorm = false;
  if (state) {
    const VnStats s = vnorm_stats(state[0], state[1], state[2]);
    mu = (float)s.mean;
    sd = (float)s.std;
    denorm = state[2] != 0.0;
  }
  float prev_v = 0.f, prev_a = 0.f;
  for (int j = i; j >= 0; --j) {
    const float mk = masks[j];
    if (j != i && mk == 0.f) break;                    // previous segment
    const float nj = head[j];
    const float vj = denorm ? __fmaf_rn(sd, nj, mu) : nj;
    float d = __fmul_rn(__fmul_rn(gamma, prev_v), mk);
    d = __fsub_rn(__fadd_rn(rewards[j], d), vj);
    const float aj = __fadd_rn(d, __fmul_rn(__fmul_rn(gamma_tau, prev_a), mk));
    const float Rj = __fadd_rn(vj, aj);
    adv[j] = aj;
    ret[j] = state ? __fdiv_rn(__fsub_rn(Rj, mu), sd) : Rj;
    anchor[j] = nj;
    prev_v = vj;
    prev_a = aj;
  }
}

}  // namespace upb
