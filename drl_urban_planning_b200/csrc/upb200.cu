// C-ABI implementation (include/upb200.h): context, launches, optimiser state.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/upb200.h"
#include "blob.h"
#include "errors.h"
#include "layout.h"
#include "optim_kernels.cuh"
#include "sgnn_kernel.cuh"
#include "mlp_kernel.cuh"

using namespace upb;

// One model (SGNN or rl-mlp) of a context: a constant description of its kernels and flat layout, and its own
// per-CTA partial rows, scratch, Adam state, step counters and first-step clip latch.  Every entry point of the C ABI
// exists once per model and runs the same code on the model's record.
struct Model {
  void (*train)(StepArgs);             // k_sgnn<true> / k_mlp<true>
  void (*infer)(StepArgs);
  int threads;
  size_t smem;
  int row;                             // floats per partial gradient row
  int num_params, encoder_end, policy_end, lu_begin, rd_begin, stat_offset, grad_stride;
  size_t (*scratch_floats)(int n_cap, int e_cap);
  void (*reduce)(const upb_ctx* ctx, int nparts, const float* params, float* grad, const unsigned int* kl_stop,
                 cudaStream_t s);     // two-call path
  bool peer_exchange;                  // the fused step adds the peers' gradients in the kernel
  int chain0_begin, chain0_end, chain1_begin, chain1_end;     // chain-owned columns (layout.h), for the global clip
  void (*train_gclip)(StepArgs);       // the fused step with the global clip or the non-finite guard on: k_sgnn_gclip /
                                       // k_mlp_gclip
  int val_w2, val_b2;                  // the value head's last layer, rescaled by upb_value_norm_update
  void (*train_pg)(StepArgs);          // the fused step with parameter groups: k_sgnn_pg / k_mlp_pg
  const int* tensor_offsets;           // [tensors + 1]: each tensor's first column (upb_param_slot order), then num_params
  int num_tensors;
  void (*values)(StepArgs);            // the value-only sweep (upb_values): k_sgnn_values / k_mlp_values

  float* gpart = nullptr;              // [grid][row]
  float* scratch = nullptr;            // [grid][scratch_stride]
  size_t scratch_stride = 0;
  float* adam_m = nullptr;
  float* adam_v = nullptr;
  long long* steps = nullptr;          // device [2][4] ping-pong step counters
  unsigned int* kl_stop = nullptr;     // device stop word of the KL stop (upb_set_target_kl, upb_reset_kl_stop)
  double* vnorm = nullptr;             // device {m1, m2, d}: the value-target normaliser's running state (upb_set_value_norm)
  int steps_cur = 0;
  bool clip_armed = true;              // UPB_CLIP_REFERENCE: the next step is the process's first one and clips (SURVEY A.6-2)
  ParamGroups* pg = nullptr;           // the table the launches read (pg_mem), NULL = none
  ParamGroups* pg_mem = nullptr;       // device parameter-group table: upb_set_param_groups's (pg_user), or one the
                                       // context synthesises from its own settings (refresh_context_table)
  bool pg_user = false;
  long long* tsteps = nullptr;         // device [2][PG_MAX_TENSORS] per-tensor step counts, ping-pong with `steps`
  float* vmax = nullptr;               // device max_exp_avg_sq [num_params] (AMSGrad), allocated on first use
  double* lr_state = nullptr;          // device [2][PG_MAX_TENSORS] lr state of the KL-adaptive lr (upb_set_adaptive_lr),
                                       // ping-pong with `steps`
  unsigned int* idle_stop = nullptr;   // device stop word nothing sets: the kernels' word while only the adaptive lr is on
  double table_lr[PG_MAX_TENSORS] = {};  // the lrs of the active table as last uploaded (upload_table)
  float* prox = nullptr;               // device [num_params] EWMA proximal parameters (upb_set_prox_ewma), allocated on
  float* prox_lp = nullptr;            // first use with [max_graphs] log-probs at them, by position in ids
  bool prox_set = false;               // prox holds parameters (upb_set_prox_params / upb_init_prox_params)
};

// Adam's settings besides lr and weight decay (upb_set_adam; upb_create: the config's betas and eps)
struct AdamSettings {
  float beta1, beta2, eps;
  bool amsgrad, decoupled;
};

namespace {
const int kSgnnTensors[] = {P_NUM_W0,   P_NUM_B0,   P_NUM_W1,    P_NUM_B1,    P_ENC_W,  P_ENC_B,  P_GCN0_W,
                            P_GCN0_B,   P_GCN1_W,   P_GCN1_B,    P_MHA_IN_W,  P_MHA_IN_B, P_MHA_OUT_W, P_MHA_OUT_B,
                            P_ATT_Q_W,  P_ATT_Q_B,  P_ATT_K_W,   P_ATT_K_B,   P_ATT_V_W, P_ATT_V_B, P_LU_W0,
                            P_LU_B0,    P_LU_W1,    P_RD_W0,     P_RD_B0,     P_RD_W1,  P_VAL_W0, P_VAL_B0,
                            P_VAL_W1,   P_VAL_B1,   P_VAL_W2,    P_VAL_B2,    NUM_PARAMS};
const int kMlpTensors[] = {M_NUM_W0, M_NUM_B0, M_NUM_W1, M_NUM_B1, M_ENC_W,  M_ENC_B,  M_LU_W0,  M_LU_B0,  M_LU_W1, M_RD_W0,
                           M_RD_B0,  M_RD_W1,  M_VAL_W0, M_VAL_B0, M_VAL_W1, M_VAL_B1, M_VAL_W2, M_VAL_B2, M_NUM_PARAMS};
static_assert(sizeof(kSgnnTensors) / sizeof(int) == PG_MAX_TENSORS + 1 && sizeof(kMlpTensors) / sizeof(int) == 19,
              "one entry per tensor, then the end");
}  // namespace

namespace {
void reduce_sgnn(const upb_ctx* ctx, int nparts, const float* params, float* grad, const unsigned int* kl_stop,
                 cudaStream_t s);
void reduce_mlp(const upb_ctx* ctx, int nparts, const float* params, float* grad, const unsigned int* kl_stop,
                cudaStream_t s);
}  // namespace

struct upb_ctx {
  upb_config cfg;
  int num_sms = 0;
  int grid = 0;
  Model sgnn{k_sgnn<true>, k_sgnn<false>, NT, SMEM_BYTES, G_ROW, NUM_PARAMS, ENCODER_END, POLICY_END, P_LU_W0,
             P_RD_W0, UPB_STAT_OFFSET, UPB_GRAD_STRIDE, scratch_floats, reduce_sgnn, true, SgnnRow::chain0_begin,
             SgnnRow::chain0_end, SgnnRow::chain1_begin, SgnnRow::chain1_end, k_sgnn_gclip, P_VAL_W2, P_VAL_B2,
             k_sgnn_pg, kSgnnTensors, 32, k_sgnn_values};
  Model mlp{k_mlp<true>, k_mlp<false>, MT, M_SMEM_BYTES, MG_ROW, M_NUM_PARAMS, M_ENCODER_END, M_POLICY_END, M_LU_W0,
            M_RD_W0, UPB_MLP_STAT_OFFSET, UPB_MLP_GRAD_STRIDE, mlp_scratch_floats, reduce_mlp, false, 0, 0, 0, 0, k_mlp_gclip,
            M_VAL_W2, M_VAL_B2, k_mlp_pg, kMlpTensors, 18, k_mlp_values};
  float* gsum = nullptr;        // [G_ROW] (two-call path: k_reduce_finish)
  unsigned int* ticket = nullptr;
  double* gns_part = nullptr;   // [grid + 1] row sums of k_grad_noise (upb_ppo_grad_noise), allocated on first use
  unsigned int* gns_ticket = nullptr;
  unsigned int* gridbar = nullptr;   // [8] fused tail: cumulative arrival counter, stage bits by parity, peer-timeout count
  unsigned int bar_total = 0;        // arrivals at gridbar[0] so far (the counter is never reset)
  double lr = 0.0;                   // Adam's learning rate of both models (upb_set_lr; upb_create: (double)cfg.lr)
  float value_pred_coef = 0.f, entropy_coef = 0.f;   // loss coefficients of both models (upb_set_loss_coefs; upb_create:
                                                     // the cfg's)
  float weight_decay = 0.f;          // Adam's weight decay of both models (upb_set_weight_decay)
  double weight_decay_d = 0.0;       // the same as the double it was set from (upb_set_weight_decay_double): the
                                     // decoupled factor forms lr * weight_decay in double, as torch does
  AdamSettings adam{};               // both models' betas, eps, AMSGrad and decoupled decay (upb_set_adam)
  bool diagnostics = false;          // step kernels fill statistics slots 8-12 (upb_set_diagnostics)
  float kl_limit = 0.f;              // KL stop of both models: fp32(1.5 * target_kl), 0 = off (upb_set_target_kl)
  float clip_lo = 0.f, clip_hi = 0.f;  // the surrogate's clip range (upb_set_clip_range; upb_create: 1.f -/+ clip_epsilon)
  float value_clip = 0.f;            // clipped value loss of both models, range c; 0 = off (upb_set_value_clip)
  float dual_clip = 0.f;             // dual-clip bound c > 1 of both models; 0 = off (upb_set_dual_clip)
  float huber_delta = 0.f;           // Huber value loss threshold of both models; 0 = off (upb_set_huber_delta)
  float max_grad_norm = 0.f;         // global gradient-norm clip of both models; 0 = off (upb_set_max_grad_norm)
  float kl_coef = 0.f;               // KL penalty coefficient beta of both models; 0 = off (upb_set_kl_penalty)
  bool nonfinite_guard = false;      // a step that is not finite applies nothing (upb_set_nonfinite_guard)
  double value_norm_beta = 0.0;      // value-target normalisation of both models, EMA weight; 0 = off (upb_set_value_norm)
  double desired_kl = 0.0;           // KL-adaptive lr of both models; 0 = off (upb_set_adaptive_lr)
  float lr_up = 0.f, lr_down = 0.f;  // its thresholds fp32(desired_kl / 2), fp32(2 desired_kl)
  double lr_min = 0.0, lr_max = 0.0; // its bounds
  bool prox_on = false;              // EWMA proximal policy of both models (upb_set_prox_ewma), weight prox_beta
  float prox_beta = 0.f;
  int coop = 0;                      // cooperative launch supported
  float* host_pinned = nullptr; // [UPB_STAT_COUNT] pinned staging for upb_read_losses
  int64_t launches = 0;
  bool profiling = false;
  long long* stamps = nullptr;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
  size_t prof_used = 0;
  // multi-GPU fused step (upb_peer_export / upb_peer_connect)
  float* xchg = nullptr;             // this rank's exchange buffer (sgnn_kernel.cuh: XCHG_FLOATS): slice sums by
                                     // [parity][source rank], then the per-slice flags
  int world = 1, rank = 0;
  unsigned int peer_seq = 0;
  std::vector<void*> peer_ptrs;      // host copy: exchange buffers of all ranks (own at [rank])
  float** peers_dev = nullptr;       // device array of the same
};

namespace {

#define UPB_CUDA(call)                                                                       \
  do {                                                                                       \
    cudaError_t err__ = (call);                                                              \
    if (err__ != cudaSuccess) {                                                              \
      char buf__[512];                                                                       \
      snprintf(buf__, sizeof(buf__), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err__), \
               __FILE__, __LINE__);                                                          \
      return set_error(UPB_ERR_CUDA, buf__);                                                 \
    }                                                                                        \
  } while (0)

struct Slot {
  const char* name;
  int offset, rows, cols;
};
const Slot kSlots[] = {
    {"num_w0", P_NUM_W0, 64, 52},      {"num_b0", P_NUM_B0, 64, 0},     {"num_w1", P_NUM_W1, 16, 64},
    {"num_b1", P_NUM_B1, 16, 0},       {"enc_w", P_ENC_W, 16, 23},      {"enc_b", P_ENC_B, 16, 0},
    {"gcn0_w", P_GCN0_W, 16, 32},      {"gcn0_b", P_GCN0_B, 16, 0},     {"gcn1_w", P_GCN1_W, 16, 32},
    {"gcn1_b", P_GCN1_B, 16, 0},       {"mha_in_w", P_MHA_IN_W, 48, 16}, {"mha_in_b", P_MHA_IN_B, 48, 0},
    {"mha_out_w", P_MHA_OUT_W, 16, 16}, {"mha_out_b", P_MHA_OUT_B, 16, 0}, {"att_q_w", P_ATT_Q_W, 16, 16},
    {"att_q_b", P_ATT_Q_B, 16, 0},     {"att_k_w", P_ATT_K_W, 16, 16},  {"att_k_b", P_ATT_K_B, 16, 0},
    {"att_v_w", P_ATT_V_W, 16, 16},    {"att_v_b", P_ATT_V_B, 16, 0},   {"lu_w0", P_LU_W0, 32, 64},
    {"lu_b0", P_LU_B0, 32, 0},         {"lu_w1", P_LU_W1, 1, 32},       {"road_w0", P_RD_W0, 32, 16},
    {"road_b0", P_RD_B0, 32, 0},       {"road_w1", P_RD_W1, 1, 32},     {"val_w0", P_VAL_W0, 32, 67},
    {"val_b0", P_VAL_B0, 32, 0},       {"val_w1", P_VAL_W1, 32, 32},    {"val_b1", P_VAL_B1, 32, 0},
    {"val_w2", P_VAL_W2, 1, 32},       {"val_b2", P_VAL_B2, 1, 0},
};
constexpr int kNumSlots = sizeof(kSlots) / sizeof(kSlots[0]);

using ModelOf = Model upb_ctx::*;      // &upb_ctx::sgnn or &upb_ctx::mlp

int check_ctx(const upb_ctx* ctx, const char* who) {
  if (!ctx) return set_error(UPB_ERR_ARG, std::string(who) + ": null context");
  return UPB_OK;
}
int bad_argument(const char* who) { return set_error(UPB_ERR_ARG, std::string(who) + ": bad argument"); }

// event pair bracketing a kernel while profiling is on (events are pooled and reused)
bool prof_begin(upb_ctx* ctx, cudaStream_t s) {
  if (!ctx->profiling) return false;
  if (ctx->prof_used == ctx->prof_events.size()) {
    cudaEvent_t a, b;
    if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return false;
    ctx->prof_events.emplace_back(a, b);
  }
  cudaEventRecord(ctx->prof_events[ctx->prof_used].first, s);
  return true;
}
void prof_end(upb_ctx* ctx, cudaStream_t s, bool on) {
  if (!on) return;
  cudaEventRecord(ctx->prof_events[ctx->prof_used].second, s);
  ctx->prof_used += 1;
}

bool clip_now(const upb_ctx* ctx, const Model& m) {
  return ctx->cfg.clip_mode == UPB_CLIP_ALWAYS || (ctx->cfg.clip_mode == UPB_CLIP_REFERENCE && m.clip_armed);
}

int refresh_context_table(upb_ctx* ctx, Model& m);

// The KL-adaptive lr's state (the "in" side) from the lrs the host set: each tensor's of the active table, or upb_set_lr's
// in every entry.  Called when the option is turned on and whenever upb_set_lr or upb_set_param_groups* sets new lrs
// while it is on; in stream order on the legacy default stream, as those calls' other copies.  Nothing while it is off.
int seed_lr_state(upb_ctx* ctx, Model& m) {
  if (!(ctx->desired_kl > 0.0) || !m.gpart) return UPB_OK;
  double h[PG_MAX_TENSORS];
  for (int t = 0; t < PG_MAX_TENSORS; ++t) h[t] = m.pg && t < m.num_tensors ? m.table_lr[t] : ctx->lr;
  UPB_CUDA(cudaMemcpy(m.lr_state + PG_MAX_TENSORS * m.steps_cur, h, sizeof(h), cudaMemcpyHostToDevice));
  return UPB_OK;
}

// the model's device state; the SGNN's is allocated by upb_create, the rl-mlp's on its first use
int model_init(upb_ctx* ctx, Model& m) {
  if (m.gpart) return UPB_OK;
  m.scratch_stride = (m.scratch_floats(ctx->cfg.n_cap, ctx->cfg.e_cap) + 63) & ~size_t(63);
  UPB_CUDA(cudaMalloc(&m.gpart, sizeof(float) * (size_t)ctx->grid * m.row));
  UPB_CUDA(cudaMalloc(&m.scratch, sizeof(float) * (size_t)ctx->grid * m.scratch_stride));
  UPB_CUDA(cudaMalloc(&m.adam_m, sizeof(float) * m.num_params));
  UPB_CUDA(cudaMalloc(&m.adam_v, sizeof(float) * m.num_params));
  UPB_CUDA(cudaMalloc(&m.steps, sizeof(long long) * 8));
  UPB_CUDA(cudaMalloc(&m.kl_stop, sizeof(unsigned int)));
  UPB_CUDA(cudaMemset(m.kl_stop, 0, sizeof(unsigned int)));
  UPB_CUDA(cudaMalloc(&m.vnorm, sizeof(double) * 3));
  UPB_CUDA(cudaMemset(m.vnorm, 0, sizeof(double) * 3));
  UPB_CUDA(cudaMalloc(&m.lr_state, sizeof(double) * 2 * PG_MAX_TENSORS));
  UPB_CUDA(cudaMemset(m.lr_state, 0, sizeof(double) * 2 * PG_MAX_TENSORS));
  UPB_CUDA(cudaMalloc(&m.idle_stop, sizeof(unsigned int)));
  UPB_CUDA(cudaMemset(m.idle_stop, 0, sizeof(unsigned int)));
  UPB_CUDA(cudaMemset(m.adam_m, 0, sizeof(float) * m.num_params));
  UPB_CUDA(cudaMemset(m.adam_v, 0, sizeof(float) * m.num_params));
  UPB_CUDA(cudaMemset(m.steps, 0, sizeof(long long) * 8));
  UPB_CUDA(cudaMemset(m.scratch, 0, sizeof(float) * (size_t)ctx->grid * m.scratch_stride));
  UPB_CUDA(cudaFuncSetAttribute(m.train, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m.smem));
  UPB_CUDA(cudaFuncSetAttribute(m.infer, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m.smem));
  UPB_CUDA(cudaFuncSetAttribute(m.train_gclip, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m.smem));
  UPB_CUDA(cudaFuncSetAttribute(m.train_pg, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m.smem));
  UPB_CUDA(cudaFuncSetAttribute(m.values, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m.smem));
  UPB_CUDA(cudaDeviceSynchronize());
  if (int rc = refresh_context_table(ctx, m)) return rc;
  return seed_lr_state(ctx, m);
}

void model_free(Model& m) {
  cudaFree(m.pg_mem);
  cudaFree(m.vmax);
  cudaFree(m.tsteps);
  cudaFree(m.gpart);
  cudaFree(m.scratch);
  cudaFree(m.adam_m);
  cudaFree(m.adam_v);
  cudaFree(m.steps);
  cudaFree(m.kl_stop);
  cudaFree(m.vnorm);
  cudaFree(m.lr_state);
  cudaFree(m.idle_stop);
  cudaFree(m.prox);
  cudaFree(m.prox_lp);
}

void reduce_sgnn(const upb_ctx* ctx, int nparts, const float* params, float* grad, const unsigned int* kl_stop,
                 cudaStream_t s) {
  k_reduce_finish<<<RF_BLOCKS, RF_THREADS, 0, s>>>(ctx->sgnn.gpart, nparts, ctx->gsum, params, grad, ctx->ticket,
                                                   kl_stop, ctx->sgnn.pg);
}
void reduce_mlp(const upb_ctx* ctx, int nparts, const float*, float* grad, const unsigned int* kl_stop,
                cudaStream_t s) {
  k_mlp_reduce<<<(MG_ROW + 255) / 256, 256, 0, s>>>(ctx->mlp.gpart, nparts, grad, kl_stop, ctx->mlp.pg);
}

// the per-tensor counts a launch reads and writes (ping-pong by steps_cur, as the per-segment ones)
const long long* tsteps_in(const Model& m) { return m.pg ? m.tsteps + PG_MAX_TENSORS * m.steps_cur : nullptr; }
long long* tsteps_out(const Model& m) { return m.pg ? m.tsteps + PG_MAX_TENSORS * (1 - m.steps_cur) : nullptr; }

// the model's stop word while the KL stop is on, else NULL (the step kernels then ignore the word).  With only the
// KL-adaptive lr on, a word nothing sets and the limit +inf: the kernels fill slot 8 and run the KL gate, which then never
// stops (sgnn_kernel.cuh: StepArgs::alr).
unsigned int* kl_stop_word(const upb_ctx* ctx, const Model& m) {
  if (ctx->kl_limit > 0.f) return m.kl_stop;
  return ctx->desired_kl > 0.0 ? m.idle_stop : nullptr;
}
float kl_stop_limit(const upb_ctx* ctx) {
  return ctx->kl_limit > 0.f || !(ctx->desired_kl > 0.0) ? ctx->kl_limit : INFINITY;
}

// the KL-adaptive lr's arguments of a launch that reads the model's lr state on the current side (before the flip)
AdaptiveLr adaptive_lr(const upb_ctx* ctx, const Model& m) {
  AdaptiveLr al{};
  if (!(ctx->desired_kl > 0.0)) return al;
  al.in = m.lr_state + PG_MAX_TENSORS * m.steps_cur;
  al.out = m.lr_state + PG_MAX_TENSORS * (1 - m.steps_cur);
  al.up = ctx->lr_up;
  al.down = ctx->lr_down;
  al.lo = ctx->lr_min;
  al.hi = ctx->lr_max;
  return al;
}

StepArgs step_args(const upb_ctx* ctx, const Model& m, const void* blob, const int32_t* ids, int count,
                   const float* params, const float* actions) {
  StepArgs a;
  memset(&a, 0, sizeof(a));
  a.blob = (const uint8_t*)blob;
  a.ids = ids;
  a.count = count;
  a.params = params;
  a.actions = actions;
  a.clip_lo = ctx->clip_lo;
  a.clip_hi = ctx->clip_hi;
  a.c_value = ctx->value_pred_coef;
  a.c_entropy = ctx->entropy_coef;
  a.diagnostics = ctx->diagnostics ? 1 : 0;
  a.gpart = m.gpart;
  a.scratch = m.scratch;
  a.scratch_stride = m.scratch_stride;
  a.n_cap = ctx->cfg.n_cap;
  a.e_cap = ctx->cfg.e_cap;
  a.stamps = ctx->stamps;
  return a;
}

// A reference array only reaches the kernels while its option is on: off, the step is that of a context that never set
// the option.  refs may be NULL (no reference data).
void set_ppo_inputs(StepArgs& a, const upb_ctx* ctx, const float* advantages, const float* returns,
                    const float* fixed_log_probs, const float* exps, const upb_step_refs* refs, float inv_batch,
                    float inv_ind) {
  a.adv = advantages;
  a.ret = returns;
  a.fixed_lp = fixed_log_probs;
  a.exps = exps;
  a.inv_batch = inv_batch;
  a.inv_ind = inv_ind;
  a.old_values = ctx->value_clip > 0.f && refs ? refs->old_values : nullptr;
  a.value_clip = ctx->value_clip;
  a.old_cand_logp = ctx->kl_coef > 0.f && refs ? refs->old_cand_log_probs : nullptr;
  a.kl_coef = ctx->kl_coef;
  a.dual_clip = ctx->dual_clip;
  a.huber_delta = ctx->huber_delta;
}

// value clipping needs the pre-pass values, the KL penalty the pre-pass candidate log-probs
int check_refs(const upb_ctx* ctx, const char* who, const upb_step_refs* refs) {
  if (ctx->value_clip > 0.f && !(refs && refs->old_values))
    return set_error(UPB_ERR_ARG, std::string(who) + ": value clipping is on (upb_set_value_clip) and old_values is null");
  if (ctx->kl_coef > 0.f && !(refs && refs->old_cand_log_probs))
    return set_error(UPB_ERR_ARG, std::string(who) + ": the KL penalty is on (upb_set_kl_penalty) and "
                                                     "old_cand_log_probs is null");
  return UPB_OK;
}

void set_kl_stop(StepArgs& a, const upb_ctx* ctx, const Model& m) {
  a.kl_stop = kl_stop_word(ctx, m);
  a.kl_limit = kl_stop_limit(ctx);
}

// The proximal forward of a training launch while the EWMA proximal policy is on: one forward launch at theta_prox over
// the same ids, writing each graph's log-prob into prox_lp by position, which the step kernel then reads
// (StepArgs::prox_lp).  It returns at entry while the model's stop word is set, as the step launch does.
int prox_forward(upb_ctx* ctx, Model& m, const char* who, const void* blob_dev, const int32_t* ids, int count,
                 const float* actions, cudaStream_t s) {
  if (!m.prox_set)
    return set_error(UPB_ERR_ARG, std::string(who) + ": the EWMA proximal policy is on (upb_set_prox_ewma) and its "
                                                     "parameters were never set");
  if (count > ctx->cfg.max_graphs)
    return set_error(UPB_ERR_ARG, std::string(who) + ": count exceeds the context's max_graphs");
  if (count <= 0) return UPB_OK;
  StepArgs a = step_args(ctx, m, blob_dev, ids, count, m.prox, actions);
  a.out_pos_logp = m.prox_lp;
  a.kl_stop = kl_stop_word(ctx, m);
  const int grid = count < ctx->grid ? count : ctx->grid;
  m.infer<<<grid, m.threads, m.smem, s>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

// the EWMA's arguments of a training launch (off: NULL, and the step is that of a context that never set the option)
void set_prox(StepArgs& a, const upb_ctx* ctx, const Model& m, bool fused) {
  if (!ctx->prox_on) return;
  a.prox_lp = m.prox_lp;
  if (fused) {
    a.prox_params = m.prox;
    a.prox_beta = ctx->prox_beta;
  }
}

// ---- one implementation per operation; `who` names the entry point in error messages ---------------------------------
// logit_rows / lu_logits / rd_logits: the masked logit rows of upb_policy_logits (NULL: none)
int forward(upb_ctx* ctx, ModelOf model, const char* who, const void* blob_dev, const int32_t* ids, int count,
            const float* params, const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
            float* cand_log_prob, const int32_t* logit_rows, float* lu_logits, float* rd_logits, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!blob_dev || !params || count < 0) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (count == 0) return UPB_OK;
  StepArgs a = step_args(ctx, m, blob_dev, ids, count, params, actions);
  a.out_value = value;
  a.out_logp = log_prob;
  a.out_entropy = entropy;
  a.out_greedy = greedy;
  a.out_cand_logp = cand_log_prob;
  a.logit_rows = logit_rows;
  a.lu_logits = lu_logits;
  a.rd_logits = rd_logits;
  const int grid = count < ctx->grid ? count : ctx->grid;
  const bool prof = prof_begin(ctx, s);
  m.infer<<<grid, m.threads, m.smem, s>>>(a);
  prof_end(ctx, s, prof);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int values(upb_ctx* ctx, ModelOf model, const char* who, const void* blob_dev, const int32_t* ids, int count,
           const float* params, float* value, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!blob_dev || !params || !value || count < 0) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (count == 0) return UPB_OK;
  StepArgs a = step_args(ctx, m, blob_dev, ids, count, params, nullptr);
  a.out_value = value;
  const int grid = count < ctx->grid ? count : ctx->grid;
  const bool prof = prof_begin(ctx, s);
  m.values<<<grid, m.threads, m.smem, s>>>(a);
  prof_end(ctx, s, prof);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int gae_targets(upb_ctx* ctx, ModelOf model, const char* who, const float* rewards, const float* masks,
                const float* head_values, int T, float gamma, float tau, float* advantages, float* returns,
                float* anchors, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!rewards || !masks || !head_values || !advantages || !returns || !anchors || T < 0) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (T == 0) return UPB_OK;
  const float gamma_tau = (float)((double)gamma * (double)tau);      // as upb_gae forms it
  k_gae_targets<<<(T + 255) / 256, 256, 0, s>>>(rewards, masks, head_values, T, gamma, gamma_tau,
                                                ctx->value_norm_beta > 0.0 ? m.vnorm : nullptr, advantages, returns,
                                                anchors);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int policy_logits(upb_ctx* ctx, ModelOf model, const char* who, const void* blob_dev, const int32_t* ids, int count,
                  const float* params, const int32_t* rows, float* land_use_logits, float* road_logits, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!rows) return bad_argument(who);
  return forward(ctx, model, who, blob_dev, ids, count, params, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                 rows, land_use_logits, road_logits, s);
}

int select_action(upb_ctx* ctx, ModelOf model, const char* who, const void* blob_dev, const int32_t* ids, int count,
                  const float* params, const float* uniforms, int32_t* action_index, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!blob_dev || !params || !action_index || count < 0) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (count == 0) return UPB_OK;
  StepArgs a = step_args(ctx, m, blob_dev, ids, count, params, nullptr);
  if (uniforms) { a.uniforms = uniforms; a.out_sample = action_index; }
  else a.out_greedy = action_index;
  const int grid = count < ctx->grid ? count : ctx->grid;
  m.infer<<<grid, m.threads, m.smem, s>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int ppo_grad(upb_ctx* ctx, ModelOf model, const char* who, const void* blob_dev, const int32_t* ids, int count,
             const float* params, const float* actions, const float* advantages, const float* returns,
             const float* fixed_log_probs, const float* exps, const upb_step_refs* refs, float inv_batch,
             float inv_ind, float* grad_out, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!blob_dev || !params || !actions || !advantages || !returns || !fixed_log_probs || !exps || !grad_out ||
      count < 0)
    return bad_argument(who);
  if (int rc = check_refs(ctx, who, refs)) return rc;
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (ctx->prox_on) {
    if (int rc = prox_forward(ctx, m, who, blob_dev, ids, count, actions, s)) return rc;
  }
  StepArgs a = step_args(ctx, m, blob_dev, ids, count, params, actions);
  set_ppo_inputs(a, ctx, advantages, returns, fixed_log_probs, exps, refs, inv_batch, inv_ind);
  set_kl_stop(a, ctx, m);
  set_prox(a, ctx, m, false);
  const int grid = count < ctx->grid ? count : ctx->grid;
  if (grid > 0) {
    const bool prof = prof_begin(ctx, s);
    m.train<<<grid, m.threads, m.smem, s>>>(a);
    prof_end(ctx, s, prof);
    ctx->launches += 1;
  }
  m.reduce(ctx, grid, params, grad_out, a.kl_stop, s);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

// ppo_grad into grad_out, then k_grad_noise over the launch's partial rows and grad_out (three launches, two while
// count is 0).  The rows and the reduction's scratch are the model's and the context's, so the measurement is one
// operation rather than a call that must follow ppo_grad.
int ppo_grad_noise(upb_ctx* ctx, ModelOf model, const char* who, const void* blob_dev, const int32_t* ids, int count,
                   const float* params, const float* actions, const float* advantages, const float* returns,
                   const float* fixed_log_probs, const float* exps, const upb_step_refs* refs, float inv_batch,
                   float inv_ind, float* grad_out, double* noise_out, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!noise_out) return bad_argument(who);
  if (int rc = ppo_grad(ctx, model, who, blob_dev, ids, count, params, actions, advantages, returns, fixed_log_probs,
                        exps, refs, inv_batch, inv_ind, grad_out, s))
    return rc;
  if (!ctx->gns_part) {
    UPB_CUDA(cudaMalloc(&ctx->gns_part, sizeof(double) * (size_t)(ctx->grid + 1)));
    UPB_CUDA(cudaMalloc(&ctx->gns_ticket, sizeof(unsigned int)));
    UPB_CUDA(cudaMemset(ctx->gns_ticket, 0, sizeof(unsigned int)));
  }
  const Model& m = ctx->*model;
  const int nparts = count < ctx->grid ? count : ctx->grid;
  const unsigned int* word = kl_stop_word(ctx, m);
  if (model == &upb_ctx::sgnn)
    k_grad_noise<SgnnRow><<<nparts + 1, GNS_THREADS, 0, s>>>(m.gpart, nparts, grad_out, params, word, m.pg, count,
                                                            ctx->gns_part, ctx->gns_ticket, noise_out);
  else
    k_grad_noise<MlpRow><<<nparts + 1, GNS_THREADS, 0, s>>>(m.gpart, nparts, grad_out, params, word, m.pg, count,
                                                           ctx->gns_part, ctx->gns_ticket, noise_out);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int apply(upb_ctx* ctx, ModelOf model, const char* who, float* params, float* grad, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!params || !grad) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (ctx->prox_on && !m.prox_set)
    return set_error(UPB_ERR_ARG, std::string(who) + ": the EWMA proximal policy is on (upb_set_prox_ewma) and its "
                                                     "parameters were never set");
  ApplyArgs a;
  a.prox = ctx->prox_on ? m.prox : nullptr;
  a.prox_beta = ctx->prox_beta;
  a.params = params;
  a.grad = grad;
  a.m = m.adam_m;
  a.v = m.adam_v;
  a.steps_in = m.steps + 4 * m.steps_cur;
  a.steps_out = m.steps + 4 * (1 - m.steps_cur);
  a.pg = m.pg;
  a.tsteps_in = tsteps_in(m);
  a.tsteps_out = tsteps_out(m);
  const AdaptiveLr alr = adaptive_lr(ctx, m);
  m.steps_cur = 1 - m.steps_cur;
  a.lr = ctx->lr;
  a.beta1 = ctx->cfg.beta1;
  a.beta2 = ctx->cfg.beta2;
  a.eps = ctx->cfg.adam_eps;
  a.weight_decay = ctx->weight_decay;
  a.clip_now = clip_now(ctx, m) ? 1 : 0;
  m.clip_armed = false;
  a.num_params = m.num_params; a.encoder_end = m.encoder_end; a.policy_end = m.policy_end;
  a.lu_begin = m.lu_begin; a.rd_begin = m.rd_begin; a.stat_offset = m.stat_offset;
  a.kl_stop = kl_stop_word(ctx, m);
  a.kl_limit = kl_stop_limit(ctx);
  a.max_norm = ctx->max_grad_norm;
  a.nslice = (m.row + SLICE - 1) / SLICE;
  a.chain0_begin = m.chain0_begin; a.chain0_end = m.chain0_end;
  a.chain1_begin = m.chain1_begin; a.chain1_end = m.chain1_end;
  a.nonfinite_guard = ctx->nonfinite_guard ? 1 : 0;
  if (alr.in) k_apply<true><<<AP_BLOCKS, AP_THREADS, 0, s>>>(a, alr);
  else k_apply<false><<<AP_BLOCKS, AP_THREADS, 0, s>>>(a, alr);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

// `grad_who` / `apply_who` name the two-call path's entry points, which report its errors
int ppo_step(upb_ctx* ctx, ModelOf model, const char* who, const char* grad_who, const char* apply_who,
             const void* blob_dev, const int32_t* ids, int count, float* params, const float* actions,
             const float* advantages, const float* returns, const float* fixed_log_probs, const float* exps,
             const upb_step_refs* refs, float inv_batch, float inv_ind, float* grad_out, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  const bool clip_step = clip_now(ctx, m);
  if (ctx->world > 1) {
    if (!m.peer_exchange)
      return set_error(UPB_ERR_ARG, std::string(who) + ": peers are connected; rl-mlp multi-GPU steps use "
                                                       "upb_mlp_ppo_grad + all-reduce + upb_mlp_apply");
    if (clip_step || !ctx->coop)
      return set_error(UPB_ERR_ARG, std::string(who) + ": peers are connected and this step clips gradients; use "
                                                       "upb_ppo_grad + all-reduce + upb_apply for it "
                                                       "(upb_next_step_fused() == 0)");
  } else if (clip_step || !ctx->coop || count <= 0) {      // clipping needs a grid-wide norm first: use the two-call path
    int rc = ppo_grad(ctx, model, grad_who, blob_dev, ids, count, params, actions, advantages, returns,
                      fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out, s);
    if (rc != UPB_OK) return rc;
    return apply(ctx, model, apply_who, params, grad_out, s);
  }
  if (!blob_dev || !params || !actions || !advantages || !returns || !fixed_log_probs || !exps || !grad_out)
    return bad_argument(who);
  if (int rc = check_refs(ctx, who, refs)) return rc;
  if (int rc = model_init(ctx, m)) return rc;
  if (ctx->prox_on) {
    if (int rc = prox_forward(ctx, m, who, blob_dev, ids, count, actions, s)) return rc;
  }
  StepArgs a = step_args(ctx, m, blob_dev, ids, count, params, actions);
  set_ppo_inputs(a, ctx, advantages, returns, fixed_log_probs, exps, refs, inv_batch, inv_ind);
  set_kl_stop(a, ctx, m);
  set_prox(a, ctx, m, true);
  a.fuse_tail = 1;
  a.params_rw = params;
  a.grad_out = grad_out;
  a.adam_m = m.adam_m;
  a.adam_v = m.adam_v;
  a.steps_in = m.steps + 4 * m.steps_cur;
  a.steps_out = m.steps + 4 * (1 - m.steps_cur);
  a.pg = m.pg;
  a.tsteps_in = tsteps_in(m);
  a.tsteps_out = tsteps_out(m);
  a.alr = adaptive_lr(ctx, m);
  a.gridbar = ctx->gridbar;
  a.lr = ctx->lr;
  a.beta1 = ctx->cfg.beta1;
  a.beta2 = ctx->cfg.beta2;
  a.adam_eps = ctx->cfg.adam_eps;
  a.weight_decay = ctx->weight_decay;
  a.max_norm = ctx->max_grad_norm;
  a.nonfinite_guard = ctx->nonfinite_guard ? 1 : 0;
  a.world = ctx->world;
  a.rank = ctx->rank;
  a.seq = ++ctx->peer_seq;           // one sequence / parity / barrier count for the fused steps of both models
  a.peers = ctx->peers_dev;
  const int grid = count < 1 ? 1 : (count < ctx->grid ? count : ctx->grid);     // an empty shard still takes part in the exchange
  ctx->bar_total += (unsigned int)grid;
  a.bar_target = ctx->bar_total;
  void* kargs[] = {&a};
  const bool prof = prof_begin(ctx, s);
  // the guard decides on the clip's norm, so it takes the clipping kernel (with coefficient 1 while the clip is off);
  // so do the parameter groups, in a kernel of their own
  const bool norm_step = a.max_norm > 0.f || a.nonfinite_guard;
  void (*kernel)(StepArgs) = m.pg ? m.train_pg : (norm_step ? m.train_gclip : m.train);
  UPB_CUDA(cudaLaunchCooperativeKernel((void*)kernel, dim3(grid), dim3(m.threads), kargs, m.smem, s));
  prof_end(ctx, s, prof);
  ctx->launches += 1;
  m.steps_cur = 1 - m.steps_cur;
  m.clip_armed = false;
  return UPB_OK;
}

int next_step_fused(upb_ctx* ctx, ModelOf model) {
  if (!ctx) return 0;
  const Model& m = ctx->*model;
  return ((m.peer_exchange || ctx->world == 1) && !clip_now(ctx, m) && ctx->coop) ? 1 : 0;
}

int rearm_clip(upb_ctx* ctx, ModelOf model, const char* who) {
  if (int rc = check_ctx(ctx, who)) return rc;
  (ctx->*model).clip_armed = true;
  return UPB_OK;
}

int reset_kl_stop(upb_ctx* ctx, ModelOf model, const char* who, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  UPB_CUDA(cudaMemsetAsync(m.kl_stop, 0, sizeof(unsigned int), s));
  return UPB_OK;
}

int read_losses(upb_ctx* ctx, ModelOf model, const char* who, const float* grad, float* out4_host, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!grad || !out4_host) return bad_argument(who);
  UPB_CUDA(cudaMemcpyAsync(ctx->host_pinned, grad + (ctx->*model).stat_offset, sizeof(float) * (KLPEN_SLOT + 1),
                           cudaMemcpyDeviceToHost, s));
  UPB_CUDA(cudaStreamSynchronize(s));
  const float* st = ctx->host_pinned;
  const float nB = st[3] > 0.f ? st[3] : 1.f, nI = st[4] > 0.f ? st[4] : 1.f;
  // while clipping or Huber is on, the value loss the step optimised (slot 15); slot 0 keeps sum (V - R)^2
  const float value_loss = (ctx->value_clip > 0.f || ctx->huber_delta > 0.f ? st[VCLIP_LOSS_SLOT] : st[0]) / nB,
              surr = st[1] / nI,
              ent = st[2] / nI;
  out4_host[0] = surr + ctx->value_pred_coef * value_loss + ctx->entropy_coef * ent;
  if (ctx->kl_coef > 0.f) out4_host[0] += ctx->kl_coef * (st[KLPEN_SLOT] / nI);    // + beta * mean exact KL
  out4_host[1] = value_loss;
  out4_host[2] = surr;
  out4_host[3] = ent;
  return UPB_OK;
}

int get_opt_state(upb_ctx* ctx, ModelOf model, const char* who, float* m_host, float* v_host, int64_t* steps4_host) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (m_host) UPB_CUDA(cudaMemcpy(m_host, m.adam_m, sizeof(float) * m.num_params, cudaMemcpyDeviceToHost));
  if (v_host) UPB_CUDA(cudaMemcpy(v_host, m.adam_v, sizeof(float) * m.num_params, cudaMemcpyDeviceToHost));
  if (steps4_host)
    UPB_CUDA(cudaMemcpy(steps4_host, m.steps + 4 * m.steps_cur, sizeof(long long) * 4, cudaMemcpyDeviceToHost));
  return UPB_OK;
}

int set_opt_state(upb_ctx* ctx, ModelOf model, const char* who, const float* m_host, const float* v_host,
                  const int64_t* steps4_host) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (m_host) UPB_CUDA(cudaMemcpy(m.adam_m, m_host, sizeof(float) * m.num_params, cudaMemcpyHostToDevice));
  if (v_host) UPB_CUDA(cudaMemcpy(m.adam_v, v_host, sizeof(float) * m.num_params, cudaMemcpyHostToDevice));
  if (steps4_host) {
    UPB_CUDA(cudaMemcpy(m.steps + 4 * m.steps_cur, steps4_host, sizeof(long long) * 4, cudaMemcpyHostToDevice));
    m.clip_armed = steps4_host[0] == 0;
    // a synthesised table's counts are its segments': restart them from the restored ones
    if (m.pg && !m.pg_user) {
      m.pg = nullptr;
      return refresh_context_table(ctx, m);
    }
  }
  return UPB_OK;
}

// the model's EWMA proximal parameters and log-prob buffer, allocated on first use
int prox_alloc(upb_ctx* ctx, Model& m) {
  if (int rc = model_init(ctx, m)) return rc;
  if (m.prox) return UPB_OK;
  UPB_CUDA(cudaMalloc(&m.prox, sizeof(float) * m.num_params));
  UPB_CUDA(cudaMalloc(&m.prox_lp, sizeof(float) * (size_t)(ctx->cfg.max_graphs > 0 ? ctx->cfg.max_graphs : 1)));
  return UPB_OK;
}

// upb_get_prox_params / upb_set_prox_params: host copies of theta_prox, n = the model's parameter count, synchronous
int prox_params_host(upb_ctx* ctx, ModelOf model, const char* who, float* get, const float* set, int n) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (n != m.num_params || !(get || set)) return bad_argument(who);
  if (int rc = prox_alloc(ctx, m)) return rc;
  if (get && !m.prox_set)
    return set_error(UPB_ERR_ARG, std::string(who) + ": the EWMA proximal parameters were never set");
  UPB_CUDA(cudaDeviceSynchronize());
  if (get) UPB_CUDA(cudaMemcpy(get, m.prox, sizeof(float) * n, cudaMemcpyDeviceToHost));
  else UPB_CUDA(cudaMemcpy(m.prox, set, sizeof(float) * n, cudaMemcpyHostToDevice));
  if (set) m.prox_set = true;
  return UPB_OK;
}

// upb_init_prox_params: theta_prox <- params (device), queued on `stream`
int init_prox_params(upb_ctx* ctx, ModelOf model, const char* who, const float* params, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!params) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = prox_alloc(ctx, m)) return rc;
  UPB_CUDA(cudaMemcpyAsync(m.prox, params, sizeof(float) * m.num_params, cudaMemcpyDeviceToDevice, s));
  m.prox_set = true;
  return UPB_OK;
}

int grad_norms(upb_ctx* ctx, ModelOf model, const char* who, const float* grad_rows, int rows, float* out,
               cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!grad_rows || !out || rows < 0) return bad_argument(who);
  if (rows == 0) return UPB_OK;
  const Model& m = ctx->*model;
  k_grad_norms<<<rows, GN_THREADS, 0, s>>>(grad_rows, m.grad_stride, m.num_params, m.encoder_end, m.policy_end, out);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int value_norm_denormalize(upb_ctx* ctx, ModelOf model, const char* who, const float* normalized, int T, float* values,
                           cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!normalized || !values || T < 0) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  if (T == 0) return UPB_OK;
  k_value_denorm<<<(T + 255) / 256, 256, 0, s>>>(normalized, T, m.vnorm, values);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int value_norm_update(upb_ctx* ctx, ModelOf model, const char* who, const float* returns, const float* values, int T,
                      float* params, float* norm_returns, float* norm_values, double* mean_std, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!(ctx->value_norm_beta > 0.0))
    return set_error(UPB_ERR_ARG, std::string(who) + ": value-target normalisation is off (upb_set_value_norm)");
  if (!returns || !params || !norm_returns || T < 1 || (values != nullptr) != (norm_values != nullptr))
    return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  k_value_norm<<<1, AN_THREADS, 0, s>>>(returns, values, T, m.vnorm, ctx->value_norm_beta, params, m.val_w2, m.val_b2,
                                        norm_returns, norm_values, mean_std);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

int get_value_norm_state(upb_ctx* ctx, ModelOf model, const char* who, double* state3_host) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!state3_host) return bad_argument(who);
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  UPB_CUDA(cudaMemcpy(state3_host, m.vnorm, sizeof(double) * 3, cudaMemcpyDeviceToHost));
  return UPB_OK;
}

int set_value_norm_state(upb_ctx* ctx, ModelOf model, const char* who, const double* state3_host) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!state3_host) return bad_argument(who);
  for (int i = 0; i < 3; ++i)
    if (!std::isfinite(state3_host[i])) return set_error(UPB_ERR_ARG, std::string(who) + ": the state must be finite");
  if (state3_host[1] < 0.0 || state3_host[2] < 0.0 || state3_host[2] > 1.0)
    return set_error(UPB_ERR_ARG, std::string(who) + ": need m2 >= 0 and 0 <= d <= 1");
  Model& m = ctx->*model;
  if (int rc = model_init(ctx, m)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  UPB_CUDA(cudaMemcpy(m.vnorm, state3_host, sizeof(double) * 3, cudaMemcpyHostToDevice));
  return UPB_OK;
}

// Adam settings of the context or of one tensor (upb_set_adam, upb_set_param_groups_adam); UPB_ERR_ARG for a beta
// outside [0, 1) or an eps that is negative or not finite, as torch.optim.Adam raises
int check_adam(const char* who, float beta1, float beta2, float eps, int t = -1) {
  const std::string at = t < 0 ? std::string() : " (tensor " + std::to_string(t) + ")";
  if (!(beta1 >= 0.f && beta1 < 1.f) || !(beta2 >= 0.f && beta2 < 1.f))
    return set_error(UPB_ERR_ARG, std::string(who) + ": betas must be in [0, 1)" + at);
  if (!std::isfinite(eps) || eps < 0.f)
    return set_error(UPB_ERR_ARG, std::string(who) + ": eps must be finite and >= 0" + at);
  return UPB_OK;
}

// Tensor t of a host table: lr, weight decay and Adam settings.  The decoupled decay is the factor fp32(1 - lr * wd),
// formed in double as torch forms the Python scalar of param.mul_; the coupled term keeps fp32(wd).  The moment
// weights are 1.f - fp32(beta), as the untabled steps form them.
void fill_tensor(ParamGroups& h, int t, double lr, double wd, const AdamSettings& s) {
  const bool decoupled = s.decoupled && wd != 0.0;
  h.lr[t] = lr;
  h.weight_decay[t] = decoupled ? 0.f : (float)wd;
  h.decay[t] = decoupled ? (float)(1.0 - lr * wd) : 1.f;
  h.decoupled_wd[t] = decoupled ? wd : 0.0;
  h.beta1[t] = s.beta1;
  h.beta2[t] = s.beta2;
  h.w1[t] = 1.f - s.beta1;
  h.w2[t] = 1.f - s.beta2;
  h.eps[t] = s.eps;
  h.amsgrad[t] = s.amsgrad ? 1 : 0;
}

// Makes h (lr, weight decay, trained flags and Adam settings filled) the model's active table.  A table that becomes
// active starts every tensor from its segment's count, exact for a run that never froze a tensor.  The AMSGrad buffer
// is allocated zero-filled when a tensor first has amsgrad.  Synchronises the device.
int upload_table(Model& m, ParamGroups& h) {
  h.n = m.num_tensors;
  bool ams = false;
  for (int t = 0; t < m.num_tensors; ++t) {
    const int b = m.tensor_offsets[t], e = m.tensor_offsets[t + 1];
    h.seg[t] = b >= m.lu_begin && b < m.rd_begin ? 1 : (b >= m.rd_begin && b < m.policy_end ? 2 : 0);
    for (int c = b; c < e; ++c) h.tensor_of[c] = (uint8_t)t;
    ams = ams || h.amsgrad[t];
  }
  UPB_CUDA(cudaDeviceSynchronize());
  if (ams && !m.vmax) {
    UPB_CUDA(cudaMalloc(&m.vmax, sizeof(float) * m.num_params));
    UPB_CUDA(cudaMemset(m.vmax, 0, sizeof(float) * m.num_params));
  }
  h.vmax = m.vmax;
  if (!m.pg_mem) {
    UPB_CUDA(cudaMalloc(&m.tsteps, sizeof(long long) * 2 * PG_MAX_TENSORS));
    UPB_CUDA(cudaMalloc(&m.pg_mem, sizeof(ParamGroups)));
  }
  if (!m.pg) {
    long long s4[4], ts[2 * PG_MAX_TENSORS] = {};
    UPB_CUDA(cudaMemcpy(s4, m.steps + 4 * m.steps_cur, sizeof(s4), cudaMemcpyDeviceToHost));
    for (int t = 0; t < m.num_tensors; ++t) ts[PG_MAX_TENSORS * m.steps_cur + t] = s4[1 + h.seg[t]];
    UPB_CUDA(cudaMemcpy(m.tsteps, ts, sizeof(ts), cudaMemcpyHostToDevice));
  }
  UPB_CUDA(cudaMemcpy(m.pg_mem, &h, sizeof(ParamGroups), cudaMemcpyHostToDevice));
  m.pg = m.pg_mem;
  for (int t = 0; t < PG_MAX_TENSORS; ++t) m.table_lr[t] = h.lr[t];
  return UPB_OK;
}

// The context's Adam settings are upb_create's: the model steps without a table unless it has one of its own
bool adam_default(const upb_ctx* ctx) {
  const AdamSettings& s = ctx->adam;
  return s.beta1 == ctx->cfg.beta1 && s.beta2 == ctx->cfg.beta2 && s.eps == ctx->cfg.adam_eps && !s.amsgrad &&
         !(s.decoupled && ctx->weight_decay != 0.f);
}

// Without upb_set_param_groups, a model steps through a table synthesised from the context's lr, weight decay and Adam
// settings while these are not the defaults, and without a table otherwise.  Called whenever one of them changes and
// when the model is initialised.
int refresh_context_table(upb_ctx* ctx, Model& m) {
  if (m.pg_user || !m.gpart) return UPB_OK;
  if (adam_default(ctx)) {
    m.pg = nullptr;
    return UPB_OK;
  }
  std::vector<char> buf(sizeof(ParamGroups), 0);
  ParamGroups& h = *reinterpret_cast<ParamGroups*>(buf.data());
  for (int t = 0; t < m.num_tensors; ++t) {
    h.trained[t] = 1;
    fill_tensor(h, t, ctx->lr, ctx->weight_decay_d, ctx->adam);
  }
  return upload_table(m, h);
}
int refresh_context_tables(upb_ctx* ctx) {
  if (int rc = refresh_context_table(ctx, ctx->sgnn)) return rc;
  return refresh_context_table(ctx, ctx->mlp);
}

// upb_set_param_groups (adam NULL: every tensor at the context's Adam settings) and upb_set_param_groups_adam
int set_param_groups(upb_ctx* ctx, ModelOf model, const char* who, const double* lr, const double* weight_decay,
                     const uint8_t* trained, const AdamSettings* adam, int n_tensors) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (!lr || !weight_decay || !trained || n_tensors != m.num_tensors)
    return set_error(UPB_ERR_ARG, std::string(who) + ": need tables of " + std::to_string(m.num_tensors) +
                                      " tensors (upb_param_slot order)");
  bool any = false;
  for (int t = 0; t < n_tensors; ++t) {
    if (!std::isfinite(lr[t]) || lr[t] < 0.0)
      return set_error(UPB_ERR_ARG, std::string(who) + ": lr must be finite and >= 0 (tensor " + std::to_string(t) + ")");
    if (!std::isfinite(weight_decay[t]) || weight_decay[t] < 0.0)
      return set_error(UPB_ERR_ARG, std::string(who) + ": weight_decay must be finite and >= 0 (tensor " +
                                        std::to_string(t) + ")");
    if (adam)
      if (int rc = check_adam(who, adam[t].beta1, adam[t].beta2, adam[t].eps, t)) return rc;
    any = any || trained[t] != 0;
  }
  if (!any) return set_error(UPB_ERR_ARG, std::string(who) + ": no tensor is trained");
  if (int rc = model_init(ctx, m)) return rc;
  std::vector<char> buf(sizeof(ParamGroups), 0);
  ParamGroups& h = *reinterpret_cast<ParamGroups*>(buf.data());
  for (int t = 0; t < n_tensors; ++t) {
    h.trained[t] = trained[t] != 0;
    fill_tensor(h, t, lr[t], weight_decay[t], adam ? adam[t] : ctx->adam);
  }
  if (int rc = upload_table(m, h)) return rc;
  m.pg_user = true;
  return seed_lr_state(ctx, m);
}

int set_param_groups_adam(upb_ctx* ctx, ModelOf model, const char* who, const double* lr, const double* weight_decay,
                          const uint8_t* trained, const float* beta1, const float* beta2, const float* eps,
                          const uint8_t* amsgrad, const uint8_t* decoupled, int n_tensors) {
  if (int rc = check_ctx(ctx, who)) return rc;
  if (!beta1 || !beta2 || !eps || !amsgrad || !decoupled || n_tensors < 0 || n_tensors > PG_MAX_TENSORS)
    return set_error(UPB_ERR_ARG, std::string(who) + ": need tables of " +
                                      std::to_string((ctx->*model).num_tensors) + " tensors (upb_param_slot order)");
  AdamSettings adam[PG_MAX_TENSORS];
  for (int t = 0; t < n_tensors; ++t) adam[t] = {beta1[t], beta2[t], eps[t], amsgrad[t] != 0, decoupled[t] != 0};
  return set_param_groups(ctx, model, who, lr, weight_decay, trained, adam, n_tensors);
}

// upb_get_amsgrad_state with no host array: 1 while the model holds max_exp_avg_sq, else 0
int has_amsgrad_state(upb_ctx* ctx, ModelOf model, const char* who) {
  if (int rc = check_ctx(ctx, who)) return rc;
  return (ctx->*model).vmax ? 1 : 0;
}

int amsgrad_state(upb_ctx* ctx, ModelOf model, const char* who, float* get, const float* set, int n) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (!(get || set) || n != m.num_params)
    return set_error(UPB_ERR_ARG, std::string(who) + ": need " + std::to_string(m.num_params) + " values");
  if (get && !m.vmax)
    return set_error(UPB_ERR_ARG, std::string(who) + ": no AMSGrad state (no tensor has had amsgrad)");
  if (int rc = model_init(ctx, m)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (get) UPB_CUDA(cudaMemcpy(get, m.vmax, sizeof(float) * n, cudaMemcpyDeviceToHost));
  if (set) {
    if (!m.vmax) {
      UPB_CUDA(cudaMalloc(&m.vmax, sizeof(float) * n));
      if (m.pg_mem) UPB_CUDA(cudaMemcpy(&m.pg_mem->vmax, &m.vmax, sizeof(float*), cudaMemcpyHostToDevice));
    }
    UPB_CUDA(cudaMemcpy(m.vmax, set, sizeof(float) * n, cudaMemcpyHostToDevice));
  }
  return UPB_OK;
}

int tensor_steps(upb_ctx* ctx, ModelOf model, const char* who, int64_t* get, const int64_t* set, int n_tensors) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (!m.pg) return set_error(UPB_ERR_ARG, std::string(who) + ": no parameter groups (upb_set_param_groups)");
  if (!(get || set) || n_tensors != m.num_tensors)
    return set_error(UPB_ERR_ARG, std::string(who) + ": need a table of " + std::to_string(m.num_tensors) + " counts");
  long long* cur = m.tsteps + PG_MAX_TENSORS * m.steps_cur;
  UPB_CUDA(cudaDeviceSynchronize());
  if (get) UPB_CUDA(cudaMemcpy(get, cur, sizeof(long long) * n_tensors, cudaMemcpyDeviceToHost));
  if (set) {
    for (int t = 0; t < n_tensors; ++t)
      if (set[t] < 0) return set_error(UPB_ERR_ARG, std::string(who) + ": counts must be >= 0");
    UPB_CUDA(cudaMemcpy(cur, set, sizeof(long long) * n_tensors, cudaMemcpyHostToDevice));
  }
  return UPB_OK;
}

}  // namespace

extern "C" int upb_num_params(void) { return NUM_PARAMS; }

extern "C" int upb_param_slot(int i, const char** name, int* offset, int* rows, int* cols) {
  if (i < 0 || i >= kNumSlots) return set_error(UPB_ERR_ARG, "param_slot: index out of range");
  if (name) *name = kSlots[i].name;
  if (offset) *offset = kSlots[i].offset;
  if (rows) *rows = kSlots[i].rows;
  if (cols) *cols = kSlots[i].cols;
  return UPB_OK;
}

extern "C" int upb_create(const upb_config* cfg, upb_ctx** out) {
  if (!cfg || !out) return set_error(UPB_ERR_ARG, "create: null argument");
  if (cfg->n_cap < 1 || cfg->n_cap > 65535 || cfg->e_cap < 0 || 2 * (int64_t)cfg->e_cap > 65535)
    return set_error(UPB_ERR_ARG, "create: caps must satisfy 1 <= n_cap <= 65535 and 2*e_cap <= 65535");
  if (cfg->clip_mode < 0 || cfg->clip_mode > 2) return set_error(UPB_ERR_ARG, "create: bad clip_mode");
  UPB_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  UPB_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)      // sm_90a code loads on compute capability 9.0 only
    return set_error(UPB_ERR_CUDA, "create: this library is built for sm_90a (H100) only");
  upb_ctx* ctx = new (std::nothrow) upb_ctx();
  if (!ctx) return set_error(UPB_ERR_ARG, "create: out of host memory");
  ctx->cfg = *cfg;
  ctx->clip_lo = 1.f - cfg->clip_epsilon;
  ctx->clip_hi = 1.f + cfg->clip_epsilon;
  ctx->lr = (double)cfg->lr;
  ctx->adam = {cfg->beta1, cfg->beta2, cfg->adam_eps, false, false};
  ctx->value_pred_coef = cfg->value_pred_coef;
  ctx->entropy_coef = cfg->entropy_coef;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->grid = ctx->num_sms;
  if (cfg->grid_limit > 0 && cfg->grid_limit < ctx->grid) ctx->grid = cfg->grid_limit;
  auto fail = [&](int rc) { upb_destroy(ctx); return rc; };
#define UPB_CUDA_F(call)                                                                     \
  do {                                                                                       \
    cudaError_t err__ = (call);                                                              \
    if (err__ != cudaSuccess) {                                                              \
      char buf__[512];                                                                       \
      snprintf(buf__, sizeof(buf__), "%s failed: %s", #call, cudaGetErrorString(err__));     \
      return fail(set_error(UPB_ERR_CUDA, buf__));                                           \
    }                                                                                        \
  } while (0)
  if (int rc = model_init(ctx, ctx->sgnn)) return fail(rc);
  UPB_CUDA_F(cudaMalloc(&ctx->gsum, sizeof(float) * G_ROW));
  UPB_CUDA_F(cudaMalloc(&ctx->ticket, sizeof(unsigned int)));
  UPB_CUDA_F(cudaMemset(ctx->ticket, 0, sizeof(unsigned int)));
  UPB_CUDA_F(cudaMalloc(&ctx->gridbar, 8 * sizeof(unsigned int)));
  UPB_CUDA_F(cudaMemset(ctx->gridbar, 0, 8 * sizeof(unsigned int)));
  UPB_CUDA_F(cudaMalloc(&ctx->xchg, sizeof(float) * XCHG_FLOATS));
  UPB_CUDA_F(cudaMemset(ctx->xchg, 0, sizeof(float) * XCHG_FLOATS));
  UPB_CUDA_F(cudaMalloc(&ctx->peers_dev, sizeof(float*) * MAX_PEERS));
  {
    float* self[MAX_PEERS] = {};
    self[0] = ctx->xchg;                 // one GPU: rank 0 of a world of 1
    UPB_CUDA_F(cudaMemcpy(ctx->peers_dev, self, sizeof(self), cudaMemcpyHostToDevice));
  }
  UPB_CUDA_F(cudaDeviceGetAttribute(&ctx->coop, cudaDevAttrCooperativeLaunch, cfg->device));
  UPB_CUDA_F(cudaMallocHost(&ctx->host_pinned, sizeof(float) * UPB_STAT_COUNT));
  UPB_CUDA_F(cudaDeviceSynchronize());
#undef UPB_CUDA_F
  *out = ctx;
  return UPB_OK;
}

extern "C" void upb_destroy(upb_ctx* ctx) {
  if (!ctx) return;
  model_free(ctx->sgnn);
  model_free(ctx->mlp);
  cudaFree(ctx->gsum);
  cudaFree(ctx->ticket);
  cudaFree(ctx->gns_part);
  cudaFree(ctx->gns_ticket);
  cudaFree(ctx->gridbar);
  for (int p = 0; p < (int)ctx->peer_ptrs.size(); ++p)
    if (p != ctx->rank && ctx->peer_ptrs[p]) cudaIpcCloseMemHandle(ctx->peer_ptrs[p]);
  cudaFree(ctx->peers_dev);
  cudaFree(ctx->xchg);
  if (ctx->host_pinned) cudaFreeHost(ctx->host_pinned);
  for (auto& ev : ctx->prof_events) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
  delete ctx;
}

// ---- per-model entry points: SGNN (upb_*) and rl-mlp (upb_mlp_*) --------------------------------------------------------
extern "C" int upb_forward(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                           const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                           void* stream) {
  return forward(ctx, &upb_ctx::sgnn, "forward", blob_dev, ids, count, params, actions, value, log_prob, entropy,
                 greedy, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}
extern "C" int upb_mlp_forward(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                               const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                               void* stream) {
  return forward(ctx, &upb_ctx::mlp, "mlp_forward", blob_dev, ids, count, params, actions, value, log_prob, entropy,
                 greedy, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}
extern "C" int upb_forward_cand(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                                const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                                float* cand_log_prob, void* stream) {
  return forward(ctx, &upb_ctx::sgnn, "forward_cand", blob_dev, ids, count, params, actions, value, log_prob, entropy,
                 greedy, cand_log_prob, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}
extern "C" int upb_mlp_forward_cand(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                    const float* params, const float* actions, float* value, float* log_prob,
                                    float* entropy, int32_t* greedy, float* cand_log_prob, void* stream) {
  return forward(ctx, &upb_ctx::mlp, "mlp_forward_cand", blob_dev, ids, count, params, actions, value, log_prob,
                 entropy, greedy, cand_log_prob, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int upb_values(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                          float* value, void* stream) {
  return values(ctx, &upb_ctx::sgnn, "values", blob_dev, ids, count, params, value, (cudaStream_t)stream);
}
extern "C" int upb_mlp_values(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                              float* value, void* stream) {
  return values(ctx, &upb_ctx::mlp, "mlp_values", blob_dev, ids, count, params, value, (cudaStream_t)stream);
}

extern "C" int upb_policy_logits(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                                 const int32_t* rows, float* land_use_logits, float* road_logits, void* stream) {
  return policy_logits(ctx, &upb_ctx::sgnn, "policy_logits", blob_dev, ids, count, params, rows, land_use_logits,
                       road_logits, (cudaStream_t)stream);
}
extern "C" int upb_mlp_policy_logits(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                     const float* params, const int32_t* rows, float* land_use_logits,
                                     float* road_logits, void* stream) {
  return policy_logits(ctx, &upb_ctx::mlp, "mlp_policy_logits", blob_dev, ids, count, params, rows, land_use_logits,
                       road_logits, (cudaStream_t)stream);
}

extern "C" int upb_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                                 const float* uniforms, int32_t* action_index, void* stream) {
  return select_action(ctx, &upb_ctx::sgnn, "select_action", blob_dev, ids, count, params, uniforms, action_index,
                       (cudaStream_t)stream);
}
extern "C" int upb_mlp_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                     const float* params, const float* uniforms, int32_t* action_index, void* stream) {
  return select_action(ctx, &upb_ctx::mlp, "mlp_select_action", blob_dev, ids, count, params, uniforms, action_index,
                       (cudaStream_t)stream);
}

extern "C" int upb_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                            const float* actions, const float* advantages, const float* returns,
                            const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                            float* grad_out, void* stream) {
  return ppo_grad(ctx, &upb_ctx::sgnn, "ppo_grad", blob_dev, ids, count, params, actions, advantages, returns,
                  fixed_log_probs, exps, nullptr, inv_batch, inv_ind, grad_out, (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                                const float* actions, const float* advantages, const float* returns,
                                const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                                float* grad_out, void* stream) {
  return ppo_grad(ctx, &upb_ctx::mlp, "mlp_ppo_grad", blob_dev, ids, count, params, actions, advantages, returns,
                  fixed_log_probs, exps, nullptr, inv_batch, inv_ind, grad_out, (cudaStream_t)stream);
}
extern "C" int upb_ppo_grad_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                  const float* params, const float* actions, const float* advantages,
                                  const float* returns, const float* fixed_log_probs, const float* exps,
                                  const float* old_values, float inv_batch, float inv_ind, float* grad_out,
                                  void* stream) {
  const upb_step_refs refs = {old_values, nullptr};
  return ppo_grad(ctx, &upb_ctx::sgnn, "ppo_grad_vclip", blob_dev, ids, count, params, actions, advantages, returns,
                  fixed_log_probs, exps, &refs, inv_batch, inv_ind, grad_out, (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_grad_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                      const float* params, const float* actions, const float* advantages,
                                      const float* returns, const float* fixed_log_probs, const float* exps,
                                      const float* old_values, float inv_batch, float inv_ind, float* grad_out,
                                      void* stream) {
  const upb_step_refs refs = {old_values, nullptr};
  return ppo_grad(ctx, &upb_ctx::mlp, "mlp_ppo_grad_vclip", blob_dev, ids, count, params, actions, advantages,
                  returns, fixed_log_probs, exps, &refs, inv_batch, inv_ind, grad_out, (cudaStream_t)stream);
}
extern "C" int upb_ppo_grad_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                 const float* params, const float* actions, const float* advantages,
                                 const float* returns, const float* fixed_log_probs, const float* exps,
                                 const upb_step_refs* refs, float inv_batch, float inv_ind, float* grad_out,
                                 void* stream) {
  return ppo_grad(ctx, &upb_ctx::sgnn, "ppo_grad_refs", blob_dev, ids, count, params, actions, advantages, returns,
                  fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out, (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_grad_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                     const float* params, const float* actions, const float* advantages,
                                     const float* returns, const float* fixed_log_probs, const float* exps,
                                     const upb_step_refs* refs, float inv_batch, float inv_ind, float* grad_out,
                                     void* stream) {
  return ppo_grad(ctx, &upb_ctx::mlp, "mlp_ppo_grad_refs", blob_dev, ids, count, params, actions, advantages,
                  returns, fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out, (cudaStream_t)stream);
}

extern "C" int upb_ppo_grad_noise(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                  const float* params, const float* actions, const float* advantages,
                                  const float* returns, const float* fixed_log_probs, const float* exps,
                                  const upb_step_refs* refs, float inv_batch, float inv_ind, float* grad_out,
                                  double* noise_out, void* stream) {
  return ppo_grad_noise(ctx, &upb_ctx::sgnn, "ppo_grad_noise", blob_dev, ids, count, params, actions, advantages,
                        returns, fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out, noise_out,
                        (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_grad_noise(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                      const float* params, const float* actions, const float* advantages,
                                      const float* returns, const float* fixed_log_probs, const float* exps,
                                      const upb_step_refs* refs, float inv_batch, float inv_ind, float* grad_out,
                                      double* noise_out, void* stream) {
  return ppo_grad_noise(ctx, &upb_ctx::mlp, "mlp_ppo_grad_noise", blob_dev, ids, count, params, actions, advantages,
                        returns, fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out, noise_out,
                        (cudaStream_t)stream);
}

extern "C" int upb_apply(upb_ctx* ctx, float* params, float* grad, void* stream) {
  return apply(ctx, &upb_ctx::sgnn, "apply", params, grad, (cudaStream_t)stream);
}
extern "C" int upb_mlp_apply(upb_ctx* ctx, float* params, float* grad, void* stream) {
  return apply(ctx, &upb_ctx::mlp, "mlp_apply", params, grad, (cudaStream_t)stream);
}

extern "C" int upb_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                            const float* actions, const float* advantages, const float* returns,
                            const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                            float* grad_out, void* stream) {
  return ppo_step(ctx, &upb_ctx::sgnn, "ppo_step", "ppo_grad", "apply", blob_dev, ids, count, params, actions,
                  advantages, returns, fixed_log_probs, exps, nullptr, inv_batch, inv_ind, grad_out,
                  (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                                const float* actions, const float* advantages, const float* returns,
                                const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                                float* grad_out, void* stream) {
  return ppo_step(ctx, &upb_ctx::mlp, "mlp_ppo_step", "mlp_ppo_grad", "mlp_apply", blob_dev, ids, count, params,
                  actions, advantages, returns, fixed_log_probs, exps, nullptr, inv_batch, inv_ind, grad_out,
                  (cudaStream_t)stream);
}
extern "C" int upb_ppo_step_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                                  const float* actions, const float* advantages, const float* returns,
                                  const float* fixed_log_probs, const float* exps, const float* old_values,
                                  float inv_batch, float inv_ind, float* grad_out, void* stream) {
  const upb_step_refs refs = {old_values, nullptr};
  return ppo_step(ctx, &upb_ctx::sgnn, "ppo_step_vclip", "ppo_grad_vclip", "apply", blob_dev, ids, count, params,
                  actions, advantages, returns, fixed_log_probs, exps, &refs, inv_batch, inv_ind, grad_out,
                  (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_step_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                      float* params, const float* actions, const float* advantages,
                                      const float* returns, const float* fixed_log_probs, const float* exps,
                                      const float* old_values, float inv_batch, float inv_ind, float* grad_out,
                                      void* stream) {
  const upb_step_refs refs = {old_values, nullptr};
  return ppo_step(ctx, &upb_ctx::mlp, "mlp_ppo_step_vclip", "mlp_ppo_grad_vclip", "mlp_apply", blob_dev, ids, count,
                  params, actions, advantages, returns, fixed_log_probs, exps, &refs, inv_batch, inv_ind,
                  grad_out, (cudaStream_t)stream);
}
extern "C" int upb_ppo_step_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                                 const float* actions, const float* advantages, const float* returns,
                                 const float* fixed_log_probs, const float* exps, const upb_step_refs* refs,
                                 float inv_batch, float inv_ind, float* grad_out, void* stream) {
  return ppo_step(ctx, &upb_ctx::sgnn, "ppo_step_refs", "ppo_grad_refs", "apply", blob_dev, ids, count, params,
                  actions, advantages, returns, fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out,
                  (cudaStream_t)stream);
}
extern "C" int upb_mlp_ppo_step_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                     float* params, const float* actions, const float* advantages,
                                     const float* returns, const float* fixed_log_probs, const float* exps,
                                     const upb_step_refs* refs, float inv_batch, float inv_ind, float* grad_out,
                                     void* stream) {
  return ppo_step(ctx, &upb_ctx::mlp, "mlp_ppo_step_refs", "mlp_ppo_grad_refs", "mlp_apply", blob_dev, ids, count,
                  params, actions, advantages, returns, fixed_log_probs, exps, refs, inv_batch, inv_ind, grad_out,
                  (cudaStream_t)stream);
}

extern "C" int upb_next_step_fused(upb_ctx* ctx) { return next_step_fused(ctx, &upb_ctx::sgnn); }
extern "C" int upb_mlp_next_step_fused(upb_ctx* ctx) { return next_step_fused(ctx, &upb_ctx::mlp); }

extern "C" int upb_rearm_clip(upb_ctx* ctx) { return rearm_clip(ctx, &upb_ctx::sgnn, "rearm_clip"); }
extern "C" int upb_mlp_rearm_clip(upb_ctx* ctx) { return rearm_clip(ctx, &upb_ctx::mlp, "mlp_rearm_clip"); }

extern "C" int upb_reset_kl_stop(upb_ctx* ctx, void* stream) {
  return reset_kl_stop(ctx, &upb_ctx::sgnn, "reset_kl_stop", (cudaStream_t)stream);
}
extern "C" int upb_mlp_reset_kl_stop(upb_ctx* ctx, void* stream) {
  return reset_kl_stop(ctx, &upb_ctx::mlp, "mlp_reset_kl_stop", (cudaStream_t)stream);
}

extern "C" int upb_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream) {
  return read_losses(ctx, &upb_ctx::sgnn, "read_losses", grad, out4_host, (cudaStream_t)stream);
}
extern "C" int upb_mlp_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream) {
  return read_losses(ctx, &upb_ctx::mlp, "mlp_read_losses", grad, out4_host, (cudaStream_t)stream);
}

extern "C" int upb_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host) {
  return get_opt_state(ctx, &upb_ctx::sgnn, "get_opt_state", m_host, v_host, steps4_host);
}
extern "C" int upb_mlp_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host) {
  return get_opt_state(ctx, &upb_ctx::mlp, "mlp_get_opt_state", m_host, v_host, steps4_host);
}

extern "C" int upb_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host, const int64_t* steps4_host) {
  return set_opt_state(ctx, &upb_ctx::sgnn, "set_opt_state", m_host, v_host, steps4_host);
}
extern "C" int upb_mlp_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host, const int64_t* steps4_host) {
  return set_opt_state(ctx, &upb_ctx::mlp, "mlp_set_opt_state", m_host, v_host, steps4_host);
}

extern "C" int upb_grad_norms(upb_ctx* ctx, const float* grad_rows, int rows, float* out, void* stream) {
  return grad_norms(ctx, &upb_ctx::sgnn, "grad_norms", grad_rows, rows, out, (cudaStream_t)stream);
}
extern "C" int upb_mlp_grad_norms(upb_ctx* ctx, const float* grad_rows, int rows, float* out, void* stream) {
  return grad_norms(ctx, &upb_ctx::mlp, "mlp_grad_norms", grad_rows, rows, out, (cudaStream_t)stream);
}

// ---- multi-GPU fused step: exchange buffers shared between the ranks' processes with CUDA IPC ---------------------------
static_assert(sizeof(cudaIpcMemHandle_t) == UPB_PEER_HANDLE_BYTES, "IPC handle size");

extern "C" int upb_peer_export(upb_ctx* ctx, void* handle_out) {
  if (int rc = check_ctx(ctx, "peer_export")) return rc;
  if (!handle_out) return set_error(UPB_ERR_ARG, "peer_export: handle_out is null");
  cudaIpcMemHandle_t h;
  UPB_CUDA(cudaIpcGetMemHandle(&h, ctx->xchg));
  memcpy(handle_out, &h, sizeof(h));
  return UPB_OK;
}

extern "C" int upb_peer_connect(upb_ctx* ctx, int world, int rank, const void* handles) {
  if (int rc = check_ctx(ctx, "peer_connect")) return rc;
  if (world < 2 || world > MAX_PEERS || rank < 0 || rank >= world || !handles)
    return set_error(UPB_ERR_ARG, "peer_connect: need 2 <= world <= 16, 0 <= rank < world and world handles");
  if (!ctx->xchg) return set_error(UPB_ERR_ARG, "peer_connect: call upb_peer_export first");
  if (!ctx->peer_ptrs.empty()) return set_error(UPB_ERR_ARG, "peer_connect: already connected");
  if (!ctx->coop) return set_error(UPB_ERR_CUDA, "peer_connect: cooperative launch is not supported on this device");
  std::vector<void*> ptrs(world, nullptr);
  for (int p = 0; p < world; ++p) {
    if (p == rank) { ptrs[p] = ctx->xchg; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + (size_t)p * sizeof(h), sizeof(h));
    cudaError_t err = cudaIpcOpenMemHandle(&ptrs[p], h, cudaIpcMemLazyEnablePeerAccess);
    if (err != cudaSuccess) {
      for (int q = 0; q < p; ++q)
        if (q != rank && ptrs[q]) cudaIpcCloseMemHandle(ptrs[q]);
      char buf[256];
      snprintf(buf, sizeof(buf), "peer_connect: cudaIpcOpenMemHandle(rank %d) failed: %s", p, cudaGetErrorString(err));
      cudaGetLastError();
      return set_error(UPB_ERR_CUDA, buf);
    }
  }
  // sequence numbers restart at 1 on every rank: forget the flags of earlier single-GPU steps.  The caller runs a
  // collective after this call and before the first fused step (Engine.connect_peers), so no peer can push into this
  // buffer before it is cleared.
  UPB_CUDA(cudaDeviceSynchronize());
  UPB_CUDA(cudaMemset(ctx->xchg + XCHG_FLAGS, 0, sizeof(float) * (XCHG_FLOATS - XCHG_FLAGS)));
  UPB_CUDA(cudaMemcpy(ctx->peers_dev, ptrs.data(), sizeof(float*) * world, cudaMemcpyHostToDevice));
  UPB_CUDA(cudaDeviceSynchronize());
  ctx->peer_ptrs = ptrs;
  ctx->world = world;
  ctx->rank = rank;
  ctx->peer_seq = 0;
  return UPB_OK;
}

extern "C" int upb_peer_timeouts(upb_ctx* ctx, int64_t* count) {
  if (int rc = check_ctx(ctx, "peer_timeouts")) return rc;
  if (!count) return set_error(UPB_ERR_ARG, "peer_timeouts: count is null");
  unsigned int n = 0;
  UPB_CUDA(cudaMemcpy(&n, ctx->gridbar + 6, sizeof(n), cudaMemcpyDeviceToHost));
  *count = (int64_t)n;
  return UPB_OK;
}

extern "C" int upb_gae(upb_ctx* ctx, const float* rewards, const float* masks, const float* values, int T,
                       float gamma, float tau, float* advantages, float* returns, void* stream) {
  if (int rc = check_ctx(ctx, "gae")) return rc;
  if (!rewards || !masks || !values || !advantages || !returns || T < 0) return set_error(UPB_ERR_ARG, "gae: bad argument");
  if (T == 0) return UPB_OK;
  const float gamma_tau = (float)((double)gamma * (double)tau);
  k_gae<<<(T + 255) / 256, 256, 0, (cudaStream_t)stream>>>(rewards, masks, values, T, gamma, gamma_tau, advantages,
                                                           returns);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_gae_targets(upb_ctx* ctx, const float* rewards, const float* masks, const float* head_values, int T,
                               float gamma, float tau, float* advantages, float* returns, float* anchors, void* stream) {
  return gae_targets(ctx, &upb_ctx::sgnn, "gae_targets", rewards, masks, head_values, T, gamma, tau, advantages, returns,
                     anchors, (cudaStream_t)stream);
}
extern "C" int upb_mlp_gae_targets(upb_ctx* ctx, const float* rewards, const float* masks, const float* head_values,
                                   int T, float gamma, float tau, float* advantages, float* returns, float* anchors,
                                   void* stream) {
  return gae_targets(ctx, &upb_ctx::mlp, "mlp_gae_targets", rewards, masks, head_values, T, gamma, tau, advantages,
                     returns, anchors, (cudaStream_t)stream);
}

// upb_set_param_groups keeps its fp32 weight decays; the tables take the double of each
static int set_param_groups_f32(upb_ctx* ctx, ModelOf model, const char* who, const double* lr,
                                const float* weight_decay, const uint8_t* trained, int n_tensors) {
  std::vector<double> wd(weight_decay && n_tensors > 0 && n_tensors <= PG_MAX_TENSORS ? n_tensors : 0);
  for (size_t t = 0; t < wd.size(); ++t) wd[t] = weight_decay[t];
  return set_param_groups(ctx, model, who, lr, wd.empty() ? nullptr : wd.data(), trained, nullptr, n_tensors);
}
extern "C" int upb_set_param_groups(upb_ctx* ctx, const double* lr, const float* weight_decay, const uint8_t* trained,
                                    int n_tensors) {
  return set_param_groups_f32(ctx, &upb_ctx::sgnn, "set_param_groups", lr, weight_decay, trained, n_tensors);
}
extern "C" int upb_mlp_set_param_groups(upb_ctx* ctx, const double* lr, const float* weight_decay,
                                        const uint8_t* trained, int n_tensors) {
  return set_param_groups_f32(ctx, &upb_ctx::mlp, "mlp_set_param_groups", lr, weight_decay, trained, n_tensors);
}
extern "C" int upb_set_param_groups_adam(upb_ctx* ctx, const double* lr, const double* weight_decay,
                                         const uint8_t* trained, const float* beta1, const float* beta2,
                                         const float* eps, const uint8_t* amsgrad, const uint8_t* decoupled,
                                         int n_tensors) {
  return set_param_groups_adam(ctx, &upb_ctx::sgnn, "set_param_groups_adam", lr, weight_decay, trained, beta1, beta2,
                               eps, amsgrad, decoupled, n_tensors);
}
extern "C" int upb_mlp_set_param_groups_adam(upb_ctx* ctx, const double* lr, const double* weight_decay,
                                             const uint8_t* trained, const float* beta1, const float* beta2,
                                             const float* eps, const uint8_t* amsgrad, const uint8_t* decoupled,
                                             int n_tensors) {
  return set_param_groups_adam(ctx, &upb_ctx::mlp, "mlp_set_param_groups_adam", lr, weight_decay, trained, beta1,
                               beta2, eps, amsgrad, decoupled, n_tensors);
}
extern "C" int upb_get_amsgrad_state(upb_ctx* ctx, float* max_exp_avg_sq, int n) {
  if (!max_exp_avg_sq) return has_amsgrad_state(ctx, &upb_ctx::sgnn, "get_amsgrad_state");
  return amsgrad_state(ctx, &upb_ctx::sgnn, "get_amsgrad_state", max_exp_avg_sq, nullptr, n);
}
extern "C" int upb_mlp_get_amsgrad_state(upb_ctx* ctx, float* max_exp_avg_sq, int n) {
  if (!max_exp_avg_sq) return has_amsgrad_state(ctx, &upb_ctx::mlp, "mlp_get_amsgrad_state");
  return amsgrad_state(ctx, &upb_ctx::mlp, "mlp_get_amsgrad_state", max_exp_avg_sq, nullptr, n);
}
extern "C" int upb_set_amsgrad_state(upb_ctx* ctx, const float* max_exp_avg_sq, int n) {
  return amsgrad_state(ctx, &upb_ctx::sgnn, "set_amsgrad_state", nullptr, max_exp_avg_sq, n);
}
extern "C" int upb_mlp_set_amsgrad_state(upb_ctx* ctx, const float* max_exp_avg_sq, int n) {
  return amsgrad_state(ctx, &upb_ctx::mlp, "mlp_set_amsgrad_state", nullptr, max_exp_avg_sq, n);
}
extern "C" int upb_get_tensor_steps(upb_ctx* ctx, int64_t* steps, int n_tensors) {
  return tensor_steps(ctx, &upb_ctx::sgnn, "get_tensor_steps", steps, nullptr, n_tensors);
}
extern "C" int upb_mlp_get_tensor_steps(upb_ctx* ctx, int64_t* steps, int n_tensors) {
  return tensor_steps(ctx, &upb_ctx::mlp, "mlp_get_tensor_steps", steps, nullptr, n_tensors);
}
extern "C" int upb_set_tensor_steps(upb_ctx* ctx, const int64_t* steps, int n_tensors) {
  return tensor_steps(ctx, &upb_ctx::sgnn, "set_tensor_steps", nullptr, steps, n_tensors);
}
extern "C" int upb_mlp_set_tensor_steps(upb_ctx* ctx, const int64_t* steps, int n_tensors) {
  return tensor_steps(ctx, &upb_ctx::mlp, "mlp_set_tensor_steps", nullptr, steps, n_tensors);
}

// a context with a parameter-group table takes each tensor's lr and weight decay from it
static int refuse_with_param_groups(const upb_ctx* ctx, const char* who) {
  if (ctx->sgnn.pg_user || ctx->mlp.pg_user)
    return set_error(UPB_ERR_ARG, std::string(who) + ": the context has parameter groups (upb_set_param_groups), "
                                                     "which set every tensor's lr, weight decay and Adam settings");
  return UPB_OK;
}

extern "C" int upb_set_adam(upb_ctx* ctx, float beta1, float beta2, float eps, int amsgrad, int decoupled) {
  if (int rc = check_ctx(ctx, "set_adam")) return rc;
  if (int rc = refuse_with_param_groups(ctx, "set_adam")) return rc;
  if (int rc = check_adam("set_adam", beta1, beta2, eps)) return rc;
  ctx->adam = {beta1, beta2, eps, amsgrad != 0, decoupled != 0};
  return refresh_context_tables(ctx);
}

extern "C" int upb_set_weight_decay(upb_ctx* ctx, float weight_decay) {
  if (int rc = check_ctx(ctx, "set_weight_decay")) return rc;
  if (int rc = refuse_with_param_groups(ctx, "set_weight_decay")) return rc;
  if (!std::isfinite(weight_decay) || weight_decay < 0.f)
    return set_error(UPB_ERR_ARG, "set_weight_decay: weight_decay must be finite and >= 0");
  ctx->weight_decay = weight_decay;
  ctx->weight_decay_d = weight_decay;
  return refresh_context_tables(ctx);
}

extern "C" int upb_set_weight_decay_double(upb_ctx* ctx, double weight_decay) {
  if (int rc = check_ctx(ctx, "set_weight_decay_double")) return rc;
  if (int rc = refuse_with_param_groups(ctx, "set_weight_decay_double")) return rc;
  if (!std::isfinite(weight_decay) || weight_decay < 0.0 || !std::isfinite((float)weight_decay))
    return set_error(UPB_ERR_ARG, "set_weight_decay_double: weight_decay must be finite and >= 0");
  ctx->weight_decay = (float)weight_decay;
  ctx->weight_decay_d = weight_decay;
  return refresh_context_tables(ctx);
}

extern "C" int upb_set_lr(upb_ctx* ctx, double lr) {
  if (int rc = check_ctx(ctx, "set_lr")) return rc;
  if (int rc = refuse_with_param_groups(ctx, "set_lr")) return rc;
  if (!std::isfinite(lr) || lr < 0.0) return set_error(UPB_ERR_ARG, "set_lr: lr must be finite and >= 0");
  ctx->lr = lr;
  if (int rc = refresh_context_tables(ctx)) return rc;
  if (int rc = seed_lr_state(ctx, ctx->sgnn)) return rc;
  return seed_lr_state(ctx, ctx->mlp);
}

extern "C" int upb_set_loss_coefs(upb_ctx* ctx, float value_pred_coef, float entropy_coef) {
  if (int rc = check_ctx(ctx, "set_loss_coefs")) return rc;
  if (!std::isfinite(value_pred_coef) || !std::isfinite(entropy_coef))
    return set_error(UPB_ERR_ARG, "set_loss_coefs: value_pred_coef and entropy_coef must be finite");
  ctx->value_pred_coef = value_pred_coef;
  ctx->entropy_coef = entropy_coef;
  return UPB_OK;
}

extern "C" int upb_set_target_kl(upb_ctx* ctx, float target_kl) {
  if (int rc = check_ctx(ctx, "set_target_kl")) return rc;
  if (!std::isfinite(target_kl) || target_kl < 0.f)
    return set_error(UPB_ERR_ARG, "set_target_kl: target_kl must be finite and >= 0");
  // Stable-Baselines3's convention: stop once approx_kl > 1.5 * target_kl
  ctx->kl_limit = (float)(1.5 * (double)target_kl);
  return UPB_OK;
}

extern "C" int upb_set_adaptive_lr(upb_ctx* ctx, double desired_kl, double lr_min, double lr_max) {
  if (int rc = check_ctx(ctx, "set_adaptive_lr")) return rc;
  if (desired_kl == 0.0) {
    ctx->desired_kl = 0.0;
    return UPB_OK;
  }
  const float up = (float)(desired_kl / 2.0), down = (float)(2.0 * desired_kl);
  if (!std::isfinite(desired_kl) || !(desired_kl > 0.0) || !(up > 0.f) || !std::isfinite(down))
    return set_error(UPB_ERR_ARG, "set_adaptive_lr: desired_kl must be 0 (off) or finite and > 0, with fp32 thresholds "
                                  "desired_kl / 2 > 0 and 2 desired_kl finite");
  if (!std::isfinite(lr_min) || !std::isfinite(lr_max) || !(lr_min > 0.0) || !(lr_min <= lr_max))
    return set_error(UPB_ERR_ARG, "set_adaptive_lr: need finite bounds with 0 < lr_min <= lr_max");
  const bool was_on = ctx->desired_kl > 0.0;
  ctx->desired_kl = desired_kl;
  ctx->lr_up = up;
  ctx->lr_down = down;
  ctx->lr_min = lr_min;
  ctx->lr_max = lr_max;
  if (was_on) return UPB_OK;                 // the state carries on
  if (int rc = seed_lr_state(ctx, ctx->sgnn)) return rc;
  return seed_lr_state(ctx, ctx->mlp);
}

namespace {
// upb_get_lr_state / upb_set_lr_state: n = 1 (every entry) or the model's tensor count (one per tensor), in stream order
int lr_state(upb_ctx* ctx, ModelOf model, const char* who, double* get, const double* set, int n, cudaStream_t s) {
  if (int rc = check_ctx(ctx, who)) return rc;
  Model& m = ctx->*model;
  if (!(ctx->desired_kl > 0.0)) return set_error(UPB_ERR_ARG, std::string(who) + ": the adaptive lr is off");
  if (!(get || set) || !(n == 1 || n == m.num_tensors))
    return set_error(UPB_ERR_ARG, std::string(who) + ": need 1 or " + std::to_string(m.num_tensors) + " values");
  if (int rc = model_init(ctx, m)) return rc;
  double* cur = m.lr_state + PG_MAX_TENSORS * m.steps_cur;
  if (get) UPB_CUDA(cudaMemcpyAsync(get, cur, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  if (set) {
    double h[PG_MAX_TENSORS];
    for (int t = 0; t < PG_MAX_TENSORS; ++t) {
      h[t] = set[n == 1 ? 0 : (t < n ? t : 0)];
      if (t < n && (!std::isfinite(h[t]) || h[t] < 0.0))
        return set_error(UPB_ERR_ARG, std::string(who) + ": lr must be finite and >= 0");
    }
    UPB_CUDA(cudaMemcpyAsync(cur, h, sizeof(h), cudaMemcpyHostToDevice, s));
    UPB_CUDA(cudaStreamSynchronize(s));      // h lives on this stack frame
  }
  return UPB_OK;
}
}  // namespace

extern "C" int upb_get_lr_state(upb_ctx* ctx, double* lr, int n, void* stream) {
  return lr_state(ctx, &upb_ctx::sgnn, "get_lr_state", lr, nullptr, n, (cudaStream_t)stream);
}
extern "C" int upb_mlp_get_lr_state(upb_ctx* ctx, double* lr, int n, void* stream) {
  return lr_state(ctx, &upb_ctx::mlp, "mlp_get_lr_state", lr, nullptr, n, (cudaStream_t)stream);
}
extern "C" int upb_set_lr_state(upb_ctx* ctx, const double* lr, int n, void* stream) {
  return lr_state(ctx, &upb_ctx::sgnn, "set_lr_state", nullptr, lr, n, (cudaStream_t)stream);
}
extern "C" int upb_mlp_set_lr_state(upb_ctx* ctx, const double* lr, int n, void* stream) {
  return lr_state(ctx, &upb_ctx::mlp, "mlp_set_lr_state", nullptr, lr, n, (cudaStream_t)stream);
}

extern "C" int upb_set_clip_range(upb_ctx* ctx, float lo, float hi) {
  if (int rc = check_ctx(ctx, "set_clip_range")) return rc;
  if (!std::isfinite(lo) || !std::isfinite(hi) || lo > hi)
    return set_error(UPB_ERR_ARG, "set_clip_range: lo and hi must be finite with lo <= hi");
  ctx->clip_lo = lo;
  ctx->clip_hi = hi;
  return UPB_OK;
}

extern "C" int upb_set_value_clip(upb_ctx* ctx, float value_clip) {
  if (int rc = check_ctx(ctx, "set_value_clip")) return rc;
  if (!std::isfinite(value_clip) || value_clip < 0.f)
    return set_error(UPB_ERR_ARG, "set_value_clip: value_clip must be finite and >= 0");
  ctx->value_clip = value_clip;
  return UPB_OK;
}

extern "C" int upb_set_dual_clip(upb_ctx* ctx, float c) {
  if (int rc = check_ctx(ctx, "set_dual_clip")) return rc;
  if (!std::isfinite(c) || (c != 0.f && !(c > 1.f)))
    return set_error(UPB_ERR_ARG, "set_dual_clip: c must be 0 (off) or finite and > 1");
  ctx->dual_clip = c;
  return UPB_OK;
}

extern "C" int upb_set_prox_ewma(upb_ctx* ctx, int enable, float beta) {
  if (int rc = check_ctx(ctx, "set_prox_ewma")) return rc;
  if (enable && !(std::isfinite(beta) && beta >= 0.f && beta < 1.f))
    return set_error(UPB_ERR_ARG, "set_prox_ewma: beta must be finite, >= 0 and < 1");
  ctx->prox_on = enable != 0;
  ctx->prox_beta = enable ? beta : 0.f;
  return UPB_OK;
}
extern "C" int upb_get_prox_params(upb_ctx* ctx, float* params_host, int n) {
  return prox_params_host(ctx, &upb_ctx::sgnn, "get_prox_params", params_host, nullptr, n);
}
extern "C" int upb_mlp_get_prox_params(upb_ctx* ctx, float* params_host, int n) {
  return prox_params_host(ctx, &upb_ctx::mlp, "mlp_get_prox_params", params_host, nullptr, n);
}
extern "C" int upb_set_prox_params(upb_ctx* ctx, const float* params_host, int n) {
  return prox_params_host(ctx, &upb_ctx::sgnn, "set_prox_params", nullptr, params_host, n);
}
extern "C" int upb_mlp_set_prox_params(upb_ctx* ctx, const float* params_host, int n) {
  return prox_params_host(ctx, &upb_ctx::mlp, "mlp_set_prox_params", nullptr, params_host, n);
}
extern "C" int upb_init_prox_params(upb_ctx* ctx, const float* params_dev, void* stream) {
  return init_prox_params(ctx, &upb_ctx::sgnn, "init_prox_params", params_dev, (cudaStream_t)stream);
}
extern "C" int upb_mlp_init_prox_params(upb_ctx* ctx, const float* params_dev, void* stream) {
  return init_prox_params(ctx, &upb_ctx::mlp, "mlp_init_prox_params", params_dev, (cudaStream_t)stream);
}

extern "C" int upb_set_huber_delta(upb_ctx* ctx, float delta) {
  if (int rc = check_ctx(ctx, "set_huber_delta")) return rc;
  if (!std::isfinite(delta) || delta < 0.f)
    return set_error(UPB_ERR_ARG, "set_huber_delta: delta must be 0 (off) or finite and > 0");
  ctx->huber_delta = delta;
  return UPB_OK;
}

extern "C" int upb_set_max_grad_norm(upb_ctx* ctx, float max_norm) {
  if (int rc = check_ctx(ctx, "set_max_grad_norm")) return rc;
  if (!std::isfinite(max_norm) || max_norm < 0.f)
    return set_error(UPB_ERR_ARG, "set_max_grad_norm: max_norm must be finite and >= 0");
  if (max_norm > 0.f && ctx->cfg.clip_mode != UPB_CLIP_NEVER)
    return set_error(UPB_ERR_ARG, "set_max_grad_norm: the global clip needs clip_mode UPB_CLIP_NEVER (the two-group "
                                  "clip of the other modes would apply as well)");
  ctx->max_grad_norm = max_norm;
  return UPB_OK;
}

extern "C" int upb_set_nonfinite_guard(upb_ctx* ctx, int enable) {
  if (int rc = check_ctx(ctx, "set_nonfinite_guard")) return rc;
  ctx->nonfinite_guard = enable != 0;
  return UPB_OK;
}

extern "C" int upb_set_kl_penalty(upb_ctx* ctx, float beta) {
  if (int rc = check_ctx(ctx, "set_kl_penalty")) return rc;
  if (!std::isfinite(beta) || beta < 0.f) return set_error(UPB_ERR_ARG, "set_kl_penalty: beta must be finite and >= 0");
  ctx->kl_coef = beta;
  return UPB_OK;
}

extern "C" int upb_normalize_advantages(upb_ctx* ctx, const float* adv_in, const float* exps, const int32_t* order,
                                        int T_used, int B, float* adv_out, void* stream) {
  if (int rc = check_ctx(ctx, "normalize_advantages")) return rc;
  if (!adv_in || !exps || !order || !adv_out || T_used < 0 || B < 1)
    return set_error(UPB_ERR_ARG, "normalize_advantages: bad argument");
  const int nb = T_used / B;
  if (nb == 0) return UPB_OK;
  k_adv_norm<<<nb, AN_THREADS, 0, (cudaStream_t)stream>>>(adv_in, exps, order, B, adv_out);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_set_value_norm(upb_ctx* ctx, double beta) {
  if (int rc = check_ctx(ctx, "set_value_norm")) return rc;
  if (!std::isfinite(beta) || beta < 0.0 || beta >= 1.0)
    return set_error(UPB_ERR_ARG, "set_value_norm: beta must be finite with 0 <= beta < 1");
  ctx->value_norm_beta = beta;
  return UPB_OK;
}

extern "C" int upb_value_norm_denormalize(upb_ctx* ctx, const float* normalized, int T, float* values, void* stream) {
  return value_norm_denormalize(ctx, &upb_ctx::sgnn, "value_norm_denormalize", normalized, T, values,
                                (cudaStream_t)stream);
}
extern "C" int upb_mlp_value_norm_denormalize(upb_ctx* ctx, const float* normalized, int T, float* values,
                                              void* stream) {
  return value_norm_denormalize(ctx, &upb_ctx::mlp, "mlp_value_norm_denormalize", normalized, T, values,
                                (cudaStream_t)stream);
}

extern "C" int upb_value_norm_update(upb_ctx* ctx, const float* returns, const float* values, int T, float* params,
                                     float* norm_returns, float* norm_values, double* mean_std, void* stream) {
  return value_norm_update(ctx, &upb_ctx::sgnn, "value_norm_update", returns, values, T, params, norm_returns,
                           norm_values, mean_std, (cudaStream_t)stream);
}
extern "C" int upb_mlp_value_norm_update(upb_ctx* ctx, const float* returns, const float* values, int T, float* params,
                                         float* norm_returns, float* norm_values, double* mean_std, void* stream) {
  return value_norm_update(ctx, &upb_ctx::mlp, "mlp_value_norm_update", returns, values, T, params, norm_returns,
                           norm_values, mean_std, (cudaStream_t)stream);
}

extern "C" int upb_get_value_norm_state(upb_ctx* ctx, double* state3_host) {
  return get_value_norm_state(ctx, &upb_ctx::sgnn, "get_value_norm_state", state3_host);
}
extern "C" int upb_mlp_get_value_norm_state(upb_ctx* ctx, double* state3_host) {
  return get_value_norm_state(ctx, &upb_ctx::mlp, "mlp_get_value_norm_state", state3_host);
}
extern "C" int upb_set_value_norm_state(upb_ctx* ctx, const double* state3_host) {
  return set_value_norm_state(ctx, &upb_ctx::sgnn, "set_value_norm_state", state3_host);
}
extern "C" int upb_mlp_set_value_norm_state(upb_ctx* ctx, const double* state3_host) {
  return set_value_norm_state(ctx, &upb_ctx::mlp, "mlp_set_value_norm_state", state3_host);
}

extern "C" int upb_set_diagnostics(upb_ctx* ctx, int enable) {
  if (int rc = check_ctx(ctx, "set_diagnostics")) return rc;
  ctx->diagnostics = enable != 0;
  return UPB_OK;
}

extern "C" int upb_profile_enable(upb_ctx* ctx, int enable) {
  if (int rc = check_ctx(ctx, "profile_enable")) return rc;
  ctx->profiling = enable != 0;
  return UPB_OK;
}

extern "C" int upb_profile_read(upb_ctx* ctx, double* total_ms, int* launches) {
  if (int rc = check_ctx(ctx, "profile_read")) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  double tot = 0.0;
  for (size_t i = 0; i < ctx->prof_used; ++i) {
    float ms = 0.f;
    UPB_CUDA(cudaEventElapsedTime(&ms, ctx->prof_events[i].first, ctx->prof_events[i].second));
    tot += ms;
  }
  if (total_ms) *total_ms = tot;
  if (launches) *launches = (int)ctx->prof_used;
  ctx->prof_used = 0;
  return UPB_OK;
}

extern "C" int upb_grid_size(const upb_ctx* ctx) { return ctx ? ctx->grid : 0; }

extern "C" int upb_set_stamp_buffer(upb_ctx* ctx, void* stamps_dev) {
  if (int rc = check_ctx(ctx, "set_stamp_buffer")) return rc;
  ctx->stamps = (long long*)stamps_dev;
  return UPB_OK;
}

extern "C" int64_t upb_launch_count(const upb_ctx* ctx) { return ctx ? ctx->launches : 0; }
