// C-ABI implementation (include/upb200.h): context, launches, optimiser state.
#include <cuda_runtime.h>

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

struct upb_ctx {
  upb_config cfg;
  int num_sms = 0;
  int grid = 0;
  float* gpart = nullptr;       // [grid][G_ROW]
  float* gsum = nullptr;        // [G_ROW] (two-call path: k_reduce_finish)
  float* scratch = nullptr;     // [grid][scratch_stride]
  size_t scratch_stride = 0;
  float* adam_m = nullptr;
  float* adam_v = nullptr;
  long long* steps = nullptr;   // device [2][4] ping-pong step counters
  int steps_cur = 0;
  unsigned int* ticket = nullptr;
  unsigned int* gridbar = nullptr;   // [8] fused tail: cumulative arrival counter, stage bits by parity, peer-timeout count
  unsigned int bar_total = 0;        // arrivals at gridbar[0] so far (the counter is never reset)
  int64_t host_steps = 0;            // optimiser steps applied so far (mirrors the device counter)
  bool clip_armed = true;            // UPB_CLIP_REFERENCE: the next step is the process's first one and clips (SURVEY A.6-2)
  int coop = 0;                      // cooperative launch supported
  float* host_pinned = nullptr; // [UPB_STAT_COUNT] pinned staging for upb_read_losses
  int64_t launches = 0;
  bool profiling = false;
  long long* stamps = nullptr;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
  size_t prof_used = 0;
  // rl-mlp ablation model: its own partial rows, scratch, Adam state and step counters (allocated on first use)
  float* m_gpart = nullptr;
  float* m_scratch = nullptr;
  size_t m_scratch_stride = 0;
  float* m_adam_m = nullptr;
  float* m_adam_v = nullptr;
  long long* m_steps = nullptr;
  int m_steps_cur = 0;
  bool m_clip_armed = true;
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

int check_ctx(const upb_ctx* ctx, const char* who) {
  if (!ctx) return set_error(UPB_ERR_ARG, std::string(who) + ": null context");
  return UPB_OK;
}

// event pair bracketing the fused kernel while profiling is on (events are pooled and reused)
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

bool clip_now(const upb_ctx* ctx) {
  return ctx->cfg.clip_mode == UPB_CLIP_ALWAYS || (ctx->cfg.clip_mode == UPB_CLIP_REFERENCE && ctx->clip_armed);
}
bool mlp_clip_now(const upb_ctx* ctx) {      // the rl-mlp model keeps its own first-step latch
  return ctx->cfg.clip_mode == UPB_CLIP_ALWAYS || (ctx->cfg.clip_mode == UPB_CLIP_REFERENCE && ctx->m_clip_armed);
}

StepArgs base_args(upb_ctx* ctx, const void* blob, const int32_t* ids, int count, const float* params,
                   const float* actions) {
  StepArgs a;
  memset(&a, 0, sizeof(a));
  a.blob = (const uint8_t*)blob;
  a.ids = ids;
  a.count = count;
  a.params = params;
  a.actions = actions;
  a.clip_eps = ctx->cfg.clip_epsilon;
  a.c_value = ctx->cfg.value_pred_coef;
  a.c_entropy = ctx->cfg.entropy_coef;
  a.gpart = ctx->gpart;
  a.scratch = ctx->scratch;
  a.scratch_stride = ctx->scratch_stride;
  a.n_cap = ctx->cfg.n_cap;
  a.e_cap = ctx->cfg.e_cap;
  a.stamps = ctx->stamps;
  return a;
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
  ctx->num_sms = prop.multiProcessorCount;
  ctx->grid = ctx->num_sms;
  if (cfg->grid_limit > 0 && cfg->grid_limit < ctx->grid) ctx->grid = cfg->grid_limit;
  ctx->scratch_stride = (scratch_floats(cfg->n_cap, cfg->e_cap) + 63) & ~size_t(63);
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
  UPB_CUDA_F(cudaMalloc(&ctx->gpart, sizeof(float) * (size_t)ctx->grid * G_ROW));
  UPB_CUDA_F(cudaMalloc(&ctx->gsum, sizeof(float) * G_ROW));
  UPB_CUDA_F(cudaMalloc(&ctx->scratch, sizeof(float) * (size_t)ctx->grid * ctx->scratch_stride));
  UPB_CUDA_F(cudaMalloc(&ctx->adam_m, sizeof(float) * NUM_PARAMS));
  UPB_CUDA_F(cudaMalloc(&ctx->adam_v, sizeof(float) * NUM_PARAMS));
  UPB_CUDA_F(cudaMalloc(&ctx->steps, sizeof(long long) * 8));
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
  UPB_CUDA_F(cudaMemset(ctx->adam_m, 0, sizeof(float) * NUM_PARAMS));
  UPB_CUDA_F(cudaMemset(ctx->adam_v, 0, sizeof(float) * NUM_PARAMS));
  UPB_CUDA_F(cudaMemset(ctx->steps, 0, sizeof(long long) * 8));
  UPB_CUDA_F(cudaMemset(ctx->scratch, 0, sizeof(float) * (size_t)ctx->grid * ctx->scratch_stride));
  UPB_CUDA_F(cudaMallocHost(&ctx->host_pinned, sizeof(float) * UPB_STAT_COUNT));
  UPB_CUDA_F(cudaFuncSetAttribute(k_sgnn<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  UPB_CUDA_F(cudaFuncSetAttribute(k_sgnn<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  UPB_CUDA_F(cudaDeviceSynchronize());
#undef UPB_CUDA_F
  *out = ctx;
  return UPB_OK;
}

extern "C" void upb_destroy(upb_ctx* ctx) {
  if (!ctx) return;
  cudaFree(ctx->gpart);
  cudaFree(ctx->gsum);
  cudaFree(ctx->scratch);
  cudaFree(ctx->adam_m);
  cudaFree(ctx->adam_v);
  cudaFree(ctx->steps);
  cudaFree(ctx->ticket);
  cudaFree(ctx->gridbar);
  cudaFree(ctx->m_gpart);
  cudaFree(ctx->m_scratch);
  cudaFree(ctx->m_adam_m);
  cudaFree(ctx->m_adam_v);
  cudaFree(ctx->m_steps);
  for (int p = 0; p < (int)ctx->peer_ptrs.size(); ++p)
    if (p != ctx->rank && ctx->peer_ptrs[p]) cudaIpcCloseMemHandle(ctx->peer_ptrs[p]);
  cudaFree(ctx->peers_dev);
  cudaFree(ctx->xchg);
  if (ctx->host_pinned) cudaFreeHost(ctx->host_pinned);
  for (auto& ev : ctx->prof_events) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
  delete ctx;
}

extern "C" int upb_forward(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                           const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                           void* stream) {
  if (int rc = check_ctx(ctx, "forward")) return rc;
  if (!blob_dev || !params || count < 0) return set_error(UPB_ERR_ARG, "forward: bad argument");
  if (count == 0) return UPB_OK;
  StepArgs a = base_args(ctx, blob_dev, ids, count, params, actions);
  a.out_value = value;
  a.out_logp = log_prob;
  a.out_entropy = entropy;
  a.out_greedy = greedy;
  const int grid = count < ctx->grid ? count : ctx->grid;
  const bool prof = prof_begin(ctx, (cudaStream_t)stream);
  k_sgnn<false><<<grid, NT, SMEM_BYTES, (cudaStream_t)stream>>>(a);
  prof_end(ctx, (cudaStream_t)stream, prof);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                                 const float* uniforms, int32_t* action_index, void* stream) {
  if (int rc = check_ctx(ctx, "select_action")) return rc;
  if (!blob_dev || !params || !action_index || count < 0) return set_error(UPB_ERR_ARG, "select_action: bad argument");
  if (count == 0) return UPB_OK;
  StepArgs a = base_args(ctx, blob_dev, ids, count, params, nullptr);
  if (uniforms) { a.uniforms = uniforms; a.out_sample = action_index; }
  else a.out_greedy = action_index;
  const int grid = count < ctx->grid ? count : ctx->grid;
  k_sgnn<false><<<grid, NT, SMEM_BYTES, (cudaStream_t)stream>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                            const float* actions, const float* advantages, const float* returns,
                            const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                            float* grad_out, void* stream) {
  if (int rc = check_ctx(ctx, "ppo_grad")) return rc;
  if (!blob_dev || !params || !actions || !advantages || !returns || !fixed_log_probs || !exps || !grad_out ||
      count < 0)
    return set_error(UPB_ERR_ARG, "ppo_grad: bad argument");
  cudaStream_t s = (cudaStream_t)stream;
  StepArgs a = base_args(ctx, blob_dev, ids, count, params, actions);
  a.adv = advantages;
  a.ret = returns;
  a.fixed_lp = fixed_log_probs;
  a.exps = exps;
  a.inv_batch = inv_batch;
  a.inv_ind = inv_ind;
  int grid = count < ctx->grid ? count : ctx->grid;
  if (grid > 0) {
    const bool prof = prof_begin(ctx, s);
    k_sgnn<true><<<grid, NT, SMEM_BYTES, s>>>(a);
    prof_end(ctx, s, prof);
    ctx->launches += 1;
  }
  k_reduce_finish<<<RF_BLOCKS, RF_THREADS, 0, s>>>(ctx->gpart, grid, ctx->gsum, params, grad_out, ctx->ticket);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_apply(upb_ctx* ctx, float* params, const float* grad, void* stream) {
  if (int rc = check_ctx(ctx, "apply")) return rc;
  if (!params || !grad) return set_error(UPB_ERR_ARG, "apply: bad argument");
  ApplyArgs a;
  a.params = params;
  a.grad = grad;
  a.m = ctx->adam_m;
  a.v = ctx->adam_v;
  a.steps_in = ctx->steps + 4 * ctx->steps_cur;
  a.steps_out = ctx->steps + 4 * (1 - ctx->steps_cur);
  ctx->steps_cur = 1 - ctx->steps_cur;
  ctx->host_steps += 1;
  a.lr = ctx->cfg.lr;
  a.beta1 = ctx->cfg.beta1;
  a.beta2 = ctx->cfg.beta2;
  a.eps = ctx->cfg.adam_eps;
  a.clip_now = clip_now(ctx) ? 1 : 0;
  ctx->clip_armed = false;
  a.num_params = NUM_PARAMS; a.encoder_end = ENCODER_END; a.policy_end = POLICY_END;
  a.lu_begin = P_LU_W0; a.rd_begin = P_RD_W0; a.stat_offset = UPB_STAT_OFFSET;
  k_apply<<<AP_BLOCKS, AP_THREADS, 0, (cudaStream_t)stream>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                            const float* actions, const float* advantages, const float* returns,
                            const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                            float* grad_out, void* stream) {
  if (int rc = check_ctx(ctx, "ppo_step")) return rc;
  const bool clip_step = clip_now(ctx);
  if (ctx->world > 1) {
    if (clip_step || !ctx->coop)
      return set_error(UPB_ERR_ARG, "ppo_step: peers are connected and this step clips gradients; use upb_ppo_grad + "
                                    "all-reduce + upb_apply for it (upb_next_step_fused() == 0)");
  } else if (clip_step || !ctx->coop || count <= 0) {      // clipping needs a grid-wide norm first: use the two-call path
    int rc = upb_ppo_grad(ctx, blob_dev, ids, count, params, actions, advantages, returns, fixed_log_probs, exps,
                          inv_batch, inv_ind, grad_out, stream);
    if (rc != UPB_OK) return rc;
    return upb_apply(ctx, params, grad_out, stream);
  }
  if (!blob_dev || !params || !actions || !advantages || !returns || !fixed_log_probs || !exps || !grad_out)
    return set_error(UPB_ERR_ARG, "ppo_step: bad argument");
  cudaStream_t s = (cudaStream_t)stream;
  StepArgs a = base_args(ctx, blob_dev, ids, count, params, actions);
  a.adv = advantages;
  a.ret = returns;
  a.fixed_lp = fixed_log_probs;
  a.exps = exps;
  a.inv_batch = inv_batch;
  a.inv_ind = inv_ind;
  a.fuse_tail = 1;
  a.params_rw = params;
  a.grad_out = grad_out;
  a.adam_m = ctx->adam_m;
  a.adam_v = ctx->adam_v;
  a.steps_in = ctx->steps + 4 * ctx->steps_cur;
  a.steps_out = ctx->steps + 4 * (1 - ctx->steps_cur);
  a.gridbar = ctx->gridbar;
  a.lr = ctx->cfg.lr;
  a.beta1 = ctx->cfg.beta1;
  a.beta2 = ctx->cfg.beta2;
  a.adam_eps = ctx->cfg.adam_eps;
  a.world = ctx->world;
  a.rank = ctx->rank;
  a.seq = ++ctx->peer_seq;
  a.peers = ctx->peers_dev;
  const int grid = count < 1 ? 1 : (count < ctx->grid ? count : ctx->grid);     // an empty shard still takes part in the exchange
  ctx->bar_total += (unsigned int)grid;
  a.bar_target = ctx->bar_total;
  void* kargs[] = {&a};
  const bool prof = prof_begin(ctx, s);
  UPB_CUDA(cudaLaunchCooperativeKernel((void*)k_sgnn<true>, dim3(grid), dim3(NT), kargs, SMEM_BYTES, s));
  prof_end(ctx, s, prof);
  ctx->launches += 1;
  ctx->steps_cur = 1 - ctx->steps_cur;
  ctx->host_steps += 1;
  return UPB_OK;
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

extern "C" int upb_next_step_fused(upb_ctx* ctx) {
  if (!ctx) return 0;
  return (!clip_now(ctx) && ctx->coop) ? 1 : 0;
}

// ---- rl-mlp ablation model ---------------------------------------------------------------------------------------------
namespace {
int mlp_init(upb_ctx* ctx) {
  if (ctx->m_gpart) return UPB_OK;
  ctx->m_scratch_stride = (mlp_scratch_floats(ctx->cfg.n_cap, ctx->cfg.e_cap) + 63) & ~size_t(63);
  UPB_CUDA(cudaMalloc(&ctx->m_gpart, sizeof(float) * (size_t)ctx->grid * MG_ROW));
  UPB_CUDA(cudaMalloc(&ctx->m_scratch, sizeof(float) * (size_t)ctx->grid * ctx->m_scratch_stride));
  UPB_CUDA(cudaMalloc(&ctx->m_adam_m, sizeof(float) * M_NUM_PARAMS));
  UPB_CUDA(cudaMalloc(&ctx->m_adam_v, sizeof(float) * M_NUM_PARAMS));
  UPB_CUDA(cudaMalloc(&ctx->m_steps, sizeof(long long) * 8));
  UPB_CUDA(cudaMemset(ctx->m_adam_m, 0, sizeof(float) * M_NUM_PARAMS));
  UPB_CUDA(cudaMemset(ctx->m_adam_v, 0, sizeof(float) * M_NUM_PARAMS));
  UPB_CUDA(cudaMemset(ctx->m_steps, 0, sizeof(long long) * 8));
  UPB_CUDA(cudaMemset(ctx->m_scratch, 0, sizeof(float) * (size_t)ctx->grid * ctx->m_scratch_stride));
  UPB_CUDA(cudaFuncSetAttribute(k_mlp<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)M_SMEM_BYTES));
  UPB_CUDA(cudaFuncSetAttribute(k_mlp<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)M_SMEM_BYTES));
  UPB_CUDA(cudaDeviceSynchronize());
  return UPB_OK;
}
StepArgs mlp_args(upb_ctx* ctx, const void* blob, const int32_t* ids, int count, const float* params,
                  const float* actions) {
  StepArgs a = base_args(ctx, blob, ids, count, params, actions);
  a.gpart = ctx->m_gpart;
  a.scratch = ctx->m_scratch;
  a.scratch_stride = ctx->m_scratch_stride;
  return a;
}
}  // namespace

extern "C" int upb_mlp_forward(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                               const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                               void* stream) {
  if (int rc = check_ctx(ctx, "mlp_forward")) return rc;
  if (!blob_dev || !params || count < 0) return set_error(UPB_ERR_ARG, "mlp_forward: bad argument");
  if (int rc = mlp_init(ctx)) return rc;
  if (count == 0) return UPB_OK;
  StepArgs a = mlp_args(ctx, blob_dev, ids, count, params, actions);
  a.out_value = value; a.out_logp = log_prob; a.out_entropy = entropy; a.out_greedy = greedy;
  const int grid = count < ctx->grid ? count : ctx->grid;
  k_mlp<false><<<grid, MT, M_SMEM_BYTES, (cudaStream_t)stream>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_mlp_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count,
                                     const float* params, const float* uniforms, int32_t* action_index, void* stream) {
  if (int rc = check_ctx(ctx, "mlp_select_action")) return rc;
  if (!blob_dev || !params || !action_index || count < 0) return set_error(UPB_ERR_ARG, "mlp_select_action: bad argument");
  if (int rc = mlp_init(ctx)) return rc;
  if (count == 0) return UPB_OK;
  StepArgs a = mlp_args(ctx, blob_dev, ids, count, params, nullptr);
  if (uniforms) { a.uniforms = uniforms; a.out_sample = action_index; }
  else a.out_greedy = action_index;
  const int grid = count < ctx->grid ? count : ctx->grid;
  k_mlp<false><<<grid, MT, M_SMEM_BYTES, (cudaStream_t)stream>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_mlp_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                                const float* actions, const float* advantages, const float* returns,
                                const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                                float* grad_out, void* stream) {
  if (int rc = check_ctx(ctx, "mlp_ppo_grad")) return rc;
  if (!blob_dev || !params || !actions || !advantages || !returns || !fixed_log_probs || !exps || !grad_out || count < 0)
    return set_error(UPB_ERR_ARG, "mlp_ppo_grad: bad argument");
  if (int rc = mlp_init(ctx)) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  StepArgs a = mlp_args(ctx, blob_dev, ids, count, params, actions);
  a.adv = advantages; a.ret = returns; a.fixed_lp = fixed_log_probs; a.exps = exps;
  a.inv_batch = inv_batch; a.inv_ind = inv_ind;
  const int grid = count < ctx->grid ? count : ctx->grid;
  if (grid > 0) {
    const bool prof = prof_begin(ctx, s);
    k_mlp<true><<<grid, MT, M_SMEM_BYTES, s>>>(a);
    prof_end(ctx, s, prof);
    ctx->launches += 1;
  }
  k_mlp_reduce<<<(MG_ROW + 255) / 256, 256, 0, s>>>(ctx->m_gpart, grid, grad_out);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_mlp_apply(upb_ctx* ctx, float* params, const float* grad, void* stream) {
  if (int rc = check_ctx(ctx, "mlp_apply")) return rc;
  if (!params || !grad) return set_error(UPB_ERR_ARG, "mlp_apply: bad argument");
  if (int rc = mlp_init(ctx)) return rc;
  ApplyArgs a;
  a.params = params; a.grad = grad; a.m = ctx->m_adam_m; a.v = ctx->m_adam_v;
  a.steps_in = ctx->m_steps + 4 * ctx->m_steps_cur;
  a.steps_out = ctx->m_steps + 4 * (1 - ctx->m_steps_cur);
  ctx->m_steps_cur = 1 - ctx->m_steps_cur;
  a.lr = ctx->cfg.lr; a.beta1 = ctx->cfg.beta1; a.beta2 = ctx->cfg.beta2; a.eps = ctx->cfg.adam_eps;
  a.clip_now = mlp_clip_now(ctx) ? 1 : 0;
  ctx->m_clip_armed = false;
  a.num_params = M_NUM_PARAMS; a.encoder_end = M_ENCODER_END; a.policy_end = M_POLICY_END;
  a.lu_begin = M_LU_W0; a.rd_begin = M_RD_W0; a.stat_offset = UPB_MLP_STAT_OFFSET;
  k_apply<<<AP_BLOCKS, AP_THREADS, 0, (cudaStream_t)stream>>>(a);
  ctx->launches += 1;
  UPB_CUDA(cudaGetLastError());
  return UPB_OK;
}

extern "C" int upb_mlp_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                                const float* actions, const float* advantages, const float* returns,
                                const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                                float* grad_out, void* stream) {
  if (int rc = check_ctx(ctx, "mlp_ppo_step")) return rc;
  if (ctx->world > 1)
    return set_error(UPB_ERR_ARG, "mlp_ppo_step: peers are connected; rl-mlp multi-GPU steps use upb_mlp_ppo_grad + "
                                  "all-reduce + upb_mlp_apply");
  if (mlp_clip_now(ctx) || !ctx->coop || count <= 0) {     // clipping needs a grid-wide norm first: two-call path
    int rc = upb_mlp_ppo_grad(ctx, blob_dev, ids, count, params, actions, advantages, returns, fixed_log_probs, exps,
                              inv_batch, inv_ind, grad_out, stream);
    if (rc != UPB_OK) return rc;
    return upb_mlp_apply(ctx, params, grad_out, stream);
  }
  if (!blob_dev || !params || !actions || !advantages || !returns || !fixed_log_probs || !exps || !grad_out)
    return set_error(UPB_ERR_ARG, "mlp_ppo_step: bad argument");
  if (int rc = mlp_init(ctx)) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  StepArgs a = mlp_args(ctx, blob_dev, ids, count, params, actions);
  a.adv = advantages; a.ret = returns; a.fixed_lp = fixed_log_probs; a.exps = exps;
  a.inv_batch = inv_batch; a.inv_ind = inv_ind;
  a.fuse_tail = 1;
  a.params_rw = params;
  a.grad_out = grad_out;
  a.adam_m = ctx->m_adam_m;
  a.adam_v = ctx->m_adam_v;
  a.steps_in = ctx->m_steps + 4 * ctx->m_steps_cur;
  a.steps_out = ctx->m_steps + 4 * (1 - ctx->m_steps_cur);
  a.gridbar = ctx->gridbar;
  a.lr = ctx->cfg.lr; a.beta1 = ctx->cfg.beta1; a.beta2 = ctx->cfg.beta2; a.adam_eps = ctx->cfg.adam_eps;
  a.world = ctx->world;
  a.rank = ctx->rank;
  a.seq = ++ctx->peer_seq;           // one sequence / parity / barrier count for the fused steps of both models
  a.peers = ctx->peers_dev;
  const int grid = count < ctx->grid ? count : ctx->grid;
  ctx->bar_total += (unsigned int)grid;
  a.bar_target = ctx->bar_total;
  void* kargs[] = {&a};
  const bool prof = prof_begin(ctx, s);
  UPB_CUDA(cudaLaunchCooperativeKernel((void*)k_mlp<true>, dim3(grid), dim3(MT), kargs, M_SMEM_BYTES, s));
  prof_end(ctx, s, prof);
  ctx->launches += 1;
  ctx->m_steps_cur = 1 - ctx->m_steps_cur;
  ctx->m_clip_armed = false;
  return UPB_OK;
}

extern "C" int upb_mlp_next_step_fused(upb_ctx* ctx) {
  if (!ctx) return 0;
  return (ctx->world == 1 && !mlp_clip_now(ctx) && ctx->coop) ? 1 : 0;
}

extern "C" int upb_mlp_rearm_clip(upb_ctx* ctx) {
  if (int rc = check_ctx(ctx, "mlp_rearm_clip")) return rc;
  ctx->m_clip_armed = true;
  return UPB_OK;
}

namespace {
int read_losses_at(upb_ctx* ctx, const float* stats_dev, float* out4_host, cudaStream_t s) {
  UPB_CUDA(cudaMemcpyAsync(ctx->host_pinned, stats_dev, sizeof(float) * 8, cudaMemcpyDeviceToHost, s));
  UPB_CUDA(cudaStreamSynchronize(s));
  const float* st = ctx->host_pinned;
  const float nB = st[3] > 0.f ? st[3] : 1.f, nI = st[4] > 0.f ? st[4] : 1.f;
  const float value_loss = st[0] / nB, surr = st[1] / nI, ent = st[2] / nI;
  out4_host[0] = surr + ctx->cfg.value_pred_coef * value_loss + ctx->cfg.entropy_coef * ent;
  out4_host[1] = value_loss;
  out4_host[2] = surr;
  out4_host[3] = ent;
  return UPB_OK;
}
}  // namespace

extern "C" int upb_mlp_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream) {
  if (int rc = check_ctx(ctx, "mlp_read_losses")) return rc;
  if (!grad || !out4_host) return set_error(UPB_ERR_ARG, "mlp_read_losses: bad argument");
  return read_losses_at(ctx, grad + UPB_MLP_STAT_OFFSET, out4_host, (cudaStream_t)stream);
}

extern "C" int upb_mlp_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host) {
  if (int rc = check_ctx(ctx, "mlp_get_opt_state")) return rc;
  if (int rc = mlp_init(ctx)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (m_host) UPB_CUDA(cudaMemcpy(m_host, ctx->m_adam_m, sizeof(float) * M_NUM_PARAMS, cudaMemcpyDeviceToHost));
  if (v_host) UPB_CUDA(cudaMemcpy(v_host, ctx->m_adam_v, sizeof(float) * M_NUM_PARAMS, cudaMemcpyDeviceToHost));
  if (steps4_host)
    UPB_CUDA(cudaMemcpy(steps4_host, ctx->m_steps + 4 * ctx->m_steps_cur, sizeof(long long) * 4, cudaMemcpyDeviceToHost));
  return UPB_OK;
}

extern "C" int upb_mlp_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host, const int64_t* steps4_host) {
  if (int rc = check_ctx(ctx, "mlp_set_opt_state")) return rc;
  if (int rc = mlp_init(ctx)) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (m_host) UPB_CUDA(cudaMemcpy(ctx->m_adam_m, m_host, sizeof(float) * M_NUM_PARAMS, cudaMemcpyHostToDevice));
  if (v_host) UPB_CUDA(cudaMemcpy(ctx->m_adam_v, v_host, sizeof(float) * M_NUM_PARAMS, cudaMemcpyHostToDevice));
  if (steps4_host) {
    UPB_CUDA(cudaMemcpy(ctx->m_steps + 4 * ctx->m_steps_cur, steps4_host, sizeof(long long) * 4, cudaMemcpyHostToDevice));
    ctx->m_clip_armed = steps4_host[0] == 0;
  }
  return UPB_OK;
}

extern "C" int upb_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream) {
  if (int rc = check_ctx(ctx, "read_losses")) return rc;
  if (!grad || !out4_host) return set_error(UPB_ERR_ARG, "read_losses: bad argument");
  cudaStream_t s = (cudaStream_t)stream;
  UPB_CUDA(cudaMemcpyAsync(ctx->host_pinned, grad + UPB_STAT_OFFSET, sizeof(float) * 8, cudaMemcpyDeviceToHost, s));
  UPB_CUDA(cudaStreamSynchronize(s));
  const float* st = ctx->host_pinned;
  const float nB = st[3] > 0.f ? st[3] : 1.f, nI = st[4] > 0.f ? st[4] : 1.f;
  const float value_loss = st[0] / nB, surr = st[1] / nI, ent = st[2] / nI;
  out4_host[0] = surr + ctx->cfg.value_pred_coef * value_loss + ctx->cfg.entropy_coef * ent;
  out4_host[1] = value_loss;
  out4_host[2] = surr;
  out4_host[3] = ent;
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

extern "C" int upb_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host) {
  if (int rc = check_ctx(ctx, "get_opt_state")) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (m_host) UPB_CUDA(cudaMemcpy(m_host, ctx->adam_m, sizeof(float) * NUM_PARAMS, cudaMemcpyDeviceToHost));
  if (v_host) UPB_CUDA(cudaMemcpy(v_host, ctx->adam_v, sizeof(float) * NUM_PARAMS, cudaMemcpyDeviceToHost));
  if (steps4_host)
    UPB_CUDA(cudaMemcpy(steps4_host, ctx->steps + 4 * ctx->steps_cur, sizeof(long long) * 4, cudaMemcpyDeviceToHost));
  return UPB_OK;
}

extern "C" int upb_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host,
                                 const int64_t* steps4_host) {
  if (int rc = check_ctx(ctx, "set_opt_state")) return rc;
  UPB_CUDA(cudaDeviceSynchronize());
  if (m_host) UPB_CUDA(cudaMemcpy(ctx->adam_m, m_host, sizeof(float) * NUM_PARAMS, cudaMemcpyHostToDevice));
  if (v_host) UPB_CUDA(cudaMemcpy(ctx->adam_v, v_host, sizeof(float) * NUM_PARAMS, cudaMemcpyHostToDevice));
  if (steps4_host) {
    UPB_CUDA(cudaMemcpy(ctx->steps + 4 * ctx->steps_cur, steps4_host, sizeof(long long) * 4, cudaMemcpyHostToDevice));
    ctx->host_steps = steps4_host[0];
    ctx->clip_armed = steps4_host[0] == 0;
  }
  return UPB_OK;
}

extern "C" int upb_rearm_clip(upb_ctx* ctx) {
  if (int rc = check_ctx(ctx, "rearm_clip")) return rc;
  ctx->clip_armed = true;
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
