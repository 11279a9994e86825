/*
 * upb200.h -- C ABI of the H100-native PPO-update path for DRL-urban-planning.
 *
 * The reference (tsinghua-fib-lab/DRL-urban-planning) is pure Python and has no FFI; its "operator
 * interface" for this path is Python duck typing between UrbanPlanningAgent and two nn.Modules
 * (SURVEY.md section 8(b)).  Every entry point below names the reference call site it replaces.
 * Conventions: every function returns 0 on success and a negative upb_status otherwise (never aborts,
 * never throws); upb_last_error() gives the message of the calling thread's last failure.  All tensor
 * arguments are caller-owned raw pointers (device pointers unless the name says `host`), never freed or
 * retained past the call.  `stream` is a cudaStream_t passed as void* (0 = legacy default stream).
 * A context belongs to one (process, device) and is not thread-safe; do not use it in a forked child
 * (the reference forks rollout workers at khrylib/rl/agents/agent.py:83-89).
 */
#ifndef UPB200_H_
#define UPB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UPB_ABI_VERSION 1

/* model dimensions: fixed by every shipped config (the yaml files under cfg/exp_cfg: state_encoder_specs,
 * policy_specs, value_specs); other shapes are rejected by the host layer. */
#define UPB_NODE_DIM 23
#define UPB_NODE_STRIDE 24      /* node-feature rows are stored padded to 24 floats (16-byte aligned rows) */
#define UPB_NUMERICAL_DIM 52
#define UPB_GCN_DIM 16
#define UPB_NUM_GCN_LAYERS 2
#define UPB_NUM_PARAMS 13729
#define UPB_GRAD_STRIDE 13760   /* flat gradient buffer: 13,729 gradients, 3 pad, then UPB_STAT_COUNT statistics */
#define UPB_STAT_OFFSET 13732
#define UPB_STAT_COUNT 28
/* statistics layout inside the gradient buffer (all sums over the graphs this rank processed, so a
 * sum-allreduce of the whole buffer yields global values):
 *   [0] sum (V-R)^2            [1] sum over ind of -min(r A, clip(r) A)   [2] sum over ind of -entropy
 *   [3] #graphs                [4] #graphs in ind                          [5] #graphs stage land_use
 *   [6] #graphs stage road     [7] #non-finite per-graph results (NaN guard)            */

/* rl-mlp ablation model (create_mlp_model, urban_planning/models/model.py:22-33): its own flat layout, 18 tensors */
#define UPB_MLP_NUM_PARAMS 10257
#define UPB_MLP_STAT_OFFSET 10260
#define UPB_MLP_GRAD_STRIDE 10288   /* 10,257 gradients, 3 pad, UPB_STAT_COUNT statistics (same meaning as above) */

typedef enum {
  UPB_OK = 0,
  UPB_ERR_ARG = -1,        /* bad argument */
  UPB_ERR_CUDA = -2,       /* a CUDA call failed */
  UPB_ERR_FORMAT = -3,     /* a state violates the layout contract (see upb_pack_measure) */
  UPB_ERR_CAPACITY = -4    /* more graphs / larger graphs than the context was created for */
} upb_status;

typedef enum {
  UPB_CLIP_REFERENCE = 0,  /* clip (policy group, then value group, max-norm 1) on the first step of the
                              context's lifetime only: khrylib/rl/agents/agent_ppo.py:43-46 consumes the two
                              parameters() generators made at urban_planning_agent.py:46 (SURVEY A.6-2) */
  UPB_CLIP_ALWAYS = 1,     /* the same two-group clip on every step */
  UPB_CLIP_NEVER = 2
} upb_clip_mode;

typedef struct upb_ctx upb_ctx;

typedef struct {
  int32_t device;          /* CUDA device ordinal */
  int32_t n_cap, e_cap;    /* largest padded widths (max_num_nodes / max_num_edges of the cfg) */
  int32_t max_graphs;      /* most graphs one launch may touch */
  float lr, beta1, beta2, adam_eps;                 /* urban_planning_agent.py:145-149; hlg.yaml:34-36 */
  float clip_epsilon, value_pred_coef, entropy_coef; /* hlg.yaml:37-39 */
  int32_t clip_mode;       /* upb_clip_mode */
  int32_t grid_limit;      /* 0 = one CTA per SM; otherwise cap on CTAs (tests) */
} upb_config;

/* ---------------------------------------------------------------- library / layout */
int upb_abi_version(void);
const char* upb_last_error(void);
int upb_num_params(void);
/* i-th tensor of the flat parameter vector, in ActorCritic.parameters() order (models/model.py:36-47).
 * `name` receives the short name used by drl_urban_planning_b200/params.py. */
int upb_param_slot(int i, const char** name, int* offset, int* rows, int* cols);

/* ---------------------------------------------------------------- host-side packing (no CUDA)
 * Replaces tensorfy + SGNNStateEncoder.batch_data (urban_planning_agent.py:16-20,
 * models/state_encoder.py:163-177): turns `count` states in the reference's padded 9-array layout
 * (envs/observation_extractor.py:207-228) into one contiguous unpadded blob (DESIGN.md "packed blob").
 * state_arrays[9*i + j] points at array j of state i:
 *   0 numerical f32[52]   1 node_features f32[n_cap*23]   2 edge_index i64[e_cap*2]   3 current_node f32[23]
 *   4 node_mask u8[n_cap] 5 edge_mask u8[e_cap]           6 land_use_mask u8[e_cap]  7 road_mask u8[n_cap]
 *   8 stage f32[3]
 * Contract checked here (UPB_ERR_FORMAT otherwise): masks 4/5 are prefix masks, real edges join real nodes,
 * action masks lie on real edges/nodes, stage is one-hot on 'land_use' or 'road', n >= 1.
 * upb_pack_measure returns the blob size; upb_pack_fill writes it (blob must be 16-byte aligned).
 * `threads` <= 0 picks the hardware concurrency. */
int upb_pack_measure(int count, const void* const* state_arrays, int n_cap, int e_cap, int threads,
                     uint64_t* blob_bytes);
int upb_pack_fill(int count, const void* const* state_arrays, int n_cap, int e_cap, int threads,
                  void* blob_host, uint64_t blob_bytes);
/* Chunked packing for large buffers (a whole iteration's rollout states, ~1 GB): plan once, then fill the states
 * [first, first + count) chunk by chunk.  Every fill returns the byte ranges of the blob it has completed -- ranges[9][2]
 * = {offset, length}: [0] header + descriptor table (first chunk only), [1..8] the x, numerical, current-node, rowptr,
 * order, adj, cand_uv, cand_idx sections -- so the caller can start the host -> device copies of a chunk while the next
 * chunk is being packed (PackedGraphs.pack_and_upload).  The result equals upb_pack_fill's byte for byte. */
typedef struct upb_pack_plan upb_pack_plan;
int upb_pack_plan_create(int count, const void* const* state_arrays, int n_cap, int e_cap, int threads,
                         upb_pack_plan** plan_out, uint64_t* blob_bytes);
int upb_pack_plan_fill(upb_pack_plan* plan, const void* const* state_arrays, int first, int count, int threads,
                       void* blob_host, uint64_t blob_bytes, uint64_t* ranges);
void upb_pack_plan_destroy(upb_pack_plan* plan);

/* per-graph (n, e, k, stage) of a packed host blob, 4 ints per graph (for tests and load balancing) */
int upb_blob_info(const void* blob_host, uint64_t blob_bytes, int* count, int32_t* per_graph4);

/* ---------------------------------------------------------------- context */
int upb_create(const upb_config* cfg, upb_ctx** out);
void upb_destroy(upb_ctx* ctx);

/* ---------------------------------------------------------------- device path
 * Per-sample arrays (actions, advantages, returns, fixed_log_probs, exps and all outputs) are indexed by the
 * graph's position in the blob.  `ids` (device int32[count]) selects the graphs of this call -- a minibatch
 * is an index list into a resident blob; ids == NULL means graphs 0..count-1. */

/* No-grad pre-passes (urban_planning_agent.py:256-264 value_net(states); :283-292
 * policy_net.get_log_prob_entropy(states, actions)) and greedy select_action (models/policy.py:67-85,
 * mean_action=True).  actions: f32[(blob count)*2] as the reference stores them, or NULL (log_prob = 0).
 * Any output pointer may be NULL. */
int upb_forward(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                void* stream);

/* UrbanPlanningPolicy.select_action (urban_planning/models/policy.py:67-85) for a batch of packed graphs:
 * action_index[g] (indexed by blob position, like upb_forward's outputs) = index of the chosen land-use edge (stage 0
 * graphs) or road node (stage 1 graphs).
 *   uniforms == NULL : mean_action=True, `probs.argmax` with the first-index tie break (bit-exact);
 *   uniforms != NULL : mean_action=False, f32[blob count] uniforms in [0,1), one per graph; the action is the first
 *                      mask-true index whose cumulative probability reaches u (inverse CDF in index order).  torch's
 *                      Categorical.sample consumes its generator differently: sampled rollouts are reproducible per
 *                      uniform stream, not bit-equal to the reference's draws. */
int upb_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                      const float* uniforms, int32_t* action_index, void* stream);

/* Forward + backward of one (shard of a) minibatch: value_loss + ppo_entropy_loss + loss.backward()
 * (urban_planning_agent.py:330-335, khrylib/rl/agents/agent_pg.py:19-23).  inv_batch = 1/B and
 * inv_ind = 1/|ind| are those of the GLOBAL minibatch, so shards on several GPUs sum to the exact batch
 * gradient.  grad_out: f32[UPB_GRAD_STRIDE] = gradients + statistics (see above), overwritten. */
int upb_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                 const float* actions, const float* advantages, const float* returns,
                 const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                 float* grad_out, void* stream);

/* clip_policy_grad + optimizer.step (agent_ppo.py:43-46, urban_planning_agent.py:336-337) on the (already
 * all-reduced) gradient buffer.  Adam moments and step counters live in the context.  A policy head whose
 * stage count in the statistics is zero is skipped, as torch does for grad None (SURVEY A.6-7). */
int upb_apply(upb_ctx* ctx, float* params, const float* grad, void* stream);

/* upb_ppo_grad + upb_apply in ONE launch for the single-GPU case (urban_planning_agent.py:330-337): when the step does
 * not clip (every step but the first in UPB_CLIP_REFERENCE mode) the fused kernel ends with grid barriers, the
 * cross-CTA gradient reduction, the attention chain rule and Adam; otherwise it falls back to the two calls above.
 * grad_out still receives the gradient + statistics buffer.  Multi-GPU callers keep upb_ppo_grad / all-reduce /
 * upb_apply. */
int upb_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                 const float* actions, const float* advantages, const float* returns,
                 const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                 float* grad_out, void* stream);

/* ---- multi-GPU fused step (one process per GPU, peers on one node reachable over NVLink / NVSwitch or PCIe P2P) ----
 * The reference is single-process; data parallelism over the graphs of a minibatch is this library's extension
 * (SURVEY.md section 8e).  Without these calls the ranks exchange upb_ppo_grad's 55 KB buffer with ncclAllReduce and
 * call upb_apply.  With them the exchange happens inside upb_ppo_step's kernel through peer memory (every rank PUSHES
 * its slice sums into all ranks' buffers with remote stores and flags each slice; nobody loads over NVLink):
 *   upb_peer_export   writes UPB_PEER_HANDLE_BYTES bytes (a CUDA IPC handle of this context's exchange buffer);
 *   upb_peer_connect  takes the `world` handles gathered from all ranks in rank order and maps the peers' buffers;
 *                     afterwards every rank must call upb_ppo_step the same number of times (empty shards included);
 *   upb_next_step_fused  1 if the next optimiser step can run as upb_ppo_step (no gradient clipping on it), else 0:
 *                     a clipping step needs the global norm first and takes upb_ppo_grad + all-reduce + upb_apply.
 * All ranks sum the per-rank gradients in rank order, so their parameters stay bit-identical. */
#define UPB_PEER_HANDLE_BYTES 64
int upb_peer_export(upb_ctx* ctx, void* handle_out);
int upb_peer_connect(upb_ctx* ctx, int world, int rank, const void* handles);
int upb_next_step_fused(upb_ctx* ctx);
/* Number of CTAs that, in any fused step of this context so far, gave up waiting for a peer rank's gradient sums
 * (bounded polling instead of hanging the GPU).  Such a CTA SKIPS its Adam / parameter writes for that step, so no
 * stale peer data is ever applied; the count is sticky.  Non-zero means the ranks are out of sync: stop and restore a
 * checkpoint.  Synchronises the device (PPOUpdater checks it once per epoch). */
int upb_peer_timeouts(upb_ctx* ctx, int64_t* count);

/* ---- rl-mlp ablation (`train.py --agent rl-mlp`; MLPStateEncoder, urban_planning/models/state_encoder.py:217-308) ----
 * Same blob, same per-sample arrays and the same meaning of every argument as upb_forward / upb_ppo_grad / upb_apply,
 * on the MLP model's flat layout (UPB_MLP_*): params / grad are f32[UPB_MLP_NUM_PARAMS] / f32[UPB_MLP_GRAD_STRIDE].  The
 * context keeps a separate set of Adam moments and step counters for this model (upb_mlp_get/set_opt_state) and its own
 * first-step clip latch (upb_mlp_rearm_clip).  On one GPU a step is upb_mlp_ppo_step: one cooperative launch of the
 * k_mlp kernel that ends with the cross-CTA gradient reduction and Adam, bit-identical to upb_mlp_ppo_grad +
 * upb_mlp_apply, into which it falls back on steps that clip.  Several GPUs use upb_mlp_ppo_grad, an all-reduce of the
 * gradient buffer and upb_mlp_apply (there is no peer exchange for this model: upb_mlp_ppo_step refuses to run with
 * peers connected). */
int upb_mlp_forward(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                    const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                    void* stream);
int upb_mlp_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                          const float* uniforms, int32_t* action_index, void* stream);
int upb_mlp_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                     const float* actions, const float* advantages, const float* returns,
                     const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                     float* grad_out, void* stream);
int upb_mlp_apply(upb_ctx* ctx, float* params, const float* grad, void* stream);
/* upb_mlp_ppo_grad + upb_mlp_apply in ONE launch (same arguments as upb_ppo_step); grad_out receives the same buffer
 * upb_mlp_ppo_grad writes.  Falls back to the two calls when the step clips, when the device has no cooperative launch
 * or when count <= 0.  UPB_ERR_ARG with peers connected (upb_peer_connect). */
int upb_mlp_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                     const float* actions, const float* advantages, const float* returns,
                     const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                     float* grad_out, void* stream);
/* 1 if the next rl-mlp step runs as one launch (no clipping on it, cooperative launch available, no peers), else 0 */
int upb_mlp_next_step_fused(upb_ctx* ctx);
/* upb_rearm_clip for the rl-mlp model's latch: its next optimiser step clips (UPB_CLIP_REFERENCE) */
int upb_mlp_rearm_clip(upb_ctx* ctx);
int upb_mlp_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream);
int upb_mlp_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host);
int upb_mlp_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host, const int64_t* steps4_host);

/* the 4 scalars the reference logs per minibatch (urban_planning_agent.py:338-345), from a gradient buffer:
 * out4 = {loss, value_loss, surr_loss, entropy_loss}.  Synchronises `stream`. */
int upb_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream);

/* estimate_advantages (khrylib/rl/core/common.py:5-26): rewards f32[T], masks f32[T], values f32[T]
 * -> advantages f32[T], returns f32[T]; same fp32 operation order as the reference. */
int upb_gae(upb_ctx* ctx, const float* rewards, const float* masks, const float* values, int T, float gamma,
            float tau, float* advantages, float* returns, void* stream);

/* optimiser state for checkpoint/resume: m f32[UPB_NUM_PARAMS], v f32[UPB_NUM_PARAMS] (device or host
 * pointers), steps int64[4] = {global step, encoder+value step, land-use-head step, road-head step}. */
int upb_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host);
int upb_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host, const int64_t* steps4_host);
/* UPB_CLIP_REFERENCE clips on the first optimiser step of a PROCESS (the parameters() generators of
 * urban_planning_agent.py:46 are consumed by the first clip_grad_norm_ calls, agent_ppo.py:43-46).  A context starts
 * armed; upb_set_opt_state with a non-zero global step disarms it ("continue as if never interrupted");
 * upb_rearm_clip arms it again so that a run resumed from a checkpoint clips its first step like the reference does. */
int upb_rearm_clip(upb_ctx* ctx);

/* Kernel timing for the roofline line of bench.py: while enabled, upb_ppo_grad / upb_ppo_step / upb_forward bracket the
 * fused SGNN kernel, and upb_mlp_ppo_grad / upb_mlp_ppo_step the k_mlp kernel, with CUDA events on the launching stream.  upb_profile_read synchronises the device and returns the
 * summed duration (ms) and the number of bracketed launches since the last read. */
int upb_profile_enable(upb_ctx* ctx, int enable);
int upb_profile_read(upb_ctx* ctx, double* total_ms, int* launches);

/* CTAs the fused kernel is launched with (one per SM unless grid_limit is set).  Graph `ids[i]` of a call is walked by
 * CTA i % grid in round i / grid, so callers can balance the static schedule (see PPOUpdater.balance_ids). */
int upb_grid_size(const upb_ctx* ctx);

/* Debug: device int64[384] that receives clock64() stamps (phases of one graph, busy cycles per CTA) at the phase boundaries of the first graph walked by CTA 0
 * of every following fused-kernel launch (NULL switches it off).  See tools/phase_times.py. */
int upb_set_stamp_buffer(upb_ctx* ctx, void* stamps_dev);

/* number of kernels this context has launched so far (bench.py "gpu_launches") */
int64_t upb_launch_count(const upb_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* UPB200_H_ */
