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
 *   [6] #graphs stage road     [7] #non-finite per-graph results (NaN guard)
 *   [8] sum over ind of expm1(d) - d, d = log_prob - fixed_log_prob  (= (r-1) - log r, an estimate of KL(old||new))
 *   [9] sum over ind of 1 where the ratio r lies outside the clip range [lo, hi] (upb_set_clip_range; the surrogate's
 *       comparisons)
 *   [10] sum R                 [11] sum R^2                                [12] sum (V-R)
 *   [13] 1 on the step the KL stop ended (upb_set_target_kl)                [14] 1 on a step skipped after it
 *   [15] sum max(a, b), the clipped value loss (upb_set_value_clip)         [16] #graphs whose clipped branch won (b > a)
 *   [17] the fp32 pre-clip global gradient norm a step that applied Adam used (upb_set_max_grad_norm); not a sum
 *   [18] sum over ind of the exact KL_g = sum_c p_old(c) (lp_old(c) - lp(c)) over the graph's candidates
 *        (upb_set_kl_penalty)
 *   [19] 1 on a step the non-finite guard skipped (upb_set_nonfinite_guard); not a sum
 *   [20] #graphs in ind whose dual-clip bound c A was strictly active (upb_set_dual_clip)
 *   [21] #graphs whose chosen value-loss term is in Huber's linear branch, |e| > delta (upb_set_huber_delta)
 *   [22] the KL-adaptive lr's decision of the step, +1 up, -1 down, 0 none (upb_set_adaptive_lr); not a sum
 *   [23] sum over ind of the behaviour weight w = exp(lp_p - fixed_log_prob) (upb_set_prox_ewma)
 *   [24] sum over ind of expm1(d) - d, d = lp_p - fixed_log_prob, the behaviour-to-proximal KL estimate
 *        (upb_set_prox_ewma)
 * R is the return and V the value at the parameters the step starts from.  [9, 13) are filled only while
 * upb_set_diagnostics is on, [8] while diagnostics or the KL stop are on (otherwise zeros, the buffer of a context
 * without diagnostics); [13] and [14] are zeros while the KL stop is off; [15] and [16] are zeros while value clipping
 * is off; [17] is written by the optimiser step (upb_ppo_step, upb_apply; the reductions write 0) while the global clip
 * is on and is 0 otherwise, on a step that stops or is skipped included; [18] is zero while the KL penalty is off; [19]
 * is written by the optimiser step (the reductions write 0) and is 0 while the guard is off and on every step that
 * applied Adam, stopped on the KL criterion or was skipped after it; [20] is zero while dual clip is off and [21] while
 * the Huber value loss is off; [22] is 0 while the adaptive lr is off; [23] and [24] are zeros while the EWMA proximal policy is off and
 * [25, 28) are zeros.  [15] also holds the value loss the step optimised while the Huber
 * value loss is on.  [0] is sum (V-R)^2 whether or not the value loss is clipped or Huber.  A skipped step's buffer is all zeros but [14]; after an all-reduce over `world` ranks
 * its [14] is `world`. */

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
  float lr, beta1, beta2, adam_eps;                 /* urban_planning_agent.py:145-149; hlg.yaml:34-36.  lr is the
                                                       initial learning rate (upb_set_lr changes it) */
  float clip_epsilon, value_pred_coef, entropy_coef; /* hlg.yaml:37-39: the initial values (upb_set_clip_range,
                                                       upb_set_loss_coefs change them) */
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
 * Caps (UPB_ERR_ARG otherwise): 1 <= n_cap <= 65535 and 0 <= 2*e_cap <= 65535, as in upb_create.  Every state within
 * them is accepted whatever its candidate count: a land-use state has k <= e <= 32767 candidates, a road state
 * k <= n <= 65535 (all of them at n_cap = 65535 and e_cap = 32767).
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
/* upb_forward plus every candidate's log-probability: cand_log_prob (device f32[sum of the blob's k], the length of its
 * candidate section, or NULL) receives z_j - logsumexp(z) of candidate j of graph g at the graph's candidate position
 * (GraphDesc.cand_off + j, the order of cand_idx).  A graph larger than the context's caps gets NaN there, as its value
 * does; entries of graphs not listed in `ids` are left untouched.  upb_forward is this call with cand_log_prob = NULL.
 * The update's one pre-pass sweep thus yields the values, the fixed log-probs and the KL penalty's reference
 * log-probs (upb_set_kl_penalty) together. */
int upb_forward_cand(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                     const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                     float* cand_log_prob, void* stream);

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

/* UrbanPlanningPolicy.forward (urban_planning/models/policy.py:45-65): the masked logits the reference hands to
 * Categorical, written by the forward kernel's softmax warp.
 *   rows: int32[blob count], indexed by blob position: the graph's row in its stage's matrix, < 0 = none;
 *   land_use_logits: f32[*][cfg.e_cap], road_logits: f32[*][cfg.n_cap]; either may be NULL (rows of that stage are
 *   then not written).
 * A written row is -2^32+1 everywhere except at the mask-true candidates, which hold their logits; a graph larger
 * than the context's caps gets a row of NaN.  Rows of graphs not listed in `ids` are left untouched. */
int upb_policy_logits(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                      const int32_t* rows, float* land_use_logits, float* road_logits, void* stream);

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
 * stage count in the statistics is zero is skipped, as torch does for grad None (SURVEY A.6-7).  With the KL stop on
 * (upb_set_target_kl) a step whose statistics pass the criterion changes nothing but sets statistics slot 13 of
 * `grad` to 1 (the only write to `grad`) and the model's stop word. */
int upb_apply(upb_ctx* ctx, float* params, float* grad, void* stream);

/* upb_ppo_grad + upb_apply in ONE launch for the single-GPU case (urban_planning_agent.py:330-337): when the step does
 * not clip with the two-group clip (every step but the first in UPB_CLIP_REFERENCE mode) the fused kernel ends with grid
 * barriers, the cross-CTA gradient reduction, the attention chain rule and Adam; otherwise it falls back to the two calls
 * above.  The global clip (upb_set_max_grad_norm) stays in the one launch: Adam waits for the in-kernel norm.
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
 *   upb_next_step_fused  1 if the next optimiser step can run as upb_ppo_step (no two-group clip on it), else 0: such
 *                     a step needs the groups' norms first and takes upb_ppo_grad + all-reduce + upb_apply.  The
 *                     global clip (upb_set_max_grad_norm) keeps every step on upb_ppo_step.
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
int upb_mlp_forward_cand(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                         const float* actions, float* value, float* log_prob, float* entropy, int32_t* greedy,
                         float* cand_log_prob, void* stream);
int upb_mlp_select_action(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                          const float* uniforms, int32_t* action_index, void* stream);
int upb_mlp_policy_logits(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                          const int32_t* rows, float* land_use_logits, float* road_logits, void* stream);
int upb_mlp_ppo_grad(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                     const float* actions, const float* advantages, const float* returns,
                     const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                     float* grad_out, void* stream);
int upb_mlp_apply(upb_ctx* ctx, float* params, float* grad, void* stream);
/* upb_mlp_ppo_grad + upb_mlp_apply in ONE launch (same arguments as upb_ppo_step); grad_out receives the same buffer
 * upb_mlp_ppo_grad writes.  Falls back to the two calls when the step takes the two-group clip (not the global clip of
 * upb_set_max_grad_norm, which stays in the launch), when the device has no cooperative launch
 * or when count <= 0.  UPB_ERR_ARG with peers connected (upb_peer_connect). */
int upb_mlp_ppo_step(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                     const float* actions, const float* advantages, const float* returns,
                     const float* fixed_log_probs, const float* exps, float inv_batch, float inv_ind,
                     float* grad_out, void* stream);
/* 1 if the next rl-mlp step runs as one launch (no two-group clip on it, cooperative launch available, no peers), else 0 */
int upb_mlp_next_step_fused(upb_ctx* ctx);
/* upb_rearm_clip for the rl-mlp model's latch: its next optimiser step clips (UPB_CLIP_REFERENCE) */
int upb_mlp_rearm_clip(upb_ctx* ctx);
int upb_mlp_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream);
int upb_mlp_get_opt_state(upb_ctx* ctx, float* m_host, float* v_host, int64_t* steps4_host);
int upb_mlp_set_opt_state(upb_ctx* ctx, const float* m_host, const float* v_host, const int64_t* steps4_host);

/* the 4 scalars the reference logs per minibatch (urban_planning_agent.py:338-345), from a gradient buffer:
 * out4 = {loss, value_loss, surr_loss, entropy_loss}.  The loss is formed with the coefficients current at the read
 * (upb_set_loss_coefs).  Synchronises `stream`. */
int upb_read_losses(upb_ctx* ctx, const float* grad, float* out4_host, void* stream);

/* Pre-clip gradient norms of `rows` gradient buffers stored back to back (device f32[rows][UPB_GRAD_STRIDE], or
 * [rows][UPB_MLP_GRAD_STRIDE] for the rl-mlp call): out (device f32[rows][3]) receives per row the sums of squares over
 * the shared encoder, the policy heads and the value head -- the three groups the clip of upb_apply scales.  The
 * reference's two clip_grad_norm_ calls (agent_ppo.py:43-46) measure sqrt(encoder + policy) and sqrt(encoder + value).
 * Float64 sums in a fixed order: deterministic.  One launch on `stream`; no synchronisation. */
/* While enabled (default off), every later upb_ppo_grad / upb_ppo_step / upb_mlp_ppo_grad / upb_mlp_ppo_step of the
 * context also adds the PPO diagnostic sums, statistics slots 8-12 (see above).  Off, those slots are written as zeros
 * and the step does no extra work. */
int upb_set_diagnostics(upb_ctx* ctx, int enable);
int upb_grad_norms(upb_ctx* ctx, const float* grad_rows, int rows, float* out, void* stream);
int upb_mlp_grad_norms(upb_ctx* ctx, const float* grad_rows, int rows, float* out, void* stream);

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
/* torch.optim.Adam(..., weight_decay=cfg.weightdecay) (urban_planning_agent.py:145-149): coupled L2, not AdamW.  Every
 * later upb_apply / upb_ppo_step / upb_mlp_apply / upb_mlp_ppo_step of the context adds weight_decay * param (the value
 * before the step) to each live element's gradient, after the clip, so the clip norms do not include it.  A policy head
 * skipped for lack of its stage is not decayed.  The gradient buffer keeps the undecayed gradient.  Default 0 (off: the
 * arithmetic is exactly the undecayed one).  UPB_ERR_ARG for a negative or non-finite value. */
int upb_set_weight_decay(upb_ctx* ctx, float weight_decay);
/* upb_set_weight_decay from the double the caller holds: the coupled term uses (float)weight_decay, exactly as
 * upb_set_weight_decay((float)weight_decay) would, and the decoupled decay of upb_set_adam forms its factor
 * fp32(1 - lr * weight_decay) from the double, as torch does (upb_set_weight_decay keeps the fp32 value for both).
 * UPB_ERR_ARG as upb_set_weight_decay, and for a value whose fp32 rounding is not finite. */
int upb_set_weight_decay_double(upb_ctx* ctx, double weight_decay);
/* Adam's learning rate for both models, what a torch.optim.lr_scheduler on the reference's optimizer changes between
 * updates (urban_planning_agent.py:337 reads param_groups' lr at every optimizer.step()).  Every later optimiser step
 * (upb_apply, upb_ppo_step and its _vclip / _refs forms, and the rl-mlp counterparts) uses the value current when it was
 * issued.  torch keeps lr as a Python double and forms lr / bias_correction1 in double before it scales the fp32 update,
 * so the context keeps a double and every Adam tail forms its step size as (float)(lr / bc1).  upb_create sets it to
 * (double)cfg.lr.  lr = 0 is legal: the moments and step counters still advance (and weight decay still enters the
 * moments), the parameters do not move.  UPB_ERR_ARG for a negative or non-finite value. */
int upb_set_lr(upb_ctx* ctx, double lr);
/* The loss coefficients of both models: every later training step (upb_ppo_grad, upb_ppo_step and their _vclip / _refs
 * forms, and the rl-mlp counterparts) weighs the value loss by value_pred_coef and the entropy loss by entropy_coef
 * (urban_planning_agent.py:334), each launch with the values current when it was issued; upb_read_losses and
 * upb_mlp_read_losses use the values current at the read.  upb_create sets them to the cfg's.  Any finite value is
 * accepted; UPB_ERR_ARG for a non-finite one. */
int upb_set_loss_coefs(upb_ctx* ctx, float value_pred_coef, float entropy_coef);
/* Early stop of a PPO update on the approximate KL (Stable-Baselines3's `target_kl`), for both models.  With
 * target_kl > 0 every later optimiser step (upb_ppo_step, upb_apply and the rl-mlp counterparts) evaluates, on its
 * minibatch's globally reduced statistics (summed over CTAs and, on several GPUs, over ranks in rank order), before any
 * parameter is written:
 *     stop  iff  slot8 > limit * max(slot4, 1),   limit = (float)(1.5 * (double)target_kl)   (fp32 product)
 * A minibatch without an exps != 0 graph, or a NaN, never stops.  The stopping step writes its gradient buffer as
 * usual plus slot 13 = 1, but no parameter, Adam moment or step counter, and sets the model's stop word.  While the word
 * is set, every training step of that model (upb_ppo_step, upb_ppo_grad, upb_apply, rl-mlp likewise) returns at entry:
 * it changes no parameter, moment or counter and writes a buffer of zeros with slot 14 = 1.  The decision is made on
 * the device, so the host never synchronises for it; read slots 13 / 14 with the statistics.  0 turns the stop off
 * (the word is then ignored; outputs are those of a context that never set it).  UPB_ERR_ARG for a negative or
 * non-finite value.
 * upb_reset_kl_stop / upb_mlp_reset_kl_stop clear the model's word in stream order (the start of the next update).  The
 * word is not part of the optimiser state.  Several GPUs: every rank takes the same decisions; synchronise the ranks
 * (any collective) between a stop and the reset, as a new update does. */
int upb_set_target_kl(upb_ctx* ctx, float target_kl);
int upb_reset_kl_stop(upb_ctx* ctx, void* stream);
int upb_mlp_reset_kl_stop(upb_ctx* ctx, void* stream);
/* KL-adaptive learning rate (RSL-RL's schedule="adaptive" with desired_kl, rl_games' lr_schedule: adaptive), decided by
 * every optimiser step inside its kernels on the step's globally reduced statistics, the same slots 8 and 4 as the KL
 * stop, measured at the parameters the step starts from, in fp32 as the KL stop's criterion:
 *     down  iff  slot8 > fp32(2 desired_kl) * max(slot4, 1)
 *     up    iff  slot8 > 0 and slot8 < fp32(desired_kl / 2) * max(slot4, 1)
 * and no change otherwise (a NaN, a minibatch without an exps != 0 graph).  The new lr is formed in double, as torch keeps
 * it: max(lr_min, lr / 1.5) down, min(lr_max, lr * 1.5) up; no change leaves lr as it is, even outside the bounds.  The
 * same step applies the new lr: its step size (float)(lr / bc1) and a decoupled weight decay's factor fp32(1 - lr * wd)
 * are formed from it.  Each model keeps its lr state on the device: one lr, or one per tensor with parameter groups
 * (upb_set_param_groups*, or the table upb_set_adam synthesises), where every tensor's lr takes the same decision and is
 * clamped on its own and a frozen tensor's lr does not move.  A step that applies nothing -- a KL stop (decided first),
 * a step skipped after it, a non-finite step upb_set_nonfinite_guard skips, a peer give-up -- leaves the state unchanged
 * and its decision 0.  Statistics slot 22 holds the step's decision (+1, -1, 0), written once by the optimiser step (the
 * reductions write 0); slot 8 is filled while the option is on.  The state is seeded, in stream order on the legacy
 * default stream, when the option is turned on and by every later upb_set_lr / upb_set_param_groups*; other setters
 * leave it alone.  Turning the option off returns the steps to the lrs those calls set.  desired_kl = 0 turns it off
 * (outputs, launches and statistics are then those of a context that never set it); a second call while it is on
 * changes the thresholds and bounds and keeps the state.  UPB_ERR_ARG for a desired_kl that is negative, not finite, or
 * whose fp32 thresholds are 0 or infinite, and for bounds that are not finite or not 0 < lr_min <= lr_max.
 * upb_get_lr_state / upb_set_lr_state (upb_mlp_ twins): the lr state the next optimiser step reads, n = 1 (the first
 * tensor's; set: every tensor's) or the model's tensor count (upb_param_slot order), queued on `stream` (get: lr must
 * stay valid until the stream reaches the copy; pinned memory makes it asynchronous).  UPB_ERR_ARG while the option is
 * off, for another n, or (set) a negative or non-finite lr. */
int upb_set_adaptive_lr(upb_ctx* ctx, double desired_kl, double lr_min, double lr_max);
int upb_get_lr_state(upb_ctx* ctx, double* lr, int n, void* stream);
int upb_mlp_get_lr_state(upb_ctx* ctx, double* lr, int n, void* stream);
int upb_set_lr_state(upb_ctx* ctx, const double* lr, int n, void* stream);
int upb_mlp_set_lr_state(upb_ctx* ctx, const double* lr, int n, void* stream);
/* The surrogate's clip range [lo, hi] for both models: every later training step clamps the ratio r to it, and
 * statistics slot 9 counts the ratios outside it; each launch uses the range current when it was issued, so a clip epsilon
 * annealed between updates takes effect from the next step.  upb_create sets it to [1.f - clip_epsilon, 1.f + clip_epsilon],
 * formed in fp32 from the fp32 epsilon.  torch.clamp(ratio, 1.0 - eps, 1.0 + eps) (urban_planning_agent.py:368) forms
 * each bound in double from the Python float and rounds it once to fp32; for 47 of the 99 values eps = 0.01 ... 0.99
 * the two differ by one ulp (eps = 0.18: hi 1.1800001 instead of 1.18).  Callers holding eps as a double pass
 * lo = (float)(1.0 - eps) and hi = (float)(1.0 + eps) to follow the reference's comparisons exactly.  UPB_ERR_ARG for a
 * non-finite bound or lo > hi. */
int upb_set_clip_range(upb_ctx* ctx, float lo, float hi);

/* Clipped value loss (OpenAI baselines' ppo2, CleanRL's clip_vloss; not Stable-Baselines3's clip_range_vf, which has no
 * max) for both models.  With value_clip = c > 0 every later training step replaces the value loss mean (V - R)^2 by
 *     d = V - V_old,  Vc = V_old + clamp(d, -c, c),  a = (V - R)^2,  b = (Vc - R)^2,  value_loss = mean max(a, b)
 * over the minibatch's B graphs, in fp32 with torch's operations and order: the clamp bounds are +-(float)c (what
 * torch.clamp(x, -c, c) uses for a Python float c), value_pred_coef multiplies it as before.  V_old is the value the
 * update's pre-pass (upb_forward) computed for the graph, passed per call to the *_vclip entry points below and indexed
 * by blob position.  Its gradient is torch autograd's: per graph 2 (V - R) where a > b, 2 (Vc - R) [-c <= d <= c] where
 * b > a, and half the sum of the two on an exact tie (torch.maximum splits ties).  Statistics slot 15 receives sum
 * max(a, b) and slot 16 the number of graphs with b > a; slot 0 keeps sum (V - R)^2.  upb_read_losses /
 * upb_mlp_read_losses report the value loss from slot 15 while clipping is on.  0 turns it off (the default: outputs are
 * those of a context that never set it, whatever old_values is).  UPB_ERR_ARG for a negative or non-finite value. */
int upb_set_value_clip(upb_ctx* ctx, float value_clip);
/* Dual-clip PPO (Ye et al. 2020; Tianshou's PPOPolicy(dual_clip=c)) for both models.  With c > 1 every later training
 * step bounds the surrogate of a graph with exps != 0 and a negative advantage from below:
 *     s1 = r A,  s2 = clamp(r, lo, hi) A,  clip1 = min(s1, s2),  clip2 = max(clip1, c A),  surr = -(A < 0 ? clip2 : clip1)
 * in fp32 (c A is one fp32 product; A is the advantage the step receives, normalised or not).  Its gradient is torch
 * autograd's: c A carries none, so where c A > clip1 the graph's log-prob seed is 0, on an exact tie half the seed
 * without the option, otherwise that seed.  Statistics slot 1 receives the dual-clipped surrogate and slot 20 the number
 * of graphs with c A > clip1; slot 9 (the clip fraction) keeps its meaning.  c may change between steps; each launch
 * uses the value current when it was issued.  0 turns it off (the default: outputs are those of a context that never
 * set it).  UPB_ERR_ARG for a non-finite value or one other than 0 that is not above 1. */
int upb_set_dual_clip(upb_ctx* ctx, float c);
/* Huber value loss (MAPPO's use_huber_loss / huber_delta) for both models.  With delta > 0 every later training step
 * replaces each graph's squared error e^2, e = V - R, by
 *     h(e) = 2 torch.nn.functional.huber_loss(V, R, delta=delta) = e^2 for |e| < delta, 2 delta (|e| - delta / 2) beyond
 * in torch's fp32 operations (inside delta, bit for bit e * e), with the gradient 2 clamp(e, -delta, delta).  The value
 * seed keeps the order 2 value_pred_coef clamp(e, -delta, delta) (1 / B), so a delta above every |V - R| gives the step of
 * a context without the option bit for bit.  With value clipping (upb_set_value_clip) both terms are Huber terms:
 * max(h(V - R), h(Vc - R)), with the same tie and inclusive-clamp rules.  With value normalisation (upb_set_value_norm)
 * e is in the normalised units the head trains in.  The Huber loss is symmetric (not MAPPO's one-sided branch test).
 * Statistics slot 15 receives the sum of the value-loss terms the step optimised and slot 21 the number of graphs whose
 * chosen term (the unclipped one on a tie) has |e| > delta; slot 0 keeps sum (V - R)^2.  upb_read_losses /
 * upb_mlp_read_losses report the value loss from slot 15 while Huber or clipping is on.  0 turns it off (the default:
 * outputs are those of a context that never set it).  UPB_ERR_ARG for a negative or non-finite value. */
int upb_set_huber_delta(upb_ctx* ctx, float delta);

/* EWMA proximal policy (PPO-EWMA) for both models.  With enable != 0 and 0 <= beta < 1 every later training launch
 * (upb_ppo_grad, upb_ppo_step and their _vclip / _refs / _grad_noise forms, and the upb_mlp_ twins) decouples the
 * clip's anchor from the behaviour policy.  For each graph in ind, with lp its log-prob at the step's parameters, lp_b
 * its fixed_log_prob and lp_p its log-prob at the model's proximal parameters theta_prox:
 *     r = exp(lp - lp_p)      w = exp(lp_p - lp_b) (a constant: no gradient, not clipped)
 *     surrogate = -w min(r A, clamp(r, lo, hi) A)     (dual clip: -w (A < 0 ? max(clip1, c A) : clip1))
 * Where the clip is inactive the gradient with respect to lp is -A exp(lp - lp_b), ordinary PPO's.  The value loss, the
 * entropy and the KL penalty's reference (old_cand_log_probs) are unchanged; statistics slot 8 (the KL stop, the
 * adaptive lr, diagnostics) stays against lp_b, slots 9 and 20 count the branches of r, slots 23 and 24 sum w and the
 * behaviour-to-proximal KL estimate.  Each training launch first runs one forward launch at theta_prox over the same
 * ids (so one more launch per call; it does nothing while the KL stop word is set), into a context buffer of
 * max_graphs log-probs.  After every optimiser step that applies Adam (upb_ppo_step's fused tails, upb_apply), every
 * parameter element, frozen tensors and absent heads included, takes
 *     theta_prox <- fmaf(beta, theta_prox - theta_new, theta_new)
 * in the thread that writes it.  A step that applies nothing (KL stop, skipped after it, non-finite guard; the elements
 * a peer timeout skipped) leaves theta_prox unchanged; upb_value_norm_update does not touch it.  The average's mean
 * age is beta / (1 - beta) optimiser steps.  A training launch while the option is on and theta_prox was never set
 * returns UPB_ERR_ARG.  enable = 0 turns it off (the default: launches and outputs are those of a context that never
 * set it).  A beta outside [0, 1) or not finite: UPB_ERR_ARG. */
int upb_set_prox_ewma(upb_ctx* ctx, int enable, float beta);
/* theta_prox of the model: host copies of n floats, the model's parameter count (the flat layout), synchronous
 * (get: UPB_ERR_ARG while it was never set); init: theta_prox <- params (device), queued on `stream` without a host
 * synchronisation. */
int upb_get_prox_params(upb_ctx* ctx, float* params_host, int n);
int upb_mlp_get_prox_params(upb_ctx* ctx, float* params_host, int n);
int upb_set_prox_params(upb_ctx* ctx, const float* params_host, int n);
int upb_mlp_set_prox_params(upb_ctx* ctx, const float* params_host, int n);
int upb_init_prox_params(upb_ctx* ctx, const float* params_dev, void* stream);
int upb_mlp_init_prox_params(upb_ctx* ctx, const float* params_dev, void* stream);
/* upb_ppo_grad / upb_ppo_step / upb_mlp_ppo_grad / upb_mlp_ppo_step with the pre-pass values old_values (device
 * f32[blob count]); the four entry points above are these with old_values = NULL.  UPB_ERR_ARG when value clipping is on
 * and old_values is NULL; ignored while it is off. */
int upb_ppo_grad_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                       const float* actions, const float* advantages, const float* returns,
                       const float* fixed_log_probs, const float* exps, const float* old_values, float inv_batch,
                       float inv_ind, float* grad_out, void* stream);
int upb_ppo_step_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                       const float* actions, const float* advantages, const float* returns,
                       const float* fixed_log_probs, const float* exps, const float* old_values, float inv_batch,
                       float inv_ind, float* grad_out, void* stream);
int upb_mlp_ppo_grad_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                           const float* actions, const float* advantages, const float* returns,
                           const float* fixed_log_probs, const float* exps, const float* old_values, float inv_batch,
                           float inv_ind, float* grad_out, void* stream);
int upb_mlp_ppo_step_vclip(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                           const float* actions, const float* advantages, const float* returns,
                           const float* fixed_log_probs, const float* exps, const float* old_values, float inv_batch,
                           float inv_ind, float* grad_out, void* stream);
/* Reference data of the update's pre-pass that a training step may need, indexed as upb_forward_cand writes them (any
 * field may be NULL while its option is off, and is then ignored):
 *   old_values          device f32[blob count]: the pre-pass values (upb_set_value_clip)
 *   old_cand_log_probs  device f32[sum of the blob's k]: the pre-pass candidate log-probs of upb_forward_cand
 *                       (upb_set_kl_penalty)
 * The *_refs entry points are upb_ppo_grad / upb_ppo_step / upb_mlp_ppo_grad / upb_mlp_ppo_step with this struct; refs
 * may be NULL.  The plain entry points are these with refs = NULL, the *_vclip ones with {old_values, NULL}.  UPB_ERR_ARG
 * when an option is on and its field is NULL. */
typedef struct {
  const float* old_values;
  const float* old_cand_log_probs;
} upb_step_refs;
int upb_ppo_grad_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                      const float* actions, const float* advantages, const float* returns,
                      const float* fixed_log_probs, const float* exps, const upb_step_refs* refs, float inv_batch,
                      float inv_ind, float* grad_out, void* stream);
int upb_ppo_step_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                      const float* actions, const float* advantages, const float* returns,
                      const float* fixed_log_probs, const float* exps, const upb_step_refs* refs, float inv_batch,
                      float inv_ind, float* grad_out, void* stream);
int upb_mlp_ppo_grad_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                          const float* actions, const float* advantages, const float* returns,
                          const float* fixed_log_probs, const float* exps, const upb_step_refs* refs,
                          float inv_batch, float inv_ind, float* grad_out, void* stream);
int upb_mlp_ppo_step_refs(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, float* params,
                          const float* actions, const float* advantages, const float* returns,
                          const float* fixed_log_probs, const float* exps, const upb_step_refs* refs,
                          float inv_batch, float inv_ind, float* grad_out, void* stream);
/* Gradient noise scale measurement (McCandlish et al. 2018, "An Empirical Model of Large-Batch Training"): upb_ppo_grad_refs
 * / upb_mlp_ppo_grad_refs into grad_out, with the same arguments and effects, then one more launch over that gradient
 * launch's per-CTA partial rows and its reduced row, writing noise_out (device double[4]):
 *     [0] A = sum over the launch's CTAs c of |G_c|^2, G_c the partial gradient of the graphs CTA c processed
 *     [1] S = |g|^2, g the reduced (pre-clip) gradient in grad_out
 *     [2] Q = sum_c n_c^2, n_c the number of items CTA c took: with grid = min(count, upb_grid_size) CTAs, CTA c takes
 *         the items c, c + grid, ..., so n_c = count / grid, one more for c < count % grid
 *     [3] N = count
 * A and S cover exactly the trained real parameters: the SGNN's virtual attention columns are chained to the six real
 * attention tensors on every partial row before squaring, and tensors frozen by upb_set_param_groups*, pads and
 * statistics are left out.  The squares are formed and summed in float64 in a fixed order: two identical calls give
 * identical bits.  While the model's KL stop word is set (upb_set_target_kl) the gradient launch writes no partial rows
 * and noise_out is {0, 0, 0, 0}: N = 0 means no sample.  Three launches on `stream` (two with count = 0); no
 * synchronisation.  The partial rows are the model's own scratch, so ids decides which graphs form each CTA's group:
 * pass them in a random order for an unbiased estimate.  UPB_ERR_ARG as upb_ppo_grad_refs, and for a NULL noise_out. */
int upb_ppo_grad_noise(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                       const float* actions, const float* advantages, const float* returns,
                       const float* fixed_log_probs, const float* exps, const upb_step_refs* refs, float inv_batch,
                       float inv_ind, float* grad_out, double* noise_out, void* stream);
int upb_mlp_ppo_grad_noise(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                           const float* actions, const float* advantages, const float* returns,
                           const float* fixed_log_probs, const float* exps, const upb_step_refs* refs,
                           float inv_batch, float inv_ind, float* grad_out, double* noise_out, void* stream);
/* KL penalty on the PPO objective (Schulman et al. 2017, section 4; RLlib's kl_coeff) for both models, on the exact
 * categorical KL over each graph's candidates instead of a sampled estimate.  With beta > 0 every later training step
 * adds beta * kl to the loss, where, per graph g with exps != 0 and its k candidates,
 *     lp_old(c) = the candidate's log-softmax at the pre-pass parameters (upb_forward_cand), lp(c) = the same now,
 *     KL_g = sum_c exp(lp_old(c)) (lp_old(c) - lp(c)),   kl = KL_g summed over ind, times inv_ind,
 * and the logit gradient of candidate c gains beta * inv_ind * (p(c) - p_old(c)) (the whole action distribution, not
 * only the action taken).  A graph with k = 0 adds 0; a candidate whose p_old is 0 in fp32 adds 0.  The sum is taken in
 * log space, so a new probability that underflows gives a large finite term where torch's kl_divergence returns inf.
 * Statistics slot 18 receives sum KL_g and slot 7 counts a non-finite KL_g.  The reference log-probs are passed per call
 * as upb_step_refs.old_cand_log_probs.  upb_read_losses / upb_mlp_read_losses add beta * slot18 / |ind| to the loss
 * while the penalty is on.  The gradient is part of what upb_set_max_grad_norm and the two-group clip measure.  beta may
 * change between steps (an adaptive coefficient); each launch uses the value current when it was issued.  0 turns it
 * off (the default: outputs are those of a context that never set it, whatever old_cand_log_probs is).  UPB_ERR_ARG for
 * a negative or non-finite value. */
int upb_set_kl_penalty(upb_ctx* ctx, float beta);
/* Global gradient-norm clip (torch.nn.utils.clip_grad_norm_(actor_critic.parameters(), max_norm): Stable-Baselines3's
 * and CleanRL's max_grad_norm) on every optimiser step of both models, before Adam and before the weight-decay term:
 *     norm = ||g||_2 over all parameters (the shared encoder once; a skipped head's gradient is 0)
 *     coef = clamp(max_norm / (norm + 1e-6), max=1) in fp32 as torch forms it (a NaN norm gives NaN);  g = g * coef
 * The norm is one float on every CTA, rank and path: float64 sums of g^2 per 128-column slice of the model's gradient
 * row in a fixed tree, the SGNN's 1632 chained attention gradients as one more partial, added in slice order, sqrt in
 * double rounded once to fp32 (optim_kernels.cuh: gclip_*).  upb_ppo_step / upb_mlp_ppo_step stay one launch (every
 * CTA waits for the norm before its Adam; the SGNN's peer exchange is kept), upb_apply / upb_mlp_apply compute it from
 * the all-reduced buffer.  Statistics slot 17 receives the norm.  Exclusive with the reference's two-group clip:
 * UPB_ERR_ARG for max_norm > 0 unless the context's clip_mode is UPB_CLIP_NEVER, and for a negative or non-finite value.
 * 0 turns it off (the default: outputs are those of a context that never set it). */
int upb_set_max_grad_norm(upb_ctx* ctx, float max_norm);
/* Non-finite guard (what GradScaler's "found inf -> skip optimizer.step()" gives a mixed-precision trainer) for both
 * models: a step that is not finite changes nothing and says so; the next step runs normally.  Default 0 (off).  With
 * enable != 0 every later optimiser step (upb_ppo_step and its _vclip / _refs forms, upb_apply, and the rl-mlp
 * counterparts) evaluates, on its minibatch's globally reduced row (summed over CTAs and, on several GPUs, over ranks
 * in rank order), before any parameter is written:
 *     bad  iff  not (slot7 == 0)  or  the global gradient norm is not finite
 * (a NaN in slot 7 is bad too).  The norm is exactly upb_set_max_grad_norm's fp32 norm (optim_kernels.cuh: gclip_*),
 * formed whether or not the global clip is on; it is finite exactly when every real-parameter gradient is finite and
 * their norm fits fp32.  The decision is on the gradient, not on the step's inputs or losses.  Slot 7 sees a non-finite
 * value, log-prob, entropy or exact KL; the norm also sees what slot 7 cannot: a ratio exp(log_prob - fixed_log_prob)
 * that overflows with both log-probs finite, a non-finite advantage or return that reaches a gradient.  An infinite
 * advantage on a graph whose ratio the surrogate clips contributes a zero policy gradient: that step is finite and is
 * applied, with an infinite slot 1.  A policy head skipped for lack of its stage has gradient 0 and cannot make a step
 * bad; pad words and the other statistics are not looked at.
 * A bad step writes its gradient / statistics buffer as usual (the non-finite entries stay visible) plus slot 19 = 1,
 * and no parameter, Adam moment or step counter (the per-segment counters included), so the next step's bias
 * corrections are those of a run that never saw the bad minibatch; it decays no weight and sets no sticky word.  A step
 * that is not bad is bit for bit the step of a context without the guard: parameters, moments, counters and the buffer;
 * upb_apply writes slot 19 = 0 on such a step, so a buffer that is applied again does not keep an earlier mark.  The
 * decision is made on the device; the host never synchronises for it.  Read slot 19 with the statistics.
 *   - Global clip on (upb_set_max_grad_norm): the guard uses the norm the clip formed; a bad step leaves slot 17 at 0.
 *     With the guard off a NaN norm still gives a NaN coefficient, as before.
 *   - Global clip off: upb_ppo_step / upb_mlp_ppo_step stay one launch, in the clipping kernel with coefficient 1; slot
 *     17 stays 0.  The guard works in every clip_mode: a step that takes the two-group clip decides in upb_apply's
 *     kernel before its coefficients are used.  In UPB_CLIP_REFERENCE a bad first step consumes the first-step clip
 *     like any first step (the host does not learn the decision).
 *   - KL stop (upb_set_target_kl): decided first.  A step that passes the criterion stops as without the guard (slot
 *     13, the word) and leaves slot 19 at 0; a NaN in slot 8 never stops, so such a step reaches the guard.
 *   - Peer give-up (upb_peer_timeouts): unchanged; a CTA that gave up applies nothing and marks nothing.
 *   - Several GPUs: with the SGNN's peer exchange every rank holds every rank's contributions and takes the same
 *     decision without another message; NCCL ranks decide in upb_apply on the all-reduced buffer.
 *   - upb_ppo_grad alone never sets slot 19: it applies nothing. */
int upb_set_nonfinite_guard(upb_ctx* ctx, int enable);
/* Per-minibatch advantage normalisation (Stable-Baselines3's normalize_advantage, CleanRL's norm_adv), model-independent.
 * order (device int32[T_used]) is an epoch's sample order; minibatch i is order[i B, (i + 1) B) for i < T_used / B (the
 * tail that floor(T_used / B) drops is not touched).  For each minibatch: mean and unbiased standard deviation (torch's
 * .std()) of adv_in over its graphs with exps != 0, accumulated in float64 in a fixed order and each rounded once to
 * fp32; then adv_out[g] = (adv_in[g] - mean) / (std + 1e-8) in fp32 for every graph g of the minibatch.  A minibatch
 * with fewer than two exps != 0 graphs gets its advantages unchanged.  adv_in, exps, adv_out: device f32 indexed by
 * blob position; adv_out must not alias adv_in.  Deterministic; one launch on `stream`, no synchronisation. */
int upb_normalize_advantages(upb_ctx* ctx, const float* adv_in, const float* exps, const int32_t* order, int T_used,
                             int B, float* adv_out, void* stream);
/* Value-target normalisation (MAPPO's ValueNorm with per_element_update=False) with PopArt's output-preserving rescale
 * of the value head's last layer (van Hasselt et al. 2016), per model.  Each model keeps a running state of three
 * doubles {m1, m2, d} on the device, 0 when the context is created.  Its statistics S(m1, m2, d) = (mean, std) are
 * (0, 1) while d == 0, else mean = m1 / max(d, 1e-5) and std = sqrt(max(m2 / max(d, 1e-5) - mean^2, 1e-2)), each
 * operation a round-to-nearest double one (no fused multiply-add).  The value head then predicts normalised values:
 *   upb_value_norm_denormalize: values[i] = fmaf((float)std, normalized[i], (float)mean) with the model's current
 *     statistics; values[i] = normalized[i] exactly while d == 0.  Works whether or not the option is on.
 *   upb_value_norm_update (one block, once per update, after GAE on the denormalised values):
 *     1. b1 = sum R / T and b2 = sum R^2 / T over all T returns, in float64 in a fixed order (deterministic).
 *     2. If every R is finite: m1 <- beta m1 + (1 - beta) b1, m2 <- beta m2 + (1 - beta) b2, d <- beta d + (1 - beta).
 *        Otherwise the state and the head are left unchanged.
 *     3. (mo, so) = S(old state), (mn, sn) = S(new state).  When the state moved, the value head's last layer in
 *        `params` (the model's val_w2 [1][32] and val_b2 [1]) becomes w2 <- (float)((w2 * so) / sn) and
 *        b2 <- (float)(((so * b2 + mo) - mn) / sn), in double from the fp32 values: the head's denormalised output is
 *        unchanged up to that rounding.  Adam moments and step counters are not touched.
 *     4. norm_returns[i] = (R[i] - (float)mn) / (float)sn in fp32, and norm_values[i] likewise from values[i] when
 *        values is not NULL (norm_values must then be given, and is NULL otherwise).  mean_std (device double[2], may
 *        be NULL) receives (mn, sn).
 *     UPB_ERR_ARG while the option is off, or for T < 1.  The outputs must not alias the inputs.
 *   The training steps are not changed: fed norm_returns (and norm_values as the clipped value loss's old values),
 *   their value loss, clip range and explained variance are in normalised units.
 * upb_set_value_norm: beta, the EMA weight, for both models; 0 (the default) turns the option off.  UPB_ERR_ARG for a
 * non-finite beta or one outside [0, 1).  Several GPUs: every rank holding the same returns and parameters computes the
 * same state, bit for bit, without a message.
 * upb_get_value_norm_state / upb_set_value_norm_state: the model's {m1, m2, d} to / from host double[3] (they
 * synchronise the device); set refuses a non-finite value, m2 < 0 or d outside [0, 1] with UPB_ERR_ARG.  The upb_mlp_*
 * twins act on the rl-mlp model's state and layout. */
int upb_set_value_norm(upb_ctx* ctx, double beta);
int upb_value_norm_denormalize(upb_ctx* ctx, const float* normalized, int T, float* values, void* stream);
int upb_mlp_value_norm_denormalize(upb_ctx* ctx, const float* normalized, int T, float* values, void* stream);
int upb_value_norm_update(upb_ctx* ctx, const float* returns, const float* values, int T, float* params,
                          float* norm_returns, float* norm_values, double* mean_std, void* stream);
int upb_mlp_value_norm_update(upb_ctx* ctx, const float* returns, const float* values, int T, float* params,
                              float* norm_returns, float* norm_values, double* mean_std, void* stream);
int upb_get_value_norm_state(upb_ctx* ctx, double* state3_host);
int upb_mlp_get_value_norm_state(upb_ctx* ctx, double* state3_host);
int upb_set_value_norm_state(upb_ctx* ctx, const double* state3_host);
int upb_mlp_set_value_norm_state(upb_ctx* ctx, const double* state3_host);

/* Advantages recomputed before every PPO epoch (Tianshou's recompute_advantage; Andrychowicz et al. 2021, section 3.5).
 * upb_values: value[g] (device f32, indexed by blob position, like upb_forward's value) of the graphs `ids` (NULL: the
 *   first `count`) from a value-only sweep: the encoder, the GCN pulls, the attention and the value head, without the
 *   policy heads, the softmax or any candidate output.  The values are upb_forward's bit for bit, tier-2 graphs, graphs
 *   above the shared-memory budget and empty masks included; a graph larger than the context's caps gets NaN.  With
 *   value normalisation on they are the head's normalised outputs, as upb_forward's.  One launch on `stream`.
 * upb_gae_targets: from the sweep's raw head outputs head_values f32[T], rewards f32[T] and masks f32[T] (device), one
 *   launch on `stream` writes advantages f32[T] (reward units), returns f32[T] (those the steps train on) and
 *   anchors f32[T] (the clipped value loss's old values).  Value normalisation off (upb_set_value_norm): upb_gae's
 *   arithmetic and order on V = head_values, and anchors = head_values.  On: V = fmaf((float)std, head_values,
 *   (float)mean) as upb_value_norm_denormalize forms it, GAE on V, returns = (R - (float)mean) / (float)std as
 *   upb_value_norm_update forms them, anchors = head_values; (mean, std) are the model's current statistics, which
 *   this call does not move (nor does it rescale the head).  The outputs must not alias the inputs or each other.
 * Both return UPB_ERR_ARG for a NULL context, a NULL pointer or a negative count / T.  The upb_mlp_* twins act on the
 * rl-mlp model (its kernel and its value-normaliser state). */
int upb_values(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params, float* value,
               void* stream);
int upb_mlp_values(upb_ctx* ctx, const void* blob_dev, const int32_t* ids, int count, const float* params,
                   float* value, void* stream);
int upb_gae_targets(upb_ctx* ctx, const float* rewards, const float* masks, const float* head_values, int T,
                    float gamma, float tau, float* advantages, float* returns, float* anchors, void* stream);
int upb_mlp_gae_targets(upb_ctx* ctx, const float* rewards, const float* masks, const float* head_values, int T,
                        float gamma, float tau, float* advantages, float* returns, float* anchors, void* stream);

/* Parameter groups and frozen tensors: torch.optim.Adam over the reference optimizer's param_groups, with
 * requires_grad=False tensors left alone.  Off until the first call; a context that never calls it is unchanged.
 * upb_set_param_groups: one entry per tensor in upb_param_slot order, n_tensors = 32 (the SGNN; the upb_mlp_ twin: 18,
 *   the rl-mlp's table in the same order without the GCN and attention tensors).  lr is kept as a double, as upb_set_lr
 *   keeps it; trained = 0 marks a frozen tensor.  Once set the table replaces the context's lr and weight decay for that
 *   model, and upb_set_lr / upb_set_weight_decay return UPB_ERR_ARG on the context.  For every later optimiser step:
 *     - a frozen tensor gets no Adam step: its parameter, moments and count are unchanged and it is not decayed;
 *     - its columns of the gradient buffer are written as 0 (upb_ppo_grad, upb_ppo_step, the rl-mlp twins), so every
 *       norm (the two-group clip, upb_set_max_grad_norm, the non-finite guard, upb_grad_norms) leaves it out, as torch's
 *       clip_grad_norm_ skips a grad that is None; the attention chain still reads the unmasked virtual sums;
 *     - a trained tensor steps with its own lr and weight decay, and its bias corrections use its own count, which
 *       advances on the steps that apply Adam when its segment is live (the head rule of the per-segment counters).
 *   The per-segment counters of upb_get_opt_state keep their meaning and advance as before.  The first call starts every
 *   tensor's count from its segment's: [1] for the encoder and value tensors, [2] / [3] for the land-use / road head.
 *   A fused step with a table runs k_sgnn_pg / k_mlp_pg, whose tail is the global clip's (coefficient 1 while the clip
 *   is off).  UPB_ERR_ARG for another n_tensors, a null table, a negative or non-finite lr or weight decay, or no trained
 *   tensor.  Synchronises the device.
 * upb_get_tensor_steps / upb_set_tensor_steps: the per-tensor counts to / from host int64[n_tensors] (they synchronise
 *   the device); UPB_ERR_ARG before the first upb_set_param_groups, for another n_tensors or a negative count. */
int upb_set_param_groups(upb_ctx* ctx, const double* lr, const float* weight_decay, const uint8_t* trained,
                         int n_tensors);
int upb_mlp_set_param_groups(upb_ctx* ctx, const double* lr, const float* weight_decay, const uint8_t* trained,
                             int n_tensors);
int upb_get_tensor_steps(upb_ctx* ctx, int64_t* steps, int n_tensors);
int upb_mlp_get_tensor_steps(upb_ctx* ctx, int64_t* steps, int n_tensors);
int upb_set_tensor_steps(upb_ctx* ctx, const int64_t* steps, int n_tensors);
int upb_mlp_set_tensor_steps(upb_ctx* ctx, const int64_t* steps, int n_tensors);

/* Adam settings besides lr and weight decay: torch 2.11's _single_tensor_adam with betas, eps, amsgrad and
 * decoupled_weight_decay (torch.optim.AdamW), per element in this order after the clip:
 *     decoupled and wd != 0: p = p * fp32(1 - lr * wd)     coupled: g = g + wd * p (the clip norms never see either)
 *     m = m.lerp(g, 1 - beta1);  v = v * beta2 + (1 - beta2) * g * g
 *     amsgrad: vmax = max(vmax, v) (a NaN propagates, as torch.maximum), denom = sqrt(vmax) / sqrt(bc2) + eps
 *     otherwise: denom = sqrt(v) / sqrt(bc2) + eps;     p = p - (float)(lr / bc1) * (m / denom)
 *   with bc1 = 1 - beta1^t and bc2 = 1 - beta2^t in double at the tensor's count t.  As in the untabled steps, betas
 *   and eps are fp32 and the moment weights 1.f - beta; lr * wd is formed in double from the double weight decay
 *   (upb_set_weight_decay_double's or upb_set_param_groups_adam's; upb_set_weight_decay's is the fp32 value).  A step
 *   that does not update a tensor's moments (a frozen tensor, an absent head, a KL stop, a non-finite step the guard
 *   skips, a peer give-up) neither decays it nor touches its vmax; upb_value_norm_update leaves vmax alone as it leaves
 *   m and v.
 * upb_set_adam: both models' settings for the optimiser steps issued from now on, live like upb_set_lr.  upb_create
 *   starts from the config's betas and eps, coupled, without AMSGrad.  While the settings are those (or decoupled with
 *   weight decay 0), a model without parameter groups steps exactly as before, through the same kernels; otherwise it
 *   steps through a parameter-group table the context synthesises from its lr, weight decay and these settings
 *   (k_sgnn_pg / k_mlp_pg and k_apply's table), rebuilt by upb_set_lr, upb_set_weight_decay and upb_set_adam, which
 *   then synchronise the device.  UPB_ERR_ARG for a beta outside [0, 1), a negative or non-finite eps, or a context
 *   with upb_set_param_groups tables, whose tensors take the settings upb_create or upb_set_adam held when the table
 *   was set.
 * upb_set_param_groups_adam: upb_set_param_groups with each tensor's weight decay as a double and its own betas, eps,
 *   amsgrad and decoupled flag (the same checks, per tensor).  Synchronises the device.
 * AMSGrad keeps max_exp_avg_sq per model, float[num_params], allocated zero-filled when a tensor first has amsgrad
 *   (a fresh torch optimizer's max(0, v) = v) and kept, unused, while amsgrad is off.  upb_get_amsgrad_state copies it
 *   to the host (UPB_ERR_ARG before it exists); with max_exp_avg_sq NULL it returns 1 while the buffer exists and 0
 *   before, and touches nothing; upb_set_amsgrad_state restores it (allocating it).  n = the model's
 *   num_params.  Both synchronise the device. */
int upb_set_adam(upb_ctx* ctx, float beta1, float beta2, float eps, int amsgrad, int decoupled);
int upb_set_param_groups_adam(upb_ctx* ctx, const double* lr, const double* weight_decay, const uint8_t* trained,
                              const float* beta1, const float* beta2, const float* eps, const uint8_t* amsgrad,
                              const uint8_t* decoupled, int n_tensors);
int upb_mlp_set_param_groups_adam(upb_ctx* ctx, const double* lr, const double* weight_decay, const uint8_t* trained,
                                  const float* beta1, const float* beta2, const float* eps, const uint8_t* amsgrad,
                                  const uint8_t* decoupled, int n_tensors);
int upb_get_amsgrad_state(upb_ctx* ctx, float* max_exp_avg_sq, int n);
int upb_mlp_get_amsgrad_state(upb_ctx* ctx, float* max_exp_avg_sq, int n);
int upb_set_amsgrad_state(upb_ctx* ctx, const float* max_exp_avg_sq, int n);
int upb_mlp_set_amsgrad_state(upb_ctx* ctx, const float* max_exp_avg_sq, int n);

/* Kernel timing for the roofline line of bench.py: while enabled, upb_ppo_grad / upb_ppo_step / upb_forward (and
 * upb_policy_logits, which runs the same forward kernel) bracket the
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
