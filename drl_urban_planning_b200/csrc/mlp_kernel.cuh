// rl-mlp ablation model: fused per-graph forward (+ backward) kernel.
//
// Reference dataflow replaced (all fp32):
//   urban_planning/models/state_encoder.py:217-308   MLPStateEncoder (node Linear, per-edge endpoint selection by raw
//                                                    node type, masked means, numeric MLP; no message passing, no attention)
//   urban_planning/models/policy.py:45-104           masked categorical heads
//   urban_planning/models/value.py:36-39             value head (51 inputs)
//   khrylib/rl/agents/agent_pg.py:19-23 + urban_planning/agents/urban_planning_agent.py:363-371   losses, and their autograd
//
// Algebra used (exact in real arithmetic):
//   * the node encoder is linear, so node_encoder(x_sel) of an edge equals the embedding h_sel of its selected endpoint:
//     edge embeddings are a gather of node embeddings and mean_j he_j = sum_i cnt_i h_i / e with cnt_i the number of edges
//     selecting node i (padded edges carry he = bias but are masked out of the mean and of the logits);
//   * land-use head first layer on [he | hc | he*hc | he-hc] = Weff he + ceff (as in the SGNN kernel);
//   * only mask-true candidates go through the head.
// One CTA of 256 threads walks one graph at a time; the whole parameter vector (41 KB) sits in shared memory.
#pragma once
#include "sgnn_kernel.cuh"

namespace upb {

// ---- flat parameter layout of the rl-mlp model (ActorCritic.parameters() order; params.py: PL.MLP)
constexpr int M_NUM_W0 = 0;        // [64][52]
constexpr int M_NUM_B0 = 3328;
constexpr int M_NUM_W1 = 3392;     // [16][64]
constexpr int M_NUM_B1 = 4416;
constexpr int M_ENC_W = 4432;      // [16][23]
constexpr int M_ENC_B = 4800;
constexpr int M_LU_W0 = 4816;      // [32][64]
constexpr int M_LU_B0 = 6864;
constexpr int M_LU_W1 = 6896;
constexpr int M_RD_W0 = 6928;      // [32][16]
constexpr int M_RD_B0 = 7440;
constexpr int M_RD_W1 = 7472;
constexpr int M_SVD = 51;          // value-head input: 16 + 16 + 16 + 3
constexpr int M_VAL_W0 = 7504;     // [32][51]
constexpr int M_VAL_B0 = 9136;
constexpr int M_VAL_W1 = 9168;     // [32][32]
constexpr int M_VAL_B1 = 10192;
constexpr int M_VAL_W2 = 10224;
constexpr int M_VAL_B2 = 10256;
constexpr int M_NUM_PARAMS = 10257;
constexpr int M_ENCODER_END = M_LU_W0, M_POLICY_END = M_VAL_W0;
constexpr int MG_STATS = 10264;    // per-CTA gradient row: gradients, pad, 8 statistics
constexpr int MG_ROW = 10304;
static_assert(UPB_MLP_NUM_PARAMS == M_NUM_PARAMS, "header constant");

constexpr int MT = 256, MW = MT / 32;
constexpr int M_NS = 464, M_AS = 5632, M_KS = 160;      // graphs beyond these run from a global scratch
static_assert(M_NS == 464 && M_AS == 5632 && M_KS == 160,
              "tests/shape_cases.py puts graphs on both sides of these limits: move its cases with them");

// shared memory map (floats)
constexpr int MS_P = 0;                                   // [10257] parameters (natural layout), padded to 10272
constexpr int MS_WET = MS_P + 10272;                      // [24][16] enc_w^T (row 23 zero)
constexpr int MS_WEFF = MS_WET + 384;                     // [32][17] effective head matrix (row stride 17)
constexpr int MS_CEFF = MS_WEFF + 544;                    // [32]
constexpr int MS_VEC = MS_CEFF + 32;                      // small vectors, see MV_*
constexpr int MV_X52 = 0, MV_XCUR = 56, MV_HC = 80, MV_A0 = 96, MV_SV = 160 /*51 -> 52*/, MV_Y0 = 212, MV_Y1 = 244,
              MV_GSV = 276 /*52*/, MV_D0 = 328, MV_D1 = 360, MV_DN0 = 392, MV_DN1 = 456, MV_GHC = 472, MV_GC = 488,
              MV_GW2 = 520, MV_T16 = 552, MV_T16B = 568, MV_SC = 584 /*24*/, MV_END = 608;
constexpr int MS_RED = MS_VEC + MV_END;                   // [MW][20]
constexpr int MS_G = MS_RED + MW * 20;                    // [32][16] head weight gradient of the graph
constexpr int MS_PART = MS_G + 512;                       // [MW][32*18] per-warp partials: G | gc | gw2
constexpr int MS_Z = MS_PART + MW * 576;                  // [KS]
constexpr int MS_GZ = MS_Z + M_KS;
constexpr int MS_CUV = MS_GZ + M_KS;
constexpr int MS_CIDX = MS_CUV + M_KS;
constexpr int MS_RP = MS_CIDX + M_KS;                     // u16 pairs
constexpr int MS_ADJ = MS_RP + (M_NS + 8) / 2;
constexpr int MS_CNT = MS_ADJ + M_AS;                     // [NS] cnt_i, sign bit = feasible flag (stored as float / int)
constexpr int MS_FEAS = MS_CNT + M_NS;
constexpr int MS_X = MS_FEAS + M_NS;                      // [NS][24]
constexpr int MS_H = MS_X + M_NS * 24;                    // [NS][16]
constexpr int MS_GH = MS_H + M_NS * 16;                   // [NS][16]
constexpr int MS_TOTAL = MS_GH + M_NS * 16;
constexpr size_t M_SMEM_BYTES = (size_t)MS_TOTAL * 4;
static_assert(M_SMEM_BYTES <= 232448, "shared memory budget");

__host__ __device__ inline size_t mlp_scratch_floats(int n_cap, int e_cap) {
  const size_t kcap = (size_t)(e_cap > n_cap ? e_cap : n_cap);
  return (size_t)n_cap * (16 + 16 + 2) + kcap * 2 + 64;
}

// deterministic block sum of a float4 per thread (channels 4q..4q+3, q = tid & 3) -> out16[16]; two barriers inside
__device__ __forceinline__ void m_block_sum_q4(float4 v, float* red, float* out16) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o); v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o); v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < 4) st4(red + warp * 16 + lane * 4, v);
  __syncthreads();
  if (threadIdx.x < 16) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < MW; ++w) s += red[w * 16 + threadIdx.x];
    out16[threadIdx.x] = s;
  }
  __syncthreads();
}

// y[row] = act(b[row] + W[row][:] . x): 8 lanes per row, all MT threads; W, b in shared memory
template <bool TANH>
__device__ __forceinline__ void m_matvec8(const float* W, const float* b, int rows, int cols, const float* x, float* y) {
  const int p = threadIdx.x & 7;
  for (int row = threadIdx.x >> 3; row < rows; row += MT / 8) {
    const float* w = W + row * cols;
    float acc = 0.f;
    for (int k = p; k < cols; k += 8) acc = fmaf(w[k], x[k], acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (p == 0) {
      acc += b[row];
      y[row] = TANH ? tanhf(acc) : acc;
    }
  }
}
// x_grad[c] = sum_r W[r][c] d[r] for c < cols (thread per column), W [rows][cols] in shared memory
__device__ __forceinline__ void m_matvec_t(const float* W, int rows, int cols, const float* d, float* out) {
  for (int c = threadIdx.x; c < cols; c += MT) {
    float s = 0.f;
    for (int r = 0; r < rows; ++r) s = fmaf(W[r * cols + c], d[r], s);
    out[c] = s;
  }
}

template <bool TRAIN>
__device__ void mlp_graph(const StepArgs& a, const BlobHeader& hd, const GraphDesc& d, int gid, float* smem, float* gp,
                          float* scr, uint64_t* mbar, unsigned mpar, bool big) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, q = tid & 3;
  const float* P = smem + MS_P;
  float* sV = smem + MS_VEC;
  float* sc = sV + MV_SC;
  float* sRed = smem + MS_RED;
  const int n = d.n, e = d.e, k = d.k, stage = d.stage;
  const float* gx = reinterpret_cast<const float*>(a.blob + hd.off_x) + (size_t)d.x_row * FS;
  const float* gnum = reinterpret_cast<const float*>(a.blob + hd.off_num) + (size_t)gid * NUMD;
  const float* gcur = reinterpret_cast<const float*>(a.blob + hd.off_cur) + (size_t)gid * FS;
  const uint16_t* rp_g = reinterpret_cast<const uint16_t*>(a.blob + hd.off_rowptr) + d.rp_off;
  const uint32_t* adj_g = reinterpret_cast<const uint32_t*>(a.blob + hd.off_adj) + d.adj_off;
  const uint32_t* cuv_g = reinterpret_cast<const uint32_t*>(a.blob + hd.off_cand_uv) + d.cand_off;
  const int* cidx_g = reinterpret_cast<const int*>(a.blob + hd.off_cand_idx) + d.cand_off;

  GraphView g;        // only the fields softmax_seeds reads
  g.n = n; g.e = e; g.k = k; g.stage = stage; g.gid = gid;
  const float* X; float* H; float* GH; float* cnt; int* feas;
  const uint16_t* rp; const uint32_t* adj;
  if (big) {          // everything per-node from global memory / scratch
    X = gx; H = scr; GH = scr + (size_t)a.n_cap * 16; cnt = scr + (size_t)a.n_cap * 32;
    feas = reinterpret_cast<int*>(scr + (size_t)a.n_cap * 33);
    const size_t kcap = (size_t)(a.e_cap > a.n_cap ? a.e_cap : a.n_cap);
    g.z = scr + (size_t)a.n_cap * 34; g.gz = g.z + kcap;
    rp = rp_g; adj = adj_g; g.cuv = cuv_g; g.cidx = cidx_g;
  } else {
    X = smem + MS_X; H = smem + MS_H; GH = smem + MS_GH; cnt = smem + MS_CNT;
    feas = reinterpret_cast<int*>(smem + MS_FEAS);
    g.z = smem + MS_Z; g.gz = smem + MS_GZ;
    uint16_t* rp_s = reinterpret_cast<uint16_t*>(smem + MS_RP);
    uint32_t* adj_s = reinterpret_cast<uint32_t*>(smem + MS_ADJ);
    uint32_t* cuv_s = reinterpret_cast<uint32_t*>(smem + MS_CUV);
    int* cidx_s = reinterpret_cast<int*>(smem + MS_CIDX);
    if (tid == 0) {   // one bulk copy (TMA) per blob section
      const unsigned b_rp = (unsigned)((n + 1 + 7) / 8) * 16u, b_adj = (unsigned)((2 * e + 3) / 4) * 16u;
      const unsigned b_k = (unsigned)((k + 3) / 4) * 16u, b_x = (unsigned)n * (FS * 4u);
      fence_proxy_async();
      mbar_expect_tx(mbar, b_rp + b_adj + 2u * b_k + b_x);
      bulk_g2s(rp_s, rp_g, b_rp, mbar);
      if (b_adj) bulk_g2s(adj_s, adj_g, b_adj, mbar);
      if (b_k) { bulk_g2s(cuv_s, cuv_g, b_k, mbar); bulk_g2s(cidx_s, cidx_g, b_k, mbar); }
      bulk_g2s(smem + MS_X, gx, b_x, mbar);
    }
    rp = rp_s; adj = adj_s; g.cuv = cuv_s; g.cidx = cidx_s;
  }
  if (tid < NUMD) sV[MV_X52 + tid] = gnum[tid];
  if (tid >= 64 && tid < 64 + FS) sV[MV_XCUR + tid - 64] = gcur[tid - 64];
  if (tid >= 96 && tid < 109) sc[tid - 96] = 0.f;
  if (tid == 109 && a.actions) sc[SC_ACT] = a.actions[(size_t)gid * 2 + stage];
  if constexpr (TRAIN) {
    if (tid == 110) sc[SC_RET] = a.ret[gid];
    if (tid == 111) sc[SC_EXP] = a.exps[gid];
    if (tid == 112) sc[SC_FLP] = a.fixed_lp[gid];
    if (tid == 113) sc[SC_ADV] = a.adv[gid];
  }
  if (!big) mbar_wait(mbar, mpar);
  __syncthreads();

  // ================================================================================ forward
  // numeric encoder layer 0, current node, node embeddings + feasibility flags
  m_matvec8<true>(P + M_NUM_W0, P + M_NUM_B0, NH0, NUMD, sV + MV_X52, sV + MV_A0);
  if (tid < 16) {
    float s = P[M_ENC_B + tid];
    for (int f = 0; f < F; ++f) s = fmaf(smem[MS_WET + f * 16 + tid], sV[MV_XCUR + f], s);
    sV[MV_HC + tid] = s;
  }
  float4 hsum = f4(0.f);
  for (int task = tid; task < n * 4; task += MT) {
    const int i = task >> 2;
    const float* xr = X + (size_t)i * FS;
    float4 acc = ld4(P + M_ENC_B + q * 4);
#pragma unroll
    for (int f4i = 0; f4i < 6; ++f4i) {
      const float4 xv = *reinterpret_cast<const float4*>(xr + f4i * 4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xs = comp(xv, j);
        const float4 w = ld4(smem + MS_WET + (f4i * 4 + j) * 16 + q * 4);
        acc.x = fmaf(w.x, xs, acc.x); acc.y = fmaf(w.y, xs, acc.y); acc.z = fmaf(w.z, xs, acc.z); acc.w = fmaf(w.w, xs, acc.w);
      }
    }
    st4(H + (size_t)i * 16 + q * 4, acc);
    hsum = hsum + acc;
    if (q == 0) {     // torch.argmax(x[:14]) == FEASIBLE (= 1): first maximum wins (state_encoder.py:271)
      bool f = xr[1] > xr[0];
#pragma unroll
      for (int j = 2; j < 14; ++j) f = f && (xr[1] >= xr[j]);
      feas[i] = f ? 1 : 0;
    }
  }
  m_block_sum_q4(hsum, sRed, sV + MV_T16);                 // sum_i h_i  (barriers inside publish H, feas, a0, hc)
  // numeric layer 1; cnt_i = #edges whose selected endpoint is i; sum_i cnt_i h_i
  m_matvec8<true>(P + M_NUM_W1, P + M_NUM_B1, 16, NH0, sV + MV_A0, sV + MV_SV);
  if (stage == 0) {                                        // Weff = Wa + Wd + Wc diag(hc), ceff = b + (Wb - Wd) hc
    for (int idx = tid; idx < 512; idx += MT) {
      const int r = idx >> 4, c = idx & 15;
      const float* w = P + M_LU_W0 + r * 64;
      smem[MS_WEFF + r * 17 + c] = w[c] + w[48 + c] + w[32 + c] * sV[MV_HC + c];
    }
    if (tid < 32) {
      const float* w = P + M_LU_W0 + tid * 64;
      float s = P[M_LU_B0 + tid];
      for (int c = 0; c < 16; ++c) s = fmaf(w[16 + c] - w[48 + c], sV[MV_HC + c], s);
      smem[MS_CEFF + tid] = s;
    }
  } else if (stage == 1) {
    for (int idx = tid; idx < 512; idx += MT) smem[MS_WEFF + (idx >> 4) * 17 + (idx & 15)] = P[M_RD_W0 + idx];
    if (tid < 32) smem[MS_CEFF + tid] = P[M_RD_B0 + tid];
  }
  float4 csum = f4(0.f);
  for (int task = tid; task < n * 4; task += MT) {
    const int i = task >> 2;
    int c = 0;
    for (int t = rp[i]; t < rp[i + 1]; ++t) {
      const uint32_t en = adj[t];
      const int nb = en & 0xffffu;
      const int v = (en & kAdjFirst) ? nb : i, u = (en & kAdjFirst) ? i : nb;      // the edge is (u, v)
      c += ((feas[v] ? v : u) == i) ? 1 : 0;
    }
    if (q == 0) cnt[i] = (float)c;
    csum = csum + ld4(H + (size_t)i * 16 + q * 4) * (float)c;
  }
  m_block_sum_q4(csum, sRed, sV + MV_T16B);                // sum_i cnt_i h_i
  if (tid < 16) {
    sV[MV_SV + 16 + tid] = sV[MV_T16 + tid] / (float)n;    // mean_features over nodes / edges (:288-289)
    sV[MV_SV + 32 + tid] = sV[MV_T16B + tid] / (float)e;
  }
  if (tid >= 32 && tid < 35) sV[MV_SV + 48 + tid - 32] = (tid - 32 == stage) ? 1.f : 0.f;
  __syncthreads();
  // value head (value.py:15-39)
  m_matvec8<true>(P + M_VAL_W0, P + M_VAL_B0, HID, M_SVD, sV + MV_SV, sV + MV_Y0);
  // policy head on the mask-true candidates: one warp per candidate, lane = hidden unit
  const float w2l = stage == 0 ? P[M_LU_W1 + lane] : P[M_RD_W1 + lane];
  float wrow[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) wrow[c] = smem[MS_WEFF + lane * 17 + c];
  const float cb = smem[MS_CEFF + lane];
  auto cand_node = [&](int j) -> int {
    const uint32_t uv = g.cuv[j];
    if (stage != 0) return (int)uv;
    const int u = uv & 0xffffu, v = uv >> 16;
    return feas[v] ? v : u;
  };
  for (int j = warp; j < k; j += MW) {
    const int node = cand_node(j);
    const float xin = H[(size_t)node * 16 + (lane & 15)];
    float pre = cb;
#pragma unroll
    for (int c = 0; c < 16; ++c) pre = fmaf(wrow[c], __shfl_sync(0xffffffffu, xin, c), pre);
    const float zj = warp_sum(w2l * tanhf(pre));
    if (lane == 0) g.z[j] = zj;
  }
  __syncthreads();
  m_matvec8<true>(P + M_VAL_W1, P + M_VAL_B1, HID, HID, sV + MV_Y0, sV + MV_Y1);
  __syncthreads();
  if (warp == 0) {
    const float v = warp_sum(P[M_VAL_W2 + lane] * sV[MV_Y1 + lane]) + P[M_VAL_B2];
    if (lane == 0) sc[SC_VALUE] = v;
    __syncwarp();
    softmax_seeds<TRAIN>(a, hd, g, sc, TRAIN ? gp + MG_STATS : nullptr, lane);
  }
  if constexpr (!TRAIN) { __syncthreads(); return; }
  __syncthreads();

  // ================================================================================ backward
  // ---- value head and numeric encoder
  const float gV = sc[SC_GV];
  if (tid < 32) {
    const float y1 = sV[MV_Y1 + tid];
    sV[MV_D1 + tid] = gV * P[M_VAL_W2 + tid] * (1.f - y1 * y1);
    gacc(gp, M_VAL_W2 + tid, gV * y1);
  }
  if (tid == 32) gacc(gp, M_VAL_B2, gV);
  for (int i = tid; i < n * 16; i += MT) GH[i] = 0.f;      // head contributions are accumulated here
  __syncthreads();
  m_matvec_t(P + M_VAL_W1, HID, HID, sV + MV_D1, sV + MV_D0);
  for (int idx = tid; idx < 1024; idx += MT) gacc(gp, M_VAL_W1 + idx, sV[MV_D1 + (idx >> 5)] * sV[MV_Y0 + (idx & 31)]);
  if (tid < 32) gacc(gp, M_VAL_B1 + tid, sV[MV_D1 + tid]);
  __syncthreads();
  if (tid < 32) { const float y0 = sV[MV_Y0 + tid]; sV[MV_D0 + tid] *= (1.f - y0 * y0); }
  __syncthreads();
  m_matvec_t(P + M_VAL_W0, HID, M_SVD, sV + MV_D0, sV + MV_GSV);
  for (int idx = tid; idx < HID * M_SVD; idx += MT) gacc(gp, M_VAL_W0 + idx, sV[MV_D0 + idx / M_SVD] * sV[MV_SV + idx % M_SVD]);
  if (tid < 32) gacc(gp, M_VAL_B0 + tid, sV[MV_D0 + tid]);
  __syncthreads();
  if (tid < 16) { const float hn = sV[MV_SV + tid]; sV[MV_DN1 + tid] = sV[MV_GSV + tid] * (1.f - hn * hn); }
  __syncthreads();
  m_matvec_t(P + M_NUM_W1, 16, NH0, sV + MV_DN1, sV + MV_DN0);
  for (int idx = tid; idx < 1024; idx += MT) gacc(gp, M_NUM_W1 + idx, sV[MV_DN1 + (idx >> 6)] * sV[MV_A0 + (idx & 63)]);
  if (tid < 16) gacc(gp, M_NUM_B1 + tid, sV[MV_DN1 + tid]);
  __syncthreads();
  if (tid < NH0) { const float a0 = sV[MV_A0 + tid]; sV[MV_DN0 + tid] *= (1.f - a0 * a0); }
  __syncthreads();
  for (int idx = tid; idx < NH0 * NUMD; idx += MT) gacc(gp, M_NUM_W0 + idx, sV[MV_DN0 + idx / NUMD] * sV[MV_X52 + idx % NUMD]);
  if (tid < NH0) gacc(gp, M_NUM_B0 + tid, sV[MV_DN0 + tid]);

  // ---- policy head backward: warp per candidate, lane = hidden unit; lane r keeps G[r][0..15], gc[r], gw2[r]
  {
    float G[16], gcr = 0.f, gw2r = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) G[c] = 0.f;
    float* part = smem + MS_PART + warp * 576;             // scratch of this warp: g_u[32] first, partials at the end
    for (int j = warp; j < k; j += MW) {
      const int node = cand_node(j);
      const float xin = H[(size_t)node * 16 + (lane & 15)];
      float pre = cb;
#pragma unroll
      for (int c = 0; c < 16; ++c) pre = fmaf(wrow[c], __shfl_sync(0xffffffffu, xin, c), pre);
      const float t = tanhf(pre), gzj = g.gz[j];
      const float gu = gzj * w2l * (1.f - t * t);
      gcr += gu;
      gw2r = fmaf(gzj, t, gw2r);
#pragma unroll
      for (int c = 0; c < 16; ++c) G[c] = fmaf(gu, __shfl_sync(0xffffffffu, xin, c), G[c]);
      part[lane] = gu;
      __syncwarp();
      if (lane < 16) {                                     // g_x[c] = sum_r W[r][c] g_u[r], added to the selected node
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < 32; ++r) s = fmaf(smem[MS_WEFF + r * 17 + lane], part[r], s);
        atomicAdd(GH + (size_t)node * 16 + lane, s);
      }
      __syncwarp();
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) part[lane * 18 + c] = G[c];
    part[lane * 18 + 16] = gcr;
    part[lane * 18 + 17] = gw2r;
  }
  __syncthreads();
  for (int idx = tid; idx < 576; idx += MT) {              // fixed-order sum over the warps
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < MW; ++w) s += smem[MS_PART + w * 576 + idx];
    const int r = idx / 18, c = idx % 18;
    if (c < 16) smem[MS_G + r * 16 + c] = s;
    else if (c == 16) sV[MV_GC + r] = s;
    else sV[MV_GW2 + r] = s;
  }
  if (tid < 16) sV[MV_GHC + tid] = 0.f;
  __syncthreads();
  if (stage == 0) {
    for (int idx = tid; idx < 512; idx += MT) {
      const int r = idx >> 4, c = idx & 15;
      const float Gv = smem[MS_G + idx], hc = sV[MV_HC + c], gc = sV[MV_GC + r];
      const int o = M_LU_W0 + r * 64 + c;
      gacc(gp, o, Gv);
      gacc(gp, o + 16, gc * hc);
      gacc(gp, o + 32, Gv * hc);
      gacc(gp, o + 48, Gv - gc * hc);
    }
    if (tid < 32) { gacc(gp, M_LU_B0 + tid, sV[MV_GC + tid]); gacc(gp, M_LU_W1 + tid, sV[MV_GW2 + tid]); }
    if (tid < 16) {                                        // d/d hc through ceff and through Wc diag(hc)
      float s = 0.f;
      for (int r = 0; r < 32; ++r) {
        const float* w = P + M_LU_W0 + r * 64;
        s = fmaf(w[16 + tid] - w[48 + tid], sV[MV_GC + r], s);
        s = fmaf(w[32 + tid], smem[MS_G + r * 16 + tid], s);
      }
      sV[MV_GHC + tid] = s;
    }
  } else {
    for (int idx = tid; idx < 512; idx += MT) gacc(gp, M_RD_W0 + idx, smem[MS_G + idx]);
    if (tid < 32) { gacc(gp, M_RD_B0 + tid, sV[MV_GC + tid]); gacc(gp, M_RD_W1 + tid, sV[MV_GW2 + tid]); }
  }
  __syncthreads();
  // ---- node gradients: g_h_i = g_mean_n / n + cnt_i g_mean_e / e + head contributions; node encoder backward
  {
    const float4 gmn = ld4(sV + MV_GSV + 16 + q * 4) * (1.f / (float)n);
    const float4 gme = e > 0 ? ld4(sV + MV_GSV + 32 + q * 4) * (1.f / (float)e) : f4(0.f);
    float4 hs = f4(0.f);
    for (int task = tid; task < n * 4; task += MT) {
      const int i = task >> 2;
      const float4 v = ld4(GH + (size_t)i * 16 + q * 4) + gmn + gme * cnt[i];
      st4(GH + (size_t)i * 16 + q * 4, v);
      hs = hs + v;
    }
    m_block_sum_q4(hs, sRed, sV + MV_T16);
  }
  for (int idx = tid; idx < 16 * F; idx += MT) {           // g_We[c][f] = sum_i g_h[i][c] x[i][f] + g_hc[c] x_cur[f]
    const int c = idx / F, f = idx % F;
    float s0 = 0.f, s1 = 0.f;
    int i = 0;
    for (; i + 1 < n; i += 2) {
      s0 = fmaf(GH[(size_t)i * 16 + c], X[(size_t)i * FS + f], s0);
      s1 = fmaf(GH[(size_t)(i + 1) * 16 + c], X[(size_t)(i + 1) * FS + f], s1);
    }
    if (i < n) s0 = fmaf(GH[(size_t)i * 16 + c], X[(size_t)i * FS + f], s0);
    gacc(gp, M_ENC_W + idx, (s0 + s1) + sV[MV_GHC + c] * sV[MV_XCUR + f]);
  }
  if (tid < 16) gacc(gp, M_ENC_B + tid, sV[MV_T16 + tid] + sV[MV_GHC + tid]);
  __syncthreads();
}

// ---- fused tail of the rl-mlp step (upb_mlp_ppo_step): the protocol of fused_tail (sgnn_kernel.cuh), minus the
// attention chain.  The 10,304-column row is cut into M_NSLICE slices of 128 columns (the last one holds 64); slice s is
// owned by CTA s % gridDim.x of every rank and goes through the exchange buffer exactly as in fused_tail: push the local
// slice sums into region [parity][rank] of every rank's buffer, release one flag per slice carrying the step sequence
// and this rank's stage bits, poll the own flags, add the ranks' contributions in rank order, Adam.
// The local sum of a column runs in k_mlp_reduce's order -- four accumulators over the rows = 0, 1, 2, 3 (mod 4) of the
// first 4 floor(nparts / 4) rows, the remaining rows added to the first, (s0 + s1) + (s2 + s3) -- so that on one GPU the
// fused step is bit-identical to upb_mlp_ppo_grad + upb_mlp_apply.  Two threads per column: threads [0, 128) keep s0 and
// s1, threads [128, 256) keep s2 and s3, so every warp load is one 128-byte line of one partial row; the two halves meet
// in shared memory.  Adam is k_apply's non-clipping arithmetic (adam_elem).
constexpr int M_NSLICE = (MG_ROW + SLICE - 1) / SLICE;
static_assert(M_NSLICE == 81 && MG_ROW - (M_NSLICE - 1) * SLICE == 64,
              "tests/test_gpu_mlp_step.py runs the rl-mlp fused tail at grids of 80 / 81 / 82 CTAs around M_NSLICE: move them");
static_assert(M_NSLICE * SLICE <= G_ROW && M_NSLICE <= FLAG_STRIDE, "the SGNN exchange buffer holds the rl-mlp row");
static_assert(MT == 2 * SLICE, "two threads per column of a slice");

__device__ void mlp_fused_tail(const StepArgs& a, float* smem, unsigned stage_bits) {
  const int tid = threadIdx.x;
  const int nparts = gridDim.x;
  const int world = a.world, me = a.rank;
  const bool sys = world > 1;
  const unsigned par = a.seq & 1u;
  __shared__ float sh_adam[12];                     // [seg][live ? 1 : 0][step_size, sqrt(bc2)]
  __shared__ long long sh_steps[6];
  __shared__ unsigned sh_bits;                      // OR of the ranks' stage bits (carried by the flags)
  __shared__ int sh_timeout;
  __shared__ float* sh_push[MAX_PEERS];             // region [par][src = me] of every rank's buffer
  float* const mine = a.peers[me];
  const float* const pull = mine + (size_t)par * MAX_PEERS * G_ROW;
  const unsigned* const myflags = reinterpret_cast<const unsigned*>(mine + XCHG_FLAGS) + (size_t)par * MAX_PEERS * FLAG_STRIDE;
  if (tid < world) sh_push[tid] = a.peers[tid] + ((size_t)par * MAX_PEERS + me) * G_ROW;
  if (tid == 32) { sh_timeout = 0; sh_bits = 0u; }
  if (tid == 0 && stage_bits) atomicOr(a.gridbar + 2 + par, stage_bits);
  if (tid == 1 && blockIdx.x == 0) a.gridbar[2 + (par ^ 1u)] = 0u;         // the next launch's word (see fused_tail)
  if (tid < 6) {      // Adam bias corrections of the three segments, for "head live" and "head skipped" (as k_apply)
    const int seg = tid >> 1, live = tid & 1;
    const long long stp = a.steps_in[1 + seg] + live;
    const double bc1 = 1.0 - ipow((double)a.beta1, stp > 0 ? stp : 1);
    const double bc2 = 1.0 - ipow((double)a.beta2, stp > 0 ? stp : 1);
    sh_adam[tid * 2 + 0] = (float)((double)a.lr / bc1);
    sh_adam[tid * 2 + 1] = (float)sqrt(bc2);
    sh_steps[tid] = stp;
  }
  const int c = tid & (SLICE - 1), half = tid >> 7;  // column of the slice; 0: rows 0, 1 (mod 4) + the rest, 1: rows 2, 3
  // the first owned column's moments / parameter do not depend on the reduction
  const int col0 = blockIdx.x * SLICE + c;
  float pm = 0.f, pv = 0.f, pp = 0.f;
  if (half == 0 && col0 < M_NUM_PARAMS) { pm = a.adam_m[col0]; pv = a.adam_v[col0]; pp = a.params_rw[col0]; }
  grid_arrive(a.gridbar);                           // all graphs of all CTAs are done, gpart rows are complete
  grid_wait(a.gridbar, a.bar_target);
  unsigned mybits;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(mybits) : "l"(a.gridbar + 2 + par) : "memory");
  const unsigned flagword = (a.seq << 2) | (mybits & 3u);

  // ---- PUSH: local column sums of the owned slices -> every rank's buffer
  float* sHalf = smem;                              // [SLICE] s2 + s3 of the slice's columns (parameters are no longer read)
  const int nq = nparts & ~3;
  for (int sl = blockIdx.x; sl < M_NSLICE; sl += gridDim.x) {
    const int col = sl * SLICE + c;
    const bool in_row = col < MG_ROW;
    const float* src = a.gpart + col + (size_t)(2 * half) * MG_ROW;
    float sa = 0.f, sb = 0.f;                       // s0, s1 (half 0) or s2, s3 (half 1)
    if (in_row) {
      int r = 0;
      for (; r + 16 <= nq; r += 16) {               // eight loads in flight, each accumulator still in row order
        float t[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          t[2 * j] = __ldcg(src + (size_t)(r + 4 * j) * MG_ROW);
          t[2 * j + 1] = __ldcg(src + (size_t)(r + 4 * j + 1) * MG_ROW);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { sa += t[2 * j]; sb += t[2 * j + 1]; }
      }
      for (; r < nq; r += 4) {
        const float x0 = __ldcg(src + (size_t)r * MG_ROW), x1 = __ldcg(src + (size_t)(r + 1) * MG_ROW);
        sa += x0; sb += x1;
      }
      if (half == 0)
        for (r = nq; r < nparts; ++r) sa += __ldcg(src + (size_t)r * MG_ROW);
    }
    const float pair = sa + sb;
    __syncthreads();                                // the previous slice's halves have been consumed
    if (half) sHalf[c] = pair;
    __syncthreads();
    if (half == 0 && in_row) {
      const float v = pair + sHalf[c];
      for (int r = 0; r < world; ++r) st_relaxed(sh_push[r] + col, v, sys);
    }
  }
  __syncthreads();                                  // this CTA's pushes are issued (ordered before the releases below)
  {
    const int nown = (M_NSLICE - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    for (int idx = tid; idx < world * nown; idx += MT) {
      const int r = idx % world, sl = blockIdx.x + (idx / world) * gridDim.x;
      unsigned* f = reinterpret_cast<unsigned*>(a.peers[r] + XCHG_FLAGS) + ((size_t)par * MAX_PEERS + me) * FLAG_STRIDE + sl;
      if (sys) __threadfence_system(); else __threadfence();
      st_release(f, flagword, sys);
    }
  }

  // ---- REDUCE + ADAM per owned slice; grad_out gets exactly what k_mlp_reduce writes
  for (int sl = blockIdx.x; sl < M_NSLICE; sl += gridDim.x) {
    if (tid < world) {                              // every rank (this one included) has delivered this slice
      unsigned polls = 0, f;
      while ((int)(((f = ld_acquire(myflags + (size_t)tid * FLAG_STRIDE + sl, sys)) >> 2) - a.seq) < 0) {
        if (++polls >= PEER_SPIN_LIMIT) { sh_timeout = 1; break; }
      }
      if (f & 3u) atomicOr(&sh_bits, f & 3u);
    }
    __syncthreads();
    const bool live_lu = sh_bits & 1u, live_rd = sh_bits & 2u;
    const bool dead = sh_timeout != 0;
    const int col = sl * SLICE + c;
    if (half == 0 && col < MG_ROW) {
      float v[MAX_PEERS];
#pragma unroll
      for (int p = 0; p < MAX_PEERS; ++p) v[p] = p < world ? ld_relaxed(pull + (size_t)p * G_ROW + col, sys) : 0.f;
      float s = v[0];
#pragma unroll
      for (int p = 1; p < MAX_PEERS; ++p) if (p < world) s += v[p];        // rank order: identical on every rank
      if (col < M_NUM_PARAMS) {
        a.grad_out[col] = s;
        int seg = 0;
        bool live = true;
        if (col >= M_LU_W0 && col < M_RD_W0) { seg = 1; live = live_lu; }
        else if (col >= M_RD_W0 && col < M_POLICY_END) { seg = 2; live = live_rd; }
        if (live && !dead) {
          if (col != col0) { pm = a.adam_m[col]; pv = a.adam_v[col]; pp = a.params_rw[col]; }    // later slices (small grids)
          adam_elem(a, col, s, pm, pv, pp, sh_adam[(seg * 2 + 1) * 2], sh_adam[(seg * 2 + 1) * 2 + 1]);
        }
      } else if (col < UPB_MLP_STAT_OFFSET) {
        a.grad_out[col] = 0.f;
      }
      if (col >= MG_STATS && col < MG_STATS + 8) a.grad_out[UPB_MLP_STAT_OFFSET + (col - MG_STATS)] = s;
      if (col >= MG_STATS + 8 && col < MG_STATS + UPB_STAT_COUNT) a.grad_out[UPB_MLP_STAT_OFFSET + (col - MG_STATS)] = 0.f;
    }
    __syncthreads();                                // sh_bits / sh_timeout are read before the next slice's polls
  }
  // step counters ([0] global, [1] encoder+value, [2] land-use head, [3] road head): CTA 0, whose flags carried the
  // stage bits of every rank
  if (blockIdx.x == 0 && tid < 4) {
    const bool live_lu = sh_bits & 1u, live_rd = sh_bits & 2u;
    if (sh_timeout == 0)
      a.steps_out[tid] = tid == 0 ? a.steps_in[0] + 1
                                  : sh_steps[(tid - 1) * 2 + (tid == 1 ? 1 : (tid == 2 ? (live_lu ? 1 : 0) : (live_rd ? 1 : 0)))];
    else
      a.steps_out[tid] = a.steps_in[tid];
  }
  if (tid == 0 && sh_timeout) atomicAdd(a.gridbar + 6, 1u);
}

template <bool TRAIN>
__global__ void __launch_bounds__(MT, 1) k_mlp(const __grid_constant__ StepArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ __align__(8) uint64_t s_mbar[1];
  if (threadIdx.x == 0) { mbar_init(s_mbar, 1); fence_mbar_init(); }
  for (int i = threadIdx.x; i < 10272; i += MT) smem[MS_P + i] = i < M_NUM_PARAMS ? a.params[i] : 0.f;
  for (int i = threadIdx.x; i < 384; i += MT) {
    const int f = i >> 4, c = i & 15;
    smem[MS_WET + i] = f < F ? a.params[M_ENC_W + c * F + f] : 0.f;
  }
  float* gp = nullptr;
  if constexpr (TRAIN) {
    gp = a.gpart + (size_t)blockIdx.x * MG_ROW;
    for (int i = threadIdx.x; i < MG_ROW; i += MT) gp[i] = 0.f;
  }
  __syncthreads();
  const BlobHeader& hd = *reinterpret_cast<const BlobHeader*>(a.blob);
  const GraphDesc* descs = reinterpret_cast<const GraphDesc*>(a.blob + hd.off_desc);
  float* scr = a.scratch + (size_t)blockIdx.x * a.scratch_stride;
  unsigned nstaged = 0;
  unsigned stage_bits = 0;     // bit 0 / bit 1: this CTA counted a land-use / road graph (statistics MG_STATS + 5 / + 6)
  for (int item = blockIdx.x; item < a.count; item += gridDim.x) {
    const int gid = a.ids ? a.ids[item] : item;
    const GraphDesc d = descs[gid];
    if (d.n > a.n_cap || d.e > a.e_cap || d.n < 1) {
      if (threadIdx.x == 0) {
        if constexpr (TRAIN) gp[MG_STATS + 7] += 1.f;
        if (a.out_value) a.out_value[gid] = CUDART_NAN_F;
        if (a.out_logp) a.out_logp[gid] = CUDART_NAN_F;
        if (a.out_entropy) a.out_entropy[gid] = CUDART_NAN_F;
      }
      continue;
    }
    stage_bits |= d.stage == 0 ? 1u : (d.stage == 1 ? 2u : 0u);     // softmax_seeds counts the graph's stage
    const bool big = d.n > M_NS || 2 * d.e > M_AS || d.k > M_KS;
    mlp_graph<TRAIN>(a, hd, d, gid, smem, gp, scr, s_mbar, nstaged & 1u, big);
    if (!big) ++nstaged;
    __syncthreads();
  }
  if constexpr (TRAIN) {
    if (a.fuse_tail) mlp_fused_tail(a, smem, stage_bits);
  }
}

// column sums of the per-CTA gradient rows -> flat gradient buffer [gradients | pad | 28 statistics]
// (mlp_fused_tail reproduces this summation order: change both together)
__global__ void __launch_bounds__(256) k_mlp_reduce(const float* __restrict__ gpart, int nparts, float* __restrict__ grad) {
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= MG_ROW) return;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int c = 0;
  for (; c + 4 <= nparts; c += 4) {
    s0 += gpart[(size_t)(c + 0) * MG_ROW + idx]; s1 += gpart[(size_t)(c + 1) * MG_ROW + idx];
    s2 += gpart[(size_t)(c + 2) * MG_ROW + idx]; s3 += gpart[(size_t)(c + 3) * MG_ROW + idx];
  }
  for (; c < nparts; ++c) s0 += gpart[(size_t)c * MG_ROW + idx];
  const float v = (s0 + s1) + (s2 + s3);
  if (idx < M_NUM_PARAMS) grad[idx] = v;
  else if (idx < UPB_MLP_STAT_OFFSET) grad[idx] = 0.f;
  if (idx >= MG_STATS && idx < MG_STATS + 8) grad[UPB_MLP_STAT_OFFSET + (idx - MG_STATS)] = v;
  if (idx >= MG_STATS + 8 && idx < MG_STATS + UPB_STAT_COUNT) grad[UPB_MLP_STAT_OFFSET + (idx - MG_STATS)] = 0.f;
}

}  // namespace upb
