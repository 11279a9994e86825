// Host-side packer: reference 9-array states -> one unpadded blob (see blob.h).  Pure CPU, no CUDA.
// Replaces tensorfy + batch_data of the reference (urban_planning_agent.py:16-20, state_encoder.py:163-177).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <memory>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include <pthread.h>
#include <sched.h>
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

#include "../../include/upb200.h"
#include "blob.h"
#include "errors.h"

namespace upb {

namespace {

struct Counts {
  int n, e, k, stage;
};

inline uint64_t align16(uint64_t v) { return (v + 15) & ~uint64_t(15); }

// The caps bound the candidate counts: a land-use state has k <= e <= e_cap <= 65535 / 2 candidates, and its largest
// adjacency tag, slot + 1 = k, must fit the 15-bit slot field below bit 31 (kAdjFirst).  Road candidates are node ids
// (k <= n <= n_cap <= 65535) and carry no slot.
constexpr int kMaxLandUseCandidates = 65535 / 2;
static_assert(kMaxLandUseCandidates <= (int)kAdjSlotMask, "land-use slot + 1 overflows the adjacency entry's slot field");

struct StateView {
  const float* numerical;
  const float* node_features;
  const int64_t* edge_index;
  const float* current_node;
  const uint8_t* node_mask;
  const uint8_t* edge_mask;
  const uint8_t* land_use_mask;
  const uint8_t* road_mask;
  const float* stage;
};

inline StateView view(const void* const* arrays, int i) {
  const void* const* a = arrays + 9 * (size_t)i;
  return StateView{(const float*)a[0],   (const float*)a[1],   (const int64_t*)a[2],
                   (const float*)a[3],   (const uint8_t*)a[4], (const uint8_t*)a[5],
                   (const uint8_t*)a[6], (const uint8_t*)a[7], (const float*)a[8]};
}

// number of set bytes of a bool mask, and whether they form a prefix.  Branch-free loops (auto-vectorised).
inline int count_prefix(const uint8_t* m, int cap, bool* is_prefix) {
  int c = 0;
  for (int i = 0; i < cap; ++i) c += m[i] != 0;
  int head = 0;
  for (int i = 0; i < c; ++i) head += m[i] != 0;
  *is_prefix = head == c;
  return c;
}

inline int count_set(const uint8_t* m, int lo, int hi) {
  int c = 0;
  for (int i = lo; i < hi; ++i) c += m[i] != 0;
  return c;
}

// Validates one state against the layout contract and returns its sizes.  Returns nullptr or an error text.
// `check_edges`: upb_pack_fill checks the edge endpoints while it builds the CSR (one read of the edge list instead of
// two), upb_pack_measure checks them here.
const char* measure_one(const StateView& s, int n_cap, int e_cap, bool check_edges, Counts* out) {
  for (int j = 0; j < 9; ++j)
    if (((const void* const*)&s)[j] == nullptr) return "null array pointer";
  bool pn, pe;
  const int n = count_prefix(s.node_mask, n_cap, &pn);
  const int e = count_prefix(s.edge_mask, e_cap, &pe);
  if (!pn || !pe) return "node_mask / edge_mask must be prefix masks (observation_extractor.py:60-66)";
  if (n < 1) return "a state needs at least one node";
  int stage;
  if (s.stage[0] != 0.f && s.stage[1] == 0.f) stage = 0;
  else if (s.stage[1] != 0.f && s.stage[0] == 0.f) stage = 1;
  else return "stage must be one-hot on 'land_use' or 'road' (stored states are pre-step states)";
  if (check_edges) {  // every endpoint of a real edge is a real node: unsigned compare catches negatives too; no
                      // early exit so the loop vectorises
    const uint64_t lim = (uint64_t)n;
    const uint64_t* ei = (const uint64_t*)s.edge_index;
    uint64_t bad = 0;
    for (int j = 0; j < 2 * e; ++j) bad |= (uint64_t)(ei[j] >= lim);
    if (bad) return "a real edge joins a padded node";
  }
  int k;
  if (stage == 0) {
    k = count_set(s.land_use_mask, 0, e);
    if (count_set(s.land_use_mask, e, e_cap)) return "land_use_mask marks a padded edge";
  } else {
    k = count_set(s.road_mask, 0, n);
    if (count_set(s.road_mask, n, n_cap)) return "road_mask marks a padded node";
  }
  // no candidate limit of its own: k <= e <= e_cap (land use) or k <= n <= n_cap (road) -- see kMaxLandUseCandidates
  *out = Counts{n, e, k, stage};
  return nullptr;
}

// The blob is written once and next read by the GPU's copy engine, never by this CPU: streaming (non-temporal) stores
// skip the read-for-ownership of every destination line and leave no dirty lines in the cores' caches for the DMA to
// snoop before it can copy the blob.
// dst 16-byte aligned, bytes a multiple of 16 (every per-graph section of the blob is; see make_plan).
#if defined(__SSE2__)
inline void stream_copy(void* dst, const void* src, size_t bytes) {
  __m128i* d = (__m128i*)dst;
  const __m128i* s = (const __m128i*)src;
  for (size_t i = 0; i < bytes / 16; ++i) _mm_stream_si128(d + i, _mm_loadu_si128(s + i));
}
// node features: rows of 23 floats -> rows of 24 floats (zero pad), never reading past a source row
inline void stream_rows(float* dst, const float* src, int n) {
  for (int i = 0; i < n; ++i) {
    const float* r = src + (size_t)i * UPB_NODE_DIM;
    float* d = dst + (size_t)i * kNodeStride;
    _mm_stream_ps(d + 0, _mm_loadu_ps(r + 0));
    _mm_stream_ps(d + 4, _mm_loadu_ps(r + 4));
    _mm_stream_ps(d + 8, _mm_loadu_ps(r + 8));
    _mm_stream_ps(d + 12, _mm_loadu_ps(r + 12));
    _mm_stream_ps(d + 16, _mm_loadu_ps(r + 16));
    const __m128 lo = _mm_castpd_ps(_mm_load_sd((const double*)(r + 20)));      // f20 f21 0 0
    _mm_stream_ps(d + 20, _mm_movelh_ps(lo, _mm_load_ss(r + 22)));              // f20 f21 f22 0
  }
}
inline void stream_fence() { _mm_sfence(); }
#else
inline void stream_copy(void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); }
inline void stream_rows(float* dst, const float* src, int n) {
  for (int i = 0; i < n; ++i) {
    memcpy(dst + (size_t)i * kNodeStride, src + (size_t)i * UPB_NODE_DIM, UPB_NODE_DIM * sizeof(float));
    dst[(size_t)i * kNodeStride + UPB_NODE_DIM] = 0.f;
  }
}
inline void stream_fence() {}
#endif
static_assert(UPB_NODE_DIM == 23 && kNodeStride == 24, "stream_rows is written for 23 -> 24 floats");

struct Plan {
  std::vector<Counts> counts;
  std::vector<GraphDesc> desc;
  BlobHeader hdr;
};

// Persistent worker pool.  The packer runs once per PPO minibatch in the end-to-end path; spawning threads per call
// (tens of microseconds each) cost more than the packing itself.  Design points:
//  * a job is finished when all its ITEMS are done, not when every helper has checked in: a helper that the kernel
//    wakes late simply finds nothing left (its shared_ptr keeps the finished job's counters alive);
//  * helpers poll for the next job for a short while before they sleep on the condition variable, so the second
//    pass of a pack call (fill, right after measure) starts on warm threads without a second wake-up ramp.
// The pool is leaked on purpose (detached threads, no static destructor order problems) and rebuilt lazily in a forked
// child (the reference forks rollout workers, khrylib/rl/agents/agent.py:83-89; worker threads do not survive a fork).
inline void cpu_relax() {
#if defined(__SSE2__)
  _mm_pause();
#endif
}

class Pool {
 public:
  static Pool* get() {
    std::lock_guard<std::mutex> lk(global_mu());
    Pool*& p = instance();
    if (p == nullptr) {
      static std::once_flag once;
      std::call_once(once, [] { pthread_atfork(nullptr, nullptr, [] { instance() = nullptr; new (&global_mu()) std::mutex(); }); });
      p = new Pool();
    }
    return p;
  }

  // fn(ctx, i) for i in [0, count), `chunk` consecutive indices per grab, on up to `threads` threads (caller included)
  void run(int count, int threads, int chunk, void (*fn)(void*, int), void* ctx) {
    std::lock_guard<std::mutex> serial(run_mu_);
    threads = std::min(threads, (count + chunk - 1) / chunk);
    grow(threads - 1);
    auto job = std::make_shared<Job>();
    job->fn = fn; job->ctx = ctx; job->count = count; job->chunk = chunk; job->max_helpers = threads - 1;
    bool wake;
    {
      std::lock_guard<std::mutex> lk(mu_);
      job_ = job;
      epoch_.fetch_add(1, std::memory_order_release);
      wake = sleepers_ > 0;
    }
    if (wake) cv_.notify_all();
    work(*job);
    for (int spins = 0; job->done.load(std::memory_order_acquire) < count; ++spins) {   // chunks still in other hands
      if (spins > 2000) std::this_thread::yield();
      else cpu_relax();
    }
  }

 private:
  struct Job {
    void (*fn)(void*, int) = nullptr;
    void* ctx = nullptr;
    int count = 0, chunk = 1, max_helpers = 0;
    std::atomic<int> next{0}, done{0}, joined{0};
  };

  static Pool*& instance() { static Pool* p = nullptr; return p; }
  static std::mutex& global_mu() { static std::mutex* m = new std::mutex(); return *m; }

  static void work(Job& j) {
    for (;;) {
      const int lo = j.next.fetch_add(j.chunk, std::memory_order_relaxed);
      if (lo >= j.count) break;
      const int hi = std::min(j.count, lo + j.chunk);
      for (int i = lo; i < hi; ++i) j.fn(j.ctx, i);
      j.done.fetch_add(hi - lo, std::memory_order_release);
    }
  }

  void helper() {
    uint64_t seen = 0;
    for (;;) {
      bool got = false;
      const auto until = std::chrono::steady_clock::now() + std::chrono::microseconds(50);
      for (int it = 0;; ++it) {
        if (epoch_.load(std::memory_order_acquire) != seen) { got = true; break; }
        if ((it & 63) == 63 && std::chrono::steady_clock::now() > until) break;
        cpu_relax();
      }
      std::shared_ptr<Job> job;
      {
        std::unique_lock<std::mutex> lk(mu_);
        if (!got) {
          ++sleepers_;
          cv_.wait(lk, [&] { return epoch_.load(std::memory_order_acquire) != seen; });
          --sleepers_;
        }
        seen = epoch_.load(std::memory_order_acquire);
        job = job_;
      }
      if (job && job->joined.fetch_add(1, std::memory_order_relaxed) < job->max_helpers) work(*job);
    }
  }

  // CPUs of the NUMA node the calling thread runs on (empty set if unknown).  The states and the pinned staging
  // buffer were normally first-touched by that thread, so helpers on the same node read and write local memory.
  static bool node_cpus(cpu_set_t* out) {
    const int cpu = sched_getcpu();
    if (cpu < 0) return false;
    for (int node = 0; node < 64; ++node) {
      char path[96];
      snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
      FILE* f = fopen(path, "r");
      if (!f) return false;
      char buf[4096];
      const bool ok = fgets(buf, sizeof(buf), f) != nullptr;
      fclose(f);
      if (!ok) return false;
      CPU_ZERO(out);
      bool mine = false;
      for (char* p = buf; *p;) {
        char* end;
        long a = strtol(p, &end, 10), b = a;
        if (end == p) break;
        if (*end == '-') { p = end + 1; b = strtol(p, &end, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, out); mine |= (c == cpu); }
        p = (*end == ',') ? end + 1 : end;
        if (*end != ',') break;
      }
      if (mine) return true;
    }
    return false;
  }

  void grow(int want) {
    if (started_ >= want) return;
    cpu_set_t node, allowed, both;
    bool pin = false;
    const char* env = getenv("UPB_PACK_NUMA");
    if (!(env && env[0] == '0') && node_cpus(&node) && sched_getaffinity(0, sizeof(allowed), &allowed) == 0) {
      CPU_AND(&both, &node, &allowed);
      pin = CPU_COUNT(&both) >= 2 && CPU_COUNT(&both) < CPU_COUNT(&allowed);     // a real choice, and not a tiny set
    }
    while (started_ < want) {
      ++started_;
      std::thread th([this] { helper(); });
      if (pin) pthread_setaffinity_np(th.native_handle(), sizeof(both), &both);
      th.detach();
    }
  }

  std::mutex run_mu_, mu_;
  std::condition_variable cv_;
  std::shared_ptr<Job> job_;            // guarded by mu_
  std::atomic<uint64_t> epoch_{0};      // bumped under mu_, polled without it
  int sleepers_ = 0;                    // guarded by mu_
  int started_ = 0;                     // guarded by run_mu_
};

template <class F>
void parallel_for(int count, int threads, F&& fn) {
  // copy-bound work: a couple of dozen threads saturate the host memory system
  if (threads <= 0) {   // CPUs this process may run on (affinity mask / container limits), not the machine's count
    cpu_set_t set;
    int avail = (int)std::thread::hardware_concurrency();
    if (sched_getaffinity(0, sizeof(set), &set) == 0) avail = CPU_COUNT(&set);
    threads = std::min(32, std::max(1, avail));
  }
  static const int kChunk = [] { const char* e = getenv("UPB_PACK_CHUNK"); const int v = e ? atoi(e) : 1; return v < 1 ? 1 : v; }();
  threads = std::min(threads, std::max(1, count / (2 * kChunk)));
  if (threads <= 1) {
    for (int i = 0; i < count; ++i) fn(i);
    return;
  }
  using Fn = typename std::remove_reference<F>::type;
  Pool::get()->run(count, threads, kChunk, [](void* c, int i) { (*static_cast<Fn*>(c))(i); }, (void*)&fn);
}

int make_plan(int count, const void* const* arrays, int n_cap, int e_cap, int threads, bool check_edges, Plan* plan) {
  if (count < 0 || (count > 0 && arrays == nullptr)) return set_error(UPB_ERR_ARG, "pack: bad count / arrays");
  if (n_cap < 1 || n_cap > 65535 || e_cap < 0 || 2 * (int64_t)e_cap > 65535)
    return set_error(UPB_ERR_ARG, "pack: caps must satisfy n_cap <= 65535 and 2*e_cap <= 65535");
  plan->counts.assign(count, Counts{0, 0, 0, 0});
  std::atomic<int> bad{-1};
  std::vector<const char*> why(count, nullptr);
  parallel_for(count, threads, [&](int i) {
    why[i] = measure_one(view(arrays, i), n_cap, e_cap, check_edges, &plan->counts[i]);
    if (why[i]) {
      int expected = -1;
      bad.compare_exchange_strong(expected, i);
    }
  });
  if (bad.load() >= 0) {
    int first = -1;
    for (int i = 0; i < count; ++i)
      if (why[i]) { first = i; break; }
    char buf[256];
    snprintf(buf, sizeof(buf), "pack: state %d: %s", first, why[first]);
    return set_error(UPB_ERR_FORMAT, buf);
  }
  plan->desc.assign(count, GraphDesc{});
  uint64_t rows = 0, rp = 0, adj = 0, cand = 0, sum_e = 0, ord = 0;
  for (int i = 0; i < count; ++i) {
    const Counts& c = plan->counts[i];
    GraphDesc& d = plan->desc[i];
    d.n = c.n; d.e = c.e; d.stage = c.stage; d.k = c.k;
    d.x_row = (int32_t)rows;
    d.rp_off = (int32_t)rp;
    d.adj_off = (int32_t)adj;
    d.cand_off = (int32_t)cand;
    d.cost = 4 * c.e + c.n + 64;
    d.ord_off = (int32_t)ord;
    d.ord_rounds = ((c.n + kPullGroup - 1) / kPullGroup + kPullWarps - 1) / kPullWarps + 1;   // upper bound, see fill_one
    ord += (uint64_t)d.ord_rounds * kPullWarps * kPullGroup;
    rows += c.n;
    rp += (uint64_t)((c.n + 1 + 7) & ~7);
    adj += (uint64_t)((2 * c.e + 3) & ~3);
    cand += (uint64_t)((c.k + 3) & ~3);
    sum_e += c.e;
    if (rows > 0x7fffffffull || adj > 0x7fffffffull) return set_error(UPB_ERR_CAPACITY, "pack: blob too large");
  }
  BlobHeader& h = plan->hdr;
  memset(&h, 0, sizeof(h));
  h.magic = kBlobMagic;
  h.count = count;
  h.n_cap = n_cap;
  h.e_cap = e_cap;
  uint64_t off = sizeof(BlobHeader);
  h.off_desc = off;      off = align16(off + sizeof(GraphDesc) * (uint64_t)count);
  h.off_x = off;         off = align16(off + rows * kNodeStride * sizeof(float));
  h.off_num = off;       off = align16(off + (uint64_t)count * kNumDim * sizeof(float));
  h.off_cur = off;       off = align16(off + (uint64_t)count * kNodeStride * sizeof(float));
  h.off_rowptr = off;    off = align16(off + rp * sizeof(uint16_t));
  h.off_order = off;     off = align16(off + ord * sizeof(uint16_t));
  h.off_adj = off;       off = align16(off + adj * sizeof(uint32_t));
  h.off_cand_uv = off;   off = align16(off + cand * sizeof(uint32_t));
  h.off_cand_idx = off;  off = align16(off + cand * sizeof(int32_t));
  h.total_bytes = off;
  h.sum_n = rows;
  h.sum_e = sum_e;
  uint64_t sk = 0;
  for (const Counts& c : plan->counts) sk += c.k;
  h.sum_k = sk;
  return UPB_OK;
}

// One graph's sections are built in per-thread scratch (cache resident) and streamed to the blob.
// Returns nullptr or an error text (edge endpoints are validated here, see measure_one).
const char* fill_one(const StateView& s, const GraphDesc& d, const BlobHeader& h, uint8_t* blob, int index) {
  const int n = d.n, e = d.e;
  stream_rows((float*)(blob + h.off_x) + (size_t)d.x_row * kNodeStride, s.node_features, n);
  {
    alignas(16) float small[kNumDim + kNodeStride];
    memcpy(small, s.numerical, kNumDim * sizeof(float));
    memcpy(small + kNumDim, s.current_node, UPB_NODE_DIM * sizeof(float));
    small[kNumDim + UPB_NODE_DIM] = 0.f;
    stream_copy((float*)(blob + h.off_num) + (size_t)index * kNumDim, small, kNumDim * sizeof(float));
    stream_copy((float*)(blob + h.off_cur) + (size_t)index * kNodeStride, small + kNumDim, kNodeStride * sizeof(float));
  }
  const int rp_len = (n + 1 + 7) & ~7, adj_len = (2 * e + 3) & ~3, cand_len = (d.k + 3) & ~3;
  const int slots = d.ord_rounds * kPullWarps * kPullGroup;
  static thread_local std::vector<uint32_t> scratch;
  const size_t need = 3 * (size_t)(n + 2) + (size_t)rp_len / 2 + adj_len + 2 * (size_t)cand_len + (size_t)slots / 2 + e + 64;
  if (scratch.size() < need) scratch.resize(need);
  // 16-byte aligned carve-up (the vector's storage is at least 16-byte aligned; every length below is a multiple of 4 words)
  uint32_t* base = scratch.data();
  uint32_t* adj = base;                             base += adj_len;
  uint32_t* cuv = base;                             base += cand_len;
  int32_t* cidx = (int32_t*)base;                   base += cand_len;
  uint16_t* rp = (uint16_t*)base;                   base += rp_len / 2;
  uint16_t* ord = (uint16_t*)base;                  base += slots / 2;
  int* pos = (int*)base;                            base += n + 2;      // [n + 1]
  int* idx = (int*)base;                            base += n + 2;      // [n] nodes by descending degree
  int* bucket = (int*)base;                         base += n + 2;      // [n + 2]
  uint32_t* euv = base;                                                 // [e] u | v << 16: the edge list, compact
  // One pass over the int64 edge list: endpoint check (unsigned compare catches negatives), compact copy, degree
  // count -> CSR row pointers over the symmetrised adjacency.  Out-of-range endpoints are clamped so that nothing is
  // written out of bounds before the error is reported.
  memset(pos, 0, sizeof(int) * (n + 1));
  {
    const uint64_t* ei = (const uint64_t*)s.edge_index;
    const uint64_t lim = (uint64_t)n;
    uint64_t bad = 0;
    for (int j = 0; j < e; ++j) {
      uint64_t u = ei[2 * j], v = ei[2 * j + 1];
      bad |= (uint64_t)(u >= lim) | (uint64_t)(v >= lim);
      u = u < lim ? u : lim - 1;
      v = v < lim ? v : lim - 1;
      euv[j] = (uint32_t)u | ((uint32_t)v << 16);
      pos[u + 1]++;
      pos[v + 1]++;
    }
    if (bad) return "a real edge joins a padded node";
  }
  {  // stable counting sort by descending degree (degrees above n land in the top bucket; ties keep node order)
    const int top = n;
    memset(bucket, 0, sizeof(int) * (top + 2));
    for (int i = 0; i < n; ++i) bucket[std::min(pos[i + 1], top)]++;
    int run = 0;
    for (int dgr = top; dgr >= 0; --dgr) { const int c = bucket[dgr]; bucket[dgr] = run; run += c; }
    for (int i = 0; i < n; ++i) idx[bucket[std::min(pos[i + 1], top)]++] = i;
  }
  for (int i = 0; i < n; ++i) pos[i + 1] += pos[i];
  for (int i = 0; i <= n; ++i) rp[i] = (uint16_t)pos[i];
  for (int i = n + 1; i < rp_len; ++i) rp[i] = (uint16_t)pos[n];
  {  // Pull schedule.  Nodes sorted by descending degree are cut into groups of 8 (one warp-task: 4 lanes per node,
     // trip count = the group's largest degree); groups are dealt to the 16 warps longest-first onto the least
     // loaded warp (LPT), so all warps finish a pull phase at about the same time.
    memset(ord, 0xff, sizeof(uint16_t) * slots);          // kNoNode
    const int groups = (n + kPullGroup - 1) / kPullGroup;
    int load[kPullWarps] = {0}, used[kPullWarps] = {0};
    for (int gi = 0; gi < groups; ++gi) {
      const int first = idx[gi * kPullGroup];
      const int cost = (pos[first + 1] - pos[first] + 1) / 2 + 2;     // trips of two neighbours + fixed overhead
      int best = -1;
      for (int w = 0; w < kPullWarps; ++w)
        if (used[w] < d.ord_rounds && (best < 0 || load[w] < load[best])) best = w;
      load[best] += cost;
      const int r = used[best]++;
      for (int j = 0; j < kPullGroup && gi * kPullGroup + j < n; ++j)
        ord[(r * kPullWarps + best) * kPullGroup + j] = (uint16_t)idx[gi * kPullGroup + j];
    }
  }
  int slot = 0;
  for (int j = 0; j < e; ++j) {
    const uint32_t u = euv[j] & 0xffffu, v = euv[j] >> 16;
    uint32_t tag = 0;
    if (d.stage == 0 && s.land_use_mask[j]) {
      cuv[slot] = u | (v << 16);
      cidx[slot] = j;
      tag = (uint32_t)(slot + 1) << 16;
      ++slot;
    }
    adj[pos[u]++] = v | tag | kAdjFirst;      // row owner u is the edge's FIRST endpoint (edge_index[j][0])
    adj[pos[v]++] = u | tag;
  }
  for (int a = 2 * e; a < adj_len; ++a) adj[a] = 0;
  if (d.stage == 1) {
    for (int i = 0; i < n; ++i)
      if (s.road_mask[i]) {
        cuv[slot] = (uint32_t)i;
        cidx[slot] = i;
        ++slot;
      }
  }
  for (int c = slot; c < cand_len; ++c) { cuv[c] = 0; cidx[c] = 0; }
  stream_copy((uint16_t*)(blob + h.off_rowptr) + d.rp_off, rp, sizeof(uint16_t) * rp_len);
  stream_copy((uint16_t*)(blob + h.off_order) + d.ord_off, ord, sizeof(uint16_t) * slots);
  stream_copy((uint32_t*)(blob + h.off_adj) + d.adj_off, adj, sizeof(uint32_t) * adj_len);
  stream_copy((uint32_t*)(blob + h.off_cand_uv) + d.cand_off, cuv, sizeof(uint32_t) * cand_len);
  stream_copy((int32_t*)(blob + h.off_cand_idx) + d.cand_off, cidx, sizeof(int32_t) * cand_len);
  stream_fence();       // streaming stores are weakly ordered: make them visible before the job is reported done
  return nullptr;
}

}  // namespace

}  // namespace upb

using namespace upb;

extern "C" int upb_pack_measure(int count, const void* const* state_arrays, int n_cap, int e_cap, int threads,
                                uint64_t* blob_bytes) {
  if (!blob_bytes) return set_error(UPB_ERR_ARG, "pack_measure: blob_bytes is null");
  Plan plan;
  int rc = make_plan(count, state_arrays, n_cap, e_cap, threads, true, &plan);
  if (rc != UPB_OK) return rc;
  *blob_bytes = plan.hdr.total_bytes;
  return UPB_OK;
}

extern "C" int upb_pack_fill(int count, const void* const* state_arrays, int n_cap, int e_cap, int threads,
                             void* blob_host, uint64_t blob_bytes) {
  if (!blob_host || ((uintptr_t)blob_host & 15)) return set_error(UPB_ERR_ARG, "pack_fill: blob must be 16-byte aligned");
  Plan plan;
  int rc = make_plan(count, state_arrays, n_cap, e_cap, threads, false, &plan);
  if (rc != UPB_OK) return rc;
  if (blob_bytes < plan.hdr.total_bytes) return set_error(UPB_ERR_CAPACITY, "pack_fill: blob buffer too small");
  uint8_t* blob = (uint8_t*)blob_host;
  memcpy(blob, &plan.hdr, sizeof(BlobHeader));
  if (count > 0) memcpy(blob + plan.hdr.off_desc, plan.desc.data(), sizeof(GraphDesc) * (size_t)count);
  std::atomic<int> bad{count};
  std::atomic<const char*> why{nullptr};
  parallel_for(count, threads, [&](int i) {
    const char* err = fill_one(view(state_arrays, i), plan.desc[i], plan.hdr, blob, i);
    if (err) {
      int cur = bad.load();
      while (i < cur && !bad.compare_exchange_weak(cur, i)) {}
      why.store(err);
    }
  });
  if (bad.load() < count) {
    char buf[256];
    snprintf(buf, sizeof(buf), "pack: state %d: %s", bad.load(), why.load());
    return set_error(UPB_ERR_FORMAT, buf);
  }
  return UPB_OK;
}

// ---- chunked packing: plan once, fill state ranges one after the other, so the caller can upload the byte ranges of a
// finished chunk (host -> device copies run asynchronously) while the next chunk is being packed
struct upb_pack_plan {
  Plan plan;
  int count = 0;
};

extern "C" int upb_pack_plan_create(int count, const void* const* state_arrays, int n_cap, int e_cap, int threads,
                                    upb_pack_plan** plan_out, uint64_t* blob_bytes) {
  if (!plan_out || !blob_bytes) return set_error(UPB_ERR_ARG, "pack_plan_create: null output");
  upb_pack_plan* p = new (std::nothrow) upb_pack_plan();
  if (!p) return set_error(UPB_ERR_ARG, "pack_plan_create: out of memory");
  int rc = make_plan(count, state_arrays, n_cap, e_cap, threads, false, &p->plan);
  if (rc != UPB_OK) { delete p; return rc; }
  p->count = count;
  *plan_out = p;
  *blob_bytes = p->plan.hdr.total_bytes;
  return UPB_OK;
}

extern "C" void upb_pack_plan_destroy(upb_pack_plan* p) { delete p; }

extern "C" int upb_pack_plan_fill(upb_pack_plan* p, const void* const* state_arrays, int first, int count, int threads,
                                  void* blob_host, uint64_t blob_bytes, uint64_t* ranges) {
  if (!p || !blob_host || ((uintptr_t)blob_host & 15) || !ranges)
    return set_error(UPB_ERR_ARG, "pack_plan_fill: bad argument (blob must be 16-byte aligned)");
  const Plan& plan = p->plan;
  if (first < 0 || count < 0 || first + count > p->count) return set_error(UPB_ERR_ARG, "pack_plan_fill: range outside the plan");
  if (blob_bytes < plan.hdr.total_bytes) return set_error(UPB_ERR_CAPACITY, "pack_plan_fill: blob buffer too small");
  uint8_t* blob = (uint8_t*)blob_host;
  const BlobHeader& h = plan.hdr;
  int nr = 0;
  auto add = [&](uint64_t off, uint64_t len) { ranges[2 * nr] = off; ranges[2 * nr + 1] = len; ++nr; };
  if (first == 0) {      // header + descriptor table travel with the first chunk
    memcpy(blob, &h, sizeof(BlobHeader));
    if (p->count > 0) memcpy(blob + h.off_desc, plan.desc.data(), sizeof(GraphDesc) * (size_t)p->count);
    add(0, h.off_x);
  } else {
    add(0, 0);
  }
  std::atomic<int> bad{p->count};
  std::atomic<const char*> why{nullptr};
  parallel_for(count, threads, [&](int j) {
    const int i = first + j;
    const char* err = fill_one(view(state_arrays, i), plan.desc[i], h, blob, i);
    if (err) {
      int cur = bad.load();
      while (i < cur && !bad.compare_exchange_weak(cur, i)) {}
      why.store(err);
    }
  });
  if (bad.load() < p->count) {
    char buf[256];
    snprintf(buf, sizeof(buf), "pack: state %d: %s", bad.load(), why.load());
    return set_error(UPB_ERR_FORMAT, buf);
  }
  // byte ranges of the eight per-graph sections written by this chunk (section start of state `first` .. of state `last`)
  const int last = first + count;
  const bool end = last >= p->count;
  const GraphDesc* d = plan.desc.data();
  auto span = [&](uint64_t base, uint64_t next_base, uint64_t unit, int64_t a, int64_t b_or_neg) {
    const uint64_t lo = base + unit * (uint64_t)a;
    const uint64_t hi = b_or_neg < 0 ? next_base : base + unit * (uint64_t)b_or_neg;
    add(lo, hi > lo ? hi - lo : 0);
  };
  if (count == 0) { for (int k = 0; k < 8; ++k) add(0, 0); return UPB_OK; }
  span(h.off_x, h.off_num, kNodeStride * sizeof(float), d[first].x_row, end ? -1 : d[last].x_row);
  span(h.off_num, h.off_cur, kNumDim * sizeof(float), first, end ? -1 : last);
  span(h.off_cur, h.off_rowptr, kNodeStride * sizeof(float), first, end ? -1 : last);
  span(h.off_rowptr, h.off_order, sizeof(uint16_t), d[first].rp_off, end ? -1 : d[last].rp_off);
  span(h.off_order, h.off_adj, sizeof(uint16_t), d[first].ord_off, end ? -1 : d[last].ord_off);
  span(h.off_adj, h.off_cand_uv, sizeof(uint32_t), d[first].adj_off, end ? -1 : d[last].adj_off);
  span(h.off_cand_uv, h.off_cand_idx, sizeof(uint32_t), d[first].cand_off, end ? -1 : d[last].cand_off);
  span(h.off_cand_idx, h.total_bytes, sizeof(int32_t), d[first].cand_off, end ? -1 : d[last].cand_off);
  return UPB_OK;
}

extern "C" int upb_blob_info(const void* blob_host, uint64_t blob_bytes, int* count, int32_t* per_graph4) {
  if (!blob_host || blob_bytes < sizeof(BlobHeader)) return set_error(UPB_ERR_ARG, "blob_info: bad blob");
  const BlobHeader* h = (const BlobHeader*)blob_host;
  if (h->magic != kBlobMagic || h->total_bytes > blob_bytes) return set_error(UPB_ERR_FORMAT, "blob_info: not a blob");
  if (count) *count = h->count;
  if (per_graph4) {
    const GraphDesc* d = (const GraphDesc*)((const uint8_t*)blob_host + h->off_desc);
    for (int i = 0; i < h->count; ++i) {
      per_graph4[4 * i + 0] = d[i].n;
      per_graph4[4 * i + 1] = d[i].e;
      per_graph4[4 * i + 2] = d[i].k;
      per_graph4[4 * i + 3] = d[i].stage;
    }
  }
  return UPB_OK;
}
