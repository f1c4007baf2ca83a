// Experience replay for the learner batch on sm_90a (H100): the contract is tb_replay_mix in include/torchbeast_b200.h.
//
// One launch copies every row of every leaf: a row is one (outer index, column) pair of row_bytes bytes, and each warp
// takes one row at a time, grid-stride over all rows of all leaves.  A fresh row is read once and written twice (mixed
// batch, ring slot); a replayed row is read from its ring slot and written once.  Every block draws the R slots itself
// into shared memory (R Philox calls, spread over its threads), so no block waits on another and there are no atomics;
// tb_replay_mix_slots runs the same kernel on slots a prioritised draw wrote (slots_in).
// The copy is bandwidth-bound: rows move as 16-byte vectors where row_bytes and the leaf's pointers allow, otherwise as
// 8-, 4- or 1-byte words (reward rows are 4 bytes, policy_logits rows at A = 7 are 28).
#include "common.cuh"

namespace tb {

namespace {

constexpr int kReplayThreads = 256;

struct ReplayTable {
  tb_replay_leaf leaf[TB_REPLAY_MAX_LEAVES];
  int64_t rows_end[TB_REPLAY_MAX_LEAVES];  // cumulative row count: leaf l owns rows [rows_end[l-1], rows_end[l])
  int vec[TB_REPLAY_MAX_LEAVES];           // copy width in bytes: 16, 8, 4 or 1
  int num_leaves;
};

template <typename V>
__device__ __forceinline__ void copy_row(const char* __restrict__ src, char* __restrict__ d1, char* __restrict__ d2,
                                         int64_t bytes, int lane) {
  const V* s = reinterpret_cast<const V*>(src);
  V* o1 = reinterpret_cast<V*>(d1);
  V* o2 = reinterpret_cast<V*>(d2);
  const int64_t n = bytes / int64_t(sizeof(V));
  int64_t i = lane;
  // four loads in flight per lane before the stores
  for (; i + 3 * kWarp < n; i += 4 * kWarp) {
    const V a = s[i], b = s[i + kWarp], c = s[i + 2 * kWarp], d = s[i + 3 * kWarp];
    if (o1) { o1[i] = a; o1[i + kWarp] = b; o1[i + 2 * kWarp] = c; o1[i + 3 * kWarp] = d; }
    if (o2) { o2[i] = a; o2[i + kWarp] = b; o2[i + 2 * kWarp] = c; o2[i + 3 * kWarp] = d; }
  }
  for (; i < n; i += kWarp) {
    const V a = s[i];
    if (o1) o1[i] = a;
    if (o2) o2[i] = a;
  }
}

// slots_in != NULL: the R slots are read from there (tb_replay_mix_slots) instead of drawn; seed_step is not read.
__global__ void __launch_bounds__(kReplayThreads) replay_mix_kernel(const ReplayTable tab, int64_t Bf, int64_t R,
                                                                    int64_t capacity,
                                                                    const uint64_t* __restrict__ seed_step,
                                                                    const int64_t* __restrict__ head_size,
                                                                    uint32_t stream_id,
                                                                    int64_t* __restrict__ slots_out,
                                                                    const int64_t* __restrict__ slots_in) {
  extern __shared__ int64_t slots[];  // [R]
  const int64_t head = head_size[0];
  if (slots_in) {
    for (int64_t j = threadIdx.x; j < R; j += blockDim.x) slots[j] = slots_in[j];
  } else {
    const uint64_t seed = seed_step[0], step = seed_step[1];
    const int64_t size = head_size[1];
    const int64_t n = size < capacity - Bf ? size : capacity - Bf;
    for (int64_t j = threadIdx.x; j < R; j += blockDim.x) {
      const uint32_t x = philox4x32_10_w0(uint32_t(step), uint32_t(step >> 32), uint32_t(j), stream_id, uint32_t(seed),
                                          uint32_t(seed >> 32));
      const int64_t k = int64_t((uint64_t(x) * uint64_t(n)) >> 32);
      const int64_t slot = (head - 1 - k + capacity) % capacity;  // k < n <= capacity - Bf, so the sum is >= 0
      slots[j] = slot;
      if (blockIdx.x == 0 && slots_out) slots_out[j] = slot;
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & (kWarp - 1);
  const int64_t warps = int64_t(gridDim.x) * (blockDim.x / kWarp);
  const int64_t total = tab.rows_end[tab.num_leaves - 1];
  int l = 0;
  for (int64_t r = int64_t(blockIdx.x) * (blockDim.x / kWarp) + threadIdx.x / kWarp; r < total; r += warps) {
    while (r >= tab.rows_end[l]) ++l;  // rows grow with r, so the leaf index only moves forward
    const tb_replay_leaf& lf = tab.leaf[l];
    const int64_t W = lf.out ? Bf + R : Bf;
    const int64_t i = r - (l ? tab.rows_end[l - 1] : 0);
    const int64_t o = i / W, c = i - o * W;
    const int64_t rb = lf.row_bytes;
    char* out = lf.out ? static_cast<char*>(lf.out) + (o * (Bf + R) + c) * rb : nullptr;
    char* ring = static_cast<char*>(lf.ring);
    const char* src;
    char* ring_dst = nullptr;
    if (c < Bf) {
      src = static_cast<const char*>(lf.fresh) + (o * Bf + c) * rb;
      ring_dst = ring + (((head + c) % capacity) * lf.outer + o) * rb;
    } else {
      src = ring + (slots[c - Bf] * lf.outer + o) * rb;
    }
    switch (tab.vec[l]) {
      case 16: copy_row<uint4>(src, out, ring_dst, rb, lane); break;
      case 8: copy_row<uint2>(src, out, ring_dst, rb, lane); break;
      case 4: copy_row<uint32_t>(src, out, ring_dst, rb, lane); break;
      default: copy_row<uint8_t>(src, out, ring_dst, rb, lane); break;
    }
  }
}

// ---- prioritised replay (include/torchbeast_b200.h states the rule) ---------------------------------------------------
// One CTA of kPrioChunks threads; thread i owns chunk i of the survivors.  Phase 1: each thread sums its chunk's q in k
// order (and its minimum); the chunk totals are combined in order, within a warp by shuffling them in lane order and
// across warps by every thread adding the preceding warps' totals in order, into C at each chunk's end (sEnd).
// Phase 2: each draw binary-searches sEnd for its chunk, then walks that chunk again, recomputing q, to the first
// C_k > u*S.  C is non-decreasing (every step adds a q >= 0), so the search finds the smallest such k.  No atomics: the
// results are bit-identical from run to run.  q is recomputed rather than stored so the kernel needs no scratch buffer
// at any capacity; a draw reads at most ceil(n / kPrioChunks) priorities twice.
constexpr int kPrioChunks = 1024;

__device__ __forceinline__ double prio_q(const float* __restrict__ priorities, int64_t slot, double eps, double alpha) {
  return pow(__dadd_rn(double(priorities[slot]), eps), alpha);
}

__global__ void __launch_bounds__(kPrioChunks) replay_sample_prio_kernel(const float* __restrict__ priorities,
                                                                         const double* __restrict__ prio,
                                                                         const int64_t* __restrict__ head_size,
                                                                         const uint64_t* __restrict__ seed_step,
                                                                         int64_t Bf, int64_t R, int64_t capacity,
                                                                         uint32_t stream_id,
                                                                         int64_t* __restrict__ batch_slots,
                                                                         float* __restrict__ column_weights) {
  __shared__ double sEnd[kPrioChunks];           // C at the end of chunk i (for an empty chunk: of the one before it)
  __shared__ double sPre[kPrioChunks];           // P_i: the totals of the earlier chunks of its warp
  __shared__ double sTot[kPrioChunks / kWarp];   // G_g: the total of warp g's chunks
  __shared__ double sBase[kPrioChunks / kWarp];  // B_g: the totals of the warps before g
  __shared__ double sMin[kPrioChunks / kWarp];
  const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid / kWarp;
  const int64_t head = head_size[0], size = head_size[1];
  for (int64_t c = tid; c < Bf; c += kPrioChunks) {
    batch_slots[c] = (head + c) % capacity;
    column_weights[c] = 1.0f;
  }
  if (R == 0) return;
  const double alpha = prio[0], beta = prio[1], eps = prio[3];
  const int64_t n = size < capacity - Bf ? size : capacity - Bf;
  const int64_t L = (n + kPrioChunks - 1) / kPrioChunks;
  const int64_t k0 = int64_t(tid) * L < n ? int64_t(tid) * L : n, k1 = k0 + L < n ? k0 + L : n;
  double r = 0.0, qmin = INFINITY;
  for (int64_t k = k0; k < k1; ++k) {
    const double q = prio_q(priorities, (head - 1 - k + capacity) % capacity, eps, alpha);
    r = __dadd_rn(r, q);
    qmin = fmin(qmin, q);
  }
  double P = 0.0, G = 0.0;
  for (int l = 0; l < kWarp; ++l) {
    const double x = __shfl_sync(0xffffffffu, r, l);
    if (l < lane) P = __dadd_rn(P, x);
    G = __dadd_rn(G, x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) qmin = fmin(qmin, __shfl_xor_sync(0xffffffffu, qmin, o));
  if (lane == 0) { sTot[warp] = G; sMin[warp] = qmin; }
  __syncthreads();
  double base = 0.0;
  for (int g = 0; g < warp; ++g) base = __dadd_rn(base, sTot[g]);
  sEnd[tid] = __dadd_rn(base, __dadd_rn(P, r));
  sPre[tid] = P;
  if (lane == 0) sBase[warp] = base;
  qmin = sMin[0];
  for (int g = 1; g < kPrioChunks / kWarp; ++g) qmin = fmin(qmin, sMin[g]);
  __syncthreads();
  const double S = sEnd[kPrioChunks - 1];
  const uint64_t seed = seed_step[0], step = seed_step[1];
  for (int64_t j = tid; j < R; j += kPrioChunks) {
    const uint2 x = philox4x32_10_w01(uint32_t(step), uint32_t(step >> 32), uint32_t(j), stream_id, uint32_t(seed),
                                      uint32_t(seed >> 32));
    const double u = double(((uint64_t(x.y) << 32) | uint64_t(x.x)) >> 11) * 0x1p-53;
    const double target = __dmul_rn(u, S);
    int lo = 0, hi = kPrioChunks;  // the first chunk whose end exceeds target
    while (lo < hi) {
      const int mid = (lo + hi) / 2;
      if (sEnd[mid] > target) hi = mid; else lo = mid + 1;
    }
    int64_t k;
    double q;
    if (lo == kPrioChunks) {  // rounding left no C_k > u*S
      k = n - 1;
      q = prio_q(priorities, (head - 1 - k + capacity) % capacity, eps, alpha);
    } else {
      const int64_t c0 = int64_t(lo) * L, c1 = c0 + L < n ? c0 + L : n;
      const double b = sBase[lo / kWarp], p0 = sPre[lo];
      double rr = 0.0;
      for (k = c0;; ++k) {
        q = prio_q(priorities, (head - 1 - k + capacity) % capacity, eps, alpha);
        rr = __dadd_rn(rr, q);
        if (k + 1 >= c1 || __dadd_rn(b, __dadd_rn(p0, rr)) > target) break;
      }
    }
    batch_slots[Bf + j] = (head - 1 - k + capacity) % capacity;
    column_weights[Bf + j] = float(pow(qmin / q, beta));
  }
}

// One thread per batch column c: p_c from the column's |vs - V| in t order; it is stored unless a later column names
// the same slot (largest column wins).  Reads are coalesced across columns.
constexpr int kPrioUpdateThreads = 128;
__global__ void __launch_bounds__(kPrioUpdateThreads) replay_update_prio_kernel(const float* __restrict__ vs,
                                                                                const float* __restrict__ values,
                                                                                int64_t T, int64_t B,
                                                                                const int64_t* __restrict__ batch_slots,
                                                                                const double* __restrict__ prio,
                                                                                float* __restrict__ priorities) {
  const int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= B) return;
  const int64_t slot = batch_slots[c];
  for (int64_t c2 = c + 1; c2 < B; ++c2)
    if (batch_slots[c2] == slot) return;
  const double eta = prio[2];
  double mx = 0.0, sum = 0.0;
  constexpr int kBatch = 16;  // loads in flight per thread before the in-order sums
  for (int64_t t0 = 0; t0 < T; t0 += kBatch) {
    float a[kBatch], v[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int64_t t = t0 + u < T ? t0 + u : T - 1;
      a[u] = vs[t * B + c];
      v[u] = values[t * B + c];
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (t0 + u >= T) break;
      const double e = fabs(__dsub_rn(double(a[u]), double(v[u])));
      mx = e > mx || e != e ? e : mx;  // NaN propagates
      sum = __dadd_rn(sum, e);
    }
  }
  const double p = __dadd_rn(__dmul_rn(eta, mx), __dmul_rn(__dsub_rn(1.0, eta), __ddiv_rn(sum, double(T))));
  const float pf = float(p);
  priorities[slot] = isfinite(pf) ? pf : 0.0f;
}

__global__ void replay_advance_kernel(int64_t* head_size, uint64_t* seed_step, int64_t Bf, int64_t capacity) {
  head_size[0] = (head_size[0] + Bf) % capacity;
  head_size[1] = head_size[1] + Bf < capacity ? head_size[1] + Bf : capacity;
  seed_step[1] += 1;
}

int copy_width(const tb_replay_leaf& lf) {
  const uintptr_t bits = uintptr_t(lf.fresh) | uintptr_t(lf.out) | uintptr_t(lf.ring) | uintptr_t(lf.row_bytes);
  for (int v = 16; v >= 4; v >>= 1)
    if (bits % v == 0) return v;
  return 1;
}

}  // namespace

}  // namespace tb

using namespace tb;

// Both mix entries: slots_in == NULL draws the slots (tb_replay_mix), else reads them (tb_replay_mix_slots).
static int launch_mix(const char* what, const tb_replay_leaf* leaves_host, int num_leaves, int64_t Bf, int64_t R,
                      int64_t capacity, const uint64_t* seed_step, const int64_t* head_size, int64_t stream_id,
                      int64_t* slots_out, const int64_t* slots_in, void* stream) {
  TB_REQUIRE(num_leaves >= 1 && num_leaves <= TB_REPLAY_MAX_LEAVES, "%s: num_leaves must be in [1, %d], got %d", what,
             TB_REPLAY_MAX_LEAVES, num_leaves);
  TB_REQUIRE(R >= 0 && R <= TB_REPLAY_MAX_R, "%s: R must be in [0, %d], got %lld", what, TB_REPLAY_MAX_R, (long long)R);
  TB_REQUIRE(Bf >= 1, "%s: Bf must be at least 1, got %lld", what, (long long)Bf);
  TB_REQUIRE(capacity > Bf, "%s: capacity (%lld) must exceed Bf (%lld)", what, (long long)capacity, (long long)Bf);
  TB_REQUIRE(stream_id >= 0 && stream_id <= int64_t(UINT32_MAX), "%s: stream_id must be in [0, 2^32), got %lld", what,
             (long long)stream_id);
  ReplayTable tab = {};
  tab.num_leaves = num_leaves;
  int64_t rows = 0;
  for (int l = 0; l < num_leaves; ++l) {
    const tb_replay_leaf& lf = leaves_host[l];
    TB_REQUIRE(lf.fresh && lf.ring, "%s: null pointer in leaf %d", what, l);
    TB_REQUIRE(lf.outer >= 1 && lf.row_bytes >= 1, "%s: leaf %d needs outer >= 1 and row_bytes >= 1, got %lld, %lld",
               what, l, (long long)lf.outer, (long long)lf.row_bytes);
    TB_REQUIRE(lf.row_bytes <= INT64_MAX / lf.outer / capacity / 2 && Bf + R <= INT64_MAX / lf.outer / lf.row_bytes,
               "%s: leaf %d size overflow", what, l);
    tab.leaf[l] = lf;
    tab.vec[l] = copy_width(lf);
    rows += lf.outer * (lf.out ? Bf + R : Bf);
    tab.rows_end[l] = rows;
  }
  const int warps_per_block = kReplayThreads / kWarp;
  int64_t blocks = (rows + warps_per_block - 1) / warps_per_block;
  if (blocks > int64_t(kNumSMs) * 4) blocks = int64_t(kNumSMs) * 4;  // 64 registers a thread: 4 blocks per SM resident
  const size_t smem = size_t(R) * sizeof(int64_t);  // <= 32 KB at TB_REPLAY_MAX_R, under the 48 KB default
  ProfScope prof("replay_mix", (cudaStream_t)stream);
  replay_mix_kernel<<<(unsigned)blocks, kReplayThreads, smem, (cudaStream_t)stream>>>(
      tab, Bf, R, capacity, seed_step, head_size, uint32_t(stream_id), slots_out, slots_in);
  return check_launch("replay_mix_kernel");
}

extern "C" int tb_replay_mix(const tb_replay_leaf* leaves_host, int num_leaves, int64_t Bf, int64_t R, int64_t capacity,
                             const uint64_t* seed_step, const int64_t* head_size, int64_t stream_id, int64_t* slots_out,
                             void* stream) {
  TB_REQUIRE(leaves_host && seed_step && head_size, "replay_mix: null pointer");
  return launch_mix("replay_mix", leaves_host, num_leaves, Bf, R, capacity, seed_step, head_size, stream_id, slots_out,
                    nullptr, stream);
}

extern "C" int tb_replay_mix_slots(const tb_replay_leaf* leaves_host, int num_leaves, int64_t Bf, int64_t R,
                                   int64_t capacity, const int64_t* slots, const int64_t* head_size, void* stream) {
  TB_REQUIRE(leaves_host && slots && head_size, "replay_mix_slots: null pointer");
  return launch_mix("replay_mix_slots", leaves_host, num_leaves, Bf, R, capacity, nullptr, head_size, 0, nullptr, slots,
                    stream);
}

extern "C" int tb_replay_sample_prioritized(const float* priorities, const double* prio, const int64_t* head_size,
                                            const uint64_t* seed_step, int64_t Bf, int64_t R, int64_t capacity,
                                            int64_t stream_id, int64_t* batch_slots, float* column_weights,
                                            void* stream) {
  TB_REQUIRE(priorities && prio && head_size && seed_step && batch_slots && column_weights,
             "replay_sample_prioritized: null pointer");
  TB_REQUIRE(R >= 0 && R <= TB_REPLAY_MAX_R, "replay_sample_prioritized: R must be in [0, %d], got %lld",
             TB_REPLAY_MAX_R, (long long)R);
  TB_REQUIRE(Bf >= 1, "replay_sample_prioritized: Bf must be at least 1, got %lld", (long long)Bf);
  TB_REQUIRE(capacity > Bf, "replay_sample_prioritized: capacity (%lld) must exceed Bf (%lld)", (long long)capacity,
             (long long)Bf);
  TB_REQUIRE(stream_id >= 0 && stream_id <= int64_t(UINT32_MAX),
             "replay_sample_prioritized: stream_id must be in [0, 2^32), got %lld", (long long)stream_id);
  ProfScope prof("replay_sample_prioritized", (cudaStream_t)stream);
  replay_sample_prio_kernel<<<1, kPrioChunks, 0, (cudaStream_t)stream>>>(
      priorities, prio, head_size, seed_step, Bf, R, capacity, uint32_t(stream_id), batch_slots, column_weights);
  return check_launch("replay_sample_prio_kernel");
}

extern "C" int tb_replay_update_priorities(const float* vs, const float* values, int64_t T, int64_t B,
                                           const int64_t* batch_slots, const double* prio, float* priorities,
                                           void* stream) {
  TB_REQUIRE(vs && values && batch_slots && prio && priorities, "replay_update_priorities: null pointer");
  TB_REQUIRE(T >= 1 && B >= 1, "replay_update_priorities: T and B must be at least 1, got %lld, %lld", (long long)T,
             (long long)B);
  ProfScope prof("replay_update_priorities", (cudaStream_t)stream);
  replay_update_prio_kernel<<<unsigned((B + kPrioUpdateThreads - 1) / kPrioUpdateThreads), kPrioUpdateThreads, 0,
                              (cudaStream_t)stream>>>(vs, values, T, B, batch_slots, prio, priorities);
  return check_launch("replay_update_prio_kernel");
}

extern "C" int tb_replay_advance(int64_t* head_size, uint64_t* seed_step, int64_t Bf, int64_t capacity, void* stream) {
  TB_REQUIRE(head_size && seed_step, "replay_advance: null pointer");
  TB_REQUIRE(Bf >= 1, "replay_advance: Bf must be at least 1, got %lld", (long long)Bf);
  TB_REQUIRE(capacity > Bf, "replay_advance: capacity (%lld) must exceed Bf (%lld)", (long long)capacity, (long long)Bf);
  ProfScope prof("replay_advance", (cudaStream_t)stream);
  replay_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(head_size, seed_step, Bf, capacity);
  return check_launch("replay_advance_kernel");
}
