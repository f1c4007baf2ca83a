// Experience replay for the learner batch on sm_90a (H100): the contract is tb_replay_mix in include/torchbeast_b200.h.
//
// One launch copies every row of every leaf: a row is one (outer index, column) pair of row_bytes bytes, and each warp
// takes one row at a time, grid-stride over all rows of all leaves.  A fresh row is read once and written twice (mixed
// batch, ring slot); a replayed row is read from its ring slot and written once.  Every block draws the R slots itself
// into shared memory (R Philox calls, spread over its threads), so no block waits on another and there are no atomics.
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

__global__ void __launch_bounds__(kReplayThreads) replay_mix_kernel(const ReplayTable tab, int64_t Bf, int64_t R,
                                                                    int64_t capacity,
                                                                    const uint64_t* __restrict__ seed_step,
                                                                    const int64_t* __restrict__ head_size,
                                                                    uint32_t stream_id,
                                                                    int64_t* __restrict__ slots_out) {
  extern __shared__ int64_t slots[];  // [R]
  const uint64_t seed = seed_step[0], step = seed_step[1];
  const int64_t head = head_size[0], size = head_size[1];
  const int64_t n = size < capacity - Bf ? size : capacity - Bf;
  for (int64_t j = threadIdx.x; j < R; j += blockDim.x) {
    const uint32_t x = philox4x32_10_w0(uint32_t(step), uint32_t(step >> 32), uint32_t(j), stream_id, uint32_t(seed),
                                        uint32_t(seed >> 32));
    const int64_t k = int64_t((uint64_t(x) * uint64_t(n)) >> 32);
    const int64_t slot = (head - 1 - k + capacity) % capacity;  // k < n <= capacity - Bf, so the sum is >= 0
    slots[j] = slot;
    if (blockIdx.x == 0 && slots_out) slots_out[j] = slot;
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

extern "C" int tb_replay_mix(const tb_replay_leaf* leaves_host, int num_leaves, int64_t Bf, int64_t R, int64_t capacity,
                             const uint64_t* seed_step, const int64_t* head_size, int64_t stream_id, int64_t* slots_out,
                             void* stream) {
  TB_REQUIRE(leaves_host && seed_step && head_size, "replay_mix: null pointer");
  TB_REQUIRE(num_leaves >= 1 && num_leaves <= TB_REPLAY_MAX_LEAVES, "replay_mix: num_leaves must be in [1, %d], got %d",
             TB_REPLAY_MAX_LEAVES, num_leaves);
  TB_REQUIRE(R >= 0 && R <= TB_REPLAY_MAX_R, "replay_mix: R must be in [0, %d], got %lld", TB_REPLAY_MAX_R, (long long)R);
  TB_REQUIRE(Bf >= 1, "replay_mix: Bf must be at least 1, got %lld", (long long)Bf);
  TB_REQUIRE(capacity > Bf, "replay_mix: capacity (%lld) must exceed Bf (%lld)", (long long)capacity, (long long)Bf);
  TB_REQUIRE(stream_id >= 0 && stream_id <= int64_t(UINT32_MAX), "replay_mix: stream_id must be in [0, 2^32), got %lld",
             (long long)stream_id);
  ReplayTable tab = {};
  tab.num_leaves = num_leaves;
  int64_t rows = 0;
  for (int l = 0; l < num_leaves; ++l) {
    const tb_replay_leaf& lf = leaves_host[l];
    TB_REQUIRE(lf.fresh && lf.ring, "replay_mix: null pointer in leaf %d", l);
    TB_REQUIRE(lf.outer >= 1 && lf.row_bytes >= 1, "replay_mix: leaf %d needs outer >= 1 and row_bytes >= 1, got %lld, %lld",
               l, (long long)lf.outer, (long long)lf.row_bytes);
    TB_REQUIRE(lf.row_bytes <= INT64_MAX / lf.outer / capacity / 2 && Bf + R <= INT64_MAX / lf.outer / lf.row_bytes,
               "replay_mix: leaf %d size overflow", l);
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
      tab, Bf, R, capacity, seed_step, head_size, uint32_t(stream_id), slots_out);
  return check_launch("replay_mix_kernel");
}

extern "C" int tb_replay_advance(int64_t* head_size, uint64_t* seed_step, int64_t Bf, int64_t capacity, void* stream) {
  TB_REQUIRE(head_size && seed_step, "replay_advance: null pointer");
  TB_REQUIRE(Bf >= 1, "replay_advance: Bf must be at least 1, got %lld", (long long)Bf);
  TB_REQUIRE(capacity > Bf, "replay_advance: capacity (%lld) must exceed Bf (%lld)", (long long)capacity, (long long)Bf);
  ProfScope prof("replay_advance", (cudaStream_t)stream);
  replay_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(head_size, seed_step, Bf, capacity);
  return check_launch("replay_advance_kernel");
}
