// Micro-benchmarks behind the LSTM recurrence design (DESIGN.md "LSTM recurrence").
//   1. mma.sync.m16n8k16 bf16 issue rate per SM (8 / 16 warps, 12 independent accumulators)
//   2. all-gather cost: 130 CTAs each pulling the same 137 KB from L2 into shared memory (cp.async 16 B vs TMA 2D boxes)
//   3. store -> remote-poll visibility latency through L2 (one CTA stores, another spins on ld.relaxed.gpu)
//   0. (printed first) the split kernels' per-warp gather: cp.async vs TMA boxes vs 2-CTA multicast TMA vs 1-D bulk copies
//      of a slice-blocked source (with and without multicast), at 1 .. 132
//      CTAs, and whether a cooperative launch with 2-CTA clusters is accepted and co-resident at their footprint; then
//      a reduce-scatter alternative to the backward gather (fp32 pair partials through an L2 ring, fence, flags, 1 KB chunk gather),
//      and the backward's k-group gate-gradient load (16-byte cp.async vs 1-D bulk copies of a blocked ring)
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o ubench_lstm ubench_lstm.cu -lcuda
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void mma_rate_kernel(float* out, int iters, long long* cycles) {
  uint32_t a[4] = {0x3f803f80u + threadIdx.x, 0x3f803f80u, 0x3f803f80u, 0x3f803f80u};
  float acc[12][4];
#pragma unroll
  for (int i = 0; i < 12; ++i) for (int e = 0; e < 4; ++e) acc[i][e] = 0.f;
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 12; ++i) mma16816(acc[i], a, 0x3f803f80u + i, 0x3f803f80u);
  }
  long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 12; ++i) for (int e = 0; e < 4; ++e) s += acc[i][e];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

// ---- all-gather: every CTA copies `bytes` from the same global buffer into smem, `reps` times
__global__ void gather_cpasync_kernel(const uint4* __restrict__ src, int chunks, int reps, long long* cycles, uint32_t* sink) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint4* dst = reinterpret_cast<uint4*>(sm);
  __syncthreads();
  long long t0 = clock64();
  for (int r = 0; r < reps; ++r) {
    for (int i = threadIdx.x; i < chunks; i += blockDim.x) {
      uint32_t d = (uint32_t)__cvta_generic_to_shared(dst + i);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src + i) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
  }
  long long t1 = clock64();
  if (threadIdx.x == 0) { cycles[blockIdx.x] = t1 - t0; sink[blockIdx.x] = dst[5].x; }
}

__global__ void gather_tma_kernel(const __grid_constant__ CUtensorMap tm, int boxes_per_plane, int planes, int rows_per_plane, int reps,
                                  long long* cycles, uint32_t* sink) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ __align__(8) uint64_t bar;
  const uint32_t base = ((uint32_t)__cvta_generic_to_shared(sm) + 1023u) & ~1023u;
  const uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  long long t0 = clock64();
  for (int r = 0; r < reps; ++r) {
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(uint32_t(boxes_per_plane * planes * 4096)) : "memory");
      for (int p = 0; p < planes; ++p)
        for (int k = 0; k < boxes_per_plane; ++k)
          asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                           base + (p * boxes_per_plane + k) * 4096), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(b), "r"(k * 64), "r"(p * rows_per_plane)
                       : "memory");
    }
    asm volatile(
        "{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(b),
        "r"(uint32_t(r & 1)) : "memory");
    __syncthreads();
  }
  long long t1 = clock64();
  if (threadIdx.x == 0) { cycles[blockIdx.x] = t1 - t0; sink[blockIdx.x] = *reinterpret_cast<uint32_t*>(sm + 1024); }
}

// ---- ping-pong through L2: CTA 0 writes seq, CTA 1 spins and echoes, `reps` round trips
__global__ void pingpong_kernel(volatile uint32_t* a, volatile uint32_t* b, int reps, long long* cycles) {
  if (threadIdx.x != 0) return;
  long long t0 = clock64();
  if (blockIdx.x == 0) {
    for (int i = 1; i <= reps; ++i) {
      asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(a), "r"(i) : "memory");
      uint32_t v;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(b) : "memory"); } while (v != (uint32_t)i);
    }
  } else {
    for (int i = 1; i <= reps; ++i) {
      uint32_t v;
      do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a) : "memory"); } while (v != (uint32_t)i);
      asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(b), "r"(i) : "memory");
    }
  }
  cycles[blockIdx.x] = clock64() - t0;
}

// ---- fence cost: thread 0 stores 128 words (other threads too), then membar.gl; time the fence
__global__ void fence_kernel(uint32_t* buf, int reps, long long* cycles) {
  long long tot = 0;
  for (int r = 0; r < reps; ++r) {
    buf[(blockIdx.x * reps + r) * 256 + threadIdx.x] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
      long long t0 = clock64();
      asm volatile("fence.acq_rel.gpu;" ::: "memory");
      tot += clock64() - t0;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) cycles[blockIdx.x] = tot / reps;
}

// ---- split-kernel gather, the way the wavefront kernels stream their tiles: 11 warps, each owning a 48-column slice of
// every [2 planes][32 rows][528] group, `groups` groups per step through a 2-slot ring per warp (forward: 2 groups =
// 135 KB of slice bytes per CTA per step, backward: 4 = 270 KB).
//   kMode 0: per-lane 16-byte cp.async of the 48 columns (the kernels before multicast);
//   kMode 1: TMA boxes {56 cols, 16 rows, 1, 2 planes}, the CTA loads both row halves itself;
//   kMode 2: 2-CTA clusters, CTA rank r loads rows [16r, 16r + 16) with .multicast::cluster into both CTAs; a "full"
//            mbarrier per slot expects both halves, an "empty" one counts this warp and the peer's warp.
//   kMode 3: as 2, but the source is slice-blocked ([group][warp][row half][plane][16 rows][56], the warp's shared-memory
//            layout) and each half is ONE 1-D cp.async.bulk of a contiguous 3,584-byte block, multicast to the pair;
//   kMode 4: the slice-blocked source, the CTA loads both halves itself with two 1-D bulk copies (no cluster).
constexpr int kGWarps = 11, kGRowE = 56;
constexpr uint32_t kGHalf = 2 * 16 * kGRowE * 2;     // one box: 2 planes x 16 rows x 112 B
constexpr uint32_t kGSlot = 2 * kGHalf;              // both row halves
__device__ __forceinline__ void g_wait(uint32_t bar, uint32_t parity) {
  asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(bar),
               "r"(parity) : "memory");
}
__device__ __forceinline__ void g_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
template <int kMode>
__global__ void __launch_bounds__(kGWarps * 32, 1) gather_split_kernel(const __grid_constant__ CUtensorMap tm, const __nv_bfloat16* __restrict__ src,
                                                                       const uint8_t* __restrict__ blk, int hq, int groups, int reps,
                                                                       long long* cycles, uint32_t* sink) {
  constexpr bool kPair = kMode == 2 || kMode == 3;
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ __align__(8) uint64_t bars[kGWarps][4];   // full[2], empty[2]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t rank = 0;
  if (kPair) asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const uint32_t xs = (uint32_t)__cvta_generic_to_shared(sm) + w * 2 * kGSlot;
  const uint32_t full0 = (uint32_t)__cvta_generic_to_shared(&bars[w][0]), empty0 = full0 + 16;
  if (lane == 0) {
    for (int i = 0; i < 2; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full0 + 8 * i) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(empty0 + 8 * i), "r"(kPair ? 2 : 1) : "memory");
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (kPair) g_cluster_sync(); else __syncthreads();
  uint32_t peer_empty0 = 0;
  if (kPair) asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_empty0) : "r"(empty0), "r"(rank ^ 1u));
  const int total = reps * groups;
  auto issue = [&](int n) {   // group n of the stream -> slot n & 1
    const int slot = n & 1, g = n % groups;
    const uint32_t dst = xs + slot * kGSlot, full = full0 + 8 * slot;
    if (kMode == 0) {
      const __nv_bfloat16* s = src + size_t(g) * 32 * hq + w * 48;
      for (int i = 0; i < 6; ++i) {
        const int j = lane + 32 * i, r = j / 6, c = j - r * 6;
        const uint32_t d = dst + (r >> 4) * kGHalf + (r & 15) * kGRowE * 2 + c * 16;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(s + r * hq + c * 8) : "memory");
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 16 * kGRowE * 2), "l"(s + size_t(groups) * 32 * hq + r * hq + c * 8) : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      return;
    }
    if (lane != 0) return;
    if (n >= 2) g_wait(empty0 + 8 * slot, ((n >> 1) - 1) & 1);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"(kGSlot) : "memory");
    for (int h = 0; h < 2; ++h) {
      if (kPair && h != int(rank)) continue;
      const uint8_t* b = blk + (size_t(g) * kGWarps + w) * kGSlot + h * kGHalf;
      if (kMode == 3)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                     ::"r"(dst + h * kGHalf), "l"(b), "r"(kGHalf), "r"(full), "h"((uint16_t)3) : "memory");
      else if (kMode == 4)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst + h * kGHalf), "l"(b), "r"(kGHalf), "r"(full) : "memory");
      else if (kMode == 2)
        asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
                     ::"r"(dst + h * kGHalf), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(full), "r"(w * 48), "r"(16 * h), "r"(g), "r"(0), "h"((uint16_t)3)
                     : "memory");
      else
        asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                     ::"r"(dst + h * kGHalf), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(full), "r"(w * 48), "r"(16 * h), "r"(g), "r"(0)
                     : "memory");
    }
  };
  uint32_t acc = 0;
  long long t0 = clock64();
  issue(0);
  issue(1);
  for (int n = 0; n < total; ++n) {
    const int slot = n & 1;
    if (kMode == 0) {
      if (n + 1 < total) asm volatile("cp.async.wait_group 1;" ::: "memory");
      else asm volatile("cp.async.wait_group 0;" ::: "memory");
    } else {
      g_wait(full0 + 8 * slot, (n >> 1) & 1);
    }
    __syncwarp();
    acc += reinterpret_cast<const uint32_t*>(sm + w * 2 * kGSlot + slot * kGSlot)[lane];
    __syncwarp();
    if (kMode != 0 && lane == 0) {
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * slot) : "memory");
      if (kPair)
        asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(peer_empty0 + 8 * slot) : "memory");
    }
    if (n + 2 < total) issue(n + 2);
  }
  long long t1 = clock64();
  if (kPair) g_cluster_sync();
  if (lane == 0) atomicMax(reinterpret_cast<unsigned long long*>(cycles + blockIdx.x), (unsigned long long)(t1 - t0));
  if (threadIdx.x == 0) sink[blockIdx.x] = acc;
}

// occupancy / launch probe at the split kernels' footprint (352 threads, 1 CTA per SM, `smem` bytes): spins until every
// CTA of the grid has arrived, which only terminates if the whole grid is co-resident
__global__ void __launch_bounds__(kGWarps * 32, 1) coresident_probe_kernel(unsigned* count, unsigned n) {
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(count, 1u);
    unsigned v;
    do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(count) : "memory"); } while (v < n);
  }
  __syncthreads();
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- reduce-scatter exchange (an alternative to the backward all-gather, see DESIGN.md) at H = 519, B = 32: 132 CTAs in 2-CTA
// clusters, CTAs [0, 66) the upper-layer role and [66, 132) the lower-layer role, 33 pairs per role.  Per step every CTA
// meets its peer at a cluster barrier (stand-in for the DSMEM pair reduction), writes its half of the pair's fp32 partial
// products to a 2-slot ring blocked [pair][8-column block][32 rows][8] - upper role: dh and dL/dh_lower, 2 x 33 blocks =
// 66 KB; lower role: dh, 33 KB - then bar.sync, fence.acq_rel.gpu, flag; it then waits for the flags of the CTAs that hold
// its column block in every pair (lower role: of both roles) and sums 33 (66) one-KB chunks in pair order.  Before it
// overwrites a dL/dh_lower slot the upper role waits until every lower pair has read it (lower flags of the step before).
constexpr int kRsPairs = 33, kRsRole = 2 * kRsPairs, kRsFlag = 32;
constexpr size_t kRsSlotF = size_t(kRsPairs) * kRsRole * 256;   // floats in one ring slot of one product
__device__ __forceinline__ void rs_wait_flag(const unsigned* f, unsigned v) {
  unsigned x;
  do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(x) : "l"(f) : "memory"); } while (x < v);
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(x) : "l"(f) : "memory");
}
__global__ void __launch_bounds__(kGWarps * 32, 1) rs_exchange_kernel(float* rec, float* ih, unsigned* flags, int reps, long long* cycles,
                                                                      long long* phase, float* sink) {
  __shared__ float red_s[256];
  const int tid = threadIdx.x;
  const bool upper = blockIdx.x < kRsRole;
  const int cidx = upper ? blockIdx.x : blockIdx.x - kRsRole, pair = cidx >> 1, rank = cidx & 1;
  const int src_rank = cidx >= kRsPairs;   // the CTA rank that holds this CTA's column block in every pair
  float* const rec_role = rec + (upper ? 0 : 2 * kRsSlotF);
  const unsigned* const up_flags = flags;
  const unsigned* const lo_flags = flags + kRsRole * kRsFlag;
  const unsigned* const own_flags = upper ? up_flags : lo_flags;
  float acc = 0.f;
  long long ph[3] = {0, 0, 0};
  g_cluster_sync();
  const long long t0 = clock64();
  for (int s = 0; s < reps; ++s) {
    const long long p0 = clock64();
    const size_t slot = size_t(s & 1) * kRsSlotF, mine = (size_t(pair) * kRsRole + size_t(rank) * kRsPairs) * 256;
    g_cluster_sync();
    if (upper && s >= 2 && tid < kRsPairs) rs_wait_flag(lo_flags + (2 * tid) * kRsFlag, unsigned(s));
    __syncthreads();
    float4* const dr = reinterpret_cast<float4*>(rec_role + slot + mine);
    float4* const di = reinterpret_cast<float4*>(ih + slot + mine);
    for (int i = tid; i < kRsPairs * 64; i += blockDim.x) {
      const float4 v = make_float4(float(s), float(i), acc, 1.f);
      dr[i] = v;
      if (upper) di[i] = v;
    }
    __syncthreads();
    if (tid == 0) {
      asm volatile("fence.acq_rel.gpu;" ::: "memory");
      asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(flags + blockIdx.x * kRsFlag), "r"(unsigned(s + 1)) : "memory");
    }
    const long long p1 = clock64();
    if (tid < kRsPairs) rs_wait_flag(own_flags + (2 * tid + src_rank) * kRsFlag, unsigned(s + 1));
    else if (!upper && tid >= 64 && tid < 64 + kRsPairs) rs_wait_flag(up_flags + (2 * (tid - 64) + src_rank) * kRsFlag, unsigned(s + 1));
    __syncthreads();
    const long long p2 = clock64();
    if (tid < 256) {
      const float* g = rec_role + slot + size_t(cidx) * 256 + tid;
      float v[kRsPairs];
#pragma unroll
      for (int p = 0; p < kRsPairs; ++p) v[p] = __ldcg(g + size_t(p) * kRsRole * 256);
      float d = 0.f;
#pragma unroll
      for (int p = 0; p < kRsPairs; ++p) d += v[p];
      if (!upper) {
        const float* gi = ih + slot + size_t(cidx) * 256 + tid;
#pragma unroll
        for (int p = 0; p < kRsPairs; ++p) v[p] = __ldcg(gi + size_t(p) * kRsRole * 256);
#pragma unroll
        for (int p = 0; p < kRsPairs; ++p) d += v[p];
      }
      red_s[tid] = d;
    }
    __syncthreads();
    acc += red_s[tid & 255] * 1e-9f;
    const long long p3 = clock64();
    ph[0] += p1 - p0; ph[1] += p2 - p1; ph[2] += p3 - p2;
  }
  const long long t1 = clock64();
  g_cluster_sync();
  if (tid == 0) {
    cycles[blockIdx.x] = t1 - t0;
    for (int i = 0; i < 3; ++i) phase[blockIdx.x * 3 + i] = ph[i];
    sink[blockIdx.x] = acc;
  }
}

static int rs_exchange() {
  const int reps = 400, grid = 2 * kRsRole;
  const size_t smem = 150 * 1024;   // one CTA per SM, as the wavefront kernels
  float *rec, *ih, *sink; unsigned* flags; long long *cyc, *ph;
  CK(cudaMalloc(&rec, 4 * kRsSlotF * sizeof(float))); CK(cudaMalloc(&ih, 2 * kRsSlotF * sizeof(float)));
  CK(cudaMalloc(&flags, size_t(grid) * kRsFlag * 4)); CK(cudaMalloc(&cyc, grid * sizeof(long long)));
  CK(cudaMalloc(&ph, 3 * grid * sizeof(long long))); CK(cudaMalloc(&sink, grid * sizeof(float)));
  CK(cudaFuncSetAttribute(rs_exchange_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kGWarps * 32); cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  at[1].id = cudaLaunchAttributeCooperative; at[1].val.cooperative = 1;
  cfg.attrs = at; cfg.numAttrs = 2;
  int clusters = -1;
  CK(cudaOccupancyMaxActiveClusters(&clusters, rs_exchange_kernel, &cfg));
  if (clusters * 2 < grid) { printf("reduce-scatter exchange: not launched, %d co-resident 2-CTA clusters\n", clusters); return 0; }
  std::vector<long long> h(grid), hp(3 * grid);
  for (int run = 0; run < 2; ++run) {   // run 0 warms up
    CK(cudaMemset(flags, 0, size_t(grid) * kRsFlag * 4));
    CK(cudaLaunchKernelEx(&cfg, rs_exchange_kernel, rec, ih, flags, reps, cyc, ph, sink));
    CK(cudaDeviceSynchronize());
  }
  CK(cudaMemcpy(h.data(), cyc, grid * sizeof(long long), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hp.data(), ph, 3 * grid * sizeof(long long), cudaMemcpyDeviceToHost));
  for (int role = 0; role < 2; ++role) {
    long long mx = 0; double p[3] = {0, 0, 0};
    for (int i = role * kRsRole; i < (role + 1) * kRsRole; ++i) {
      mx = h[i] > mx ? h[i] : mx;
      for (int k = 0; k < 3; ++k) p[k] += double(hp[3 * i + k]) / reps / kRsRole;
    }
    printf("reduce-scatter exchange, %s role (%d CTAs of %d): write %4.1f KB + read %4.1f KB per CTA per step: %6.0f cycles/step (max CTA); "
           "mean split: cluster barrier + write + fence %5.0f, flag wait %5.0f, gather %5.0f\n",
           role ? "lower" : "upper", kRsRole, grid, role ? 33.0 : 66.0, role ? 66.0 : 33.0, double(mx) / reps, p[0], p[1], p[2]);
  }
  CK(cudaFree(rec)); CK(cudaFree(ih)); CK(cudaFree(flags)); CK(cudaFree(cyc)); CK(cudaFree(ph)); CK(cudaFree(sink));
  return 0;
}

// ---- the split backward's k-group gate-gradient load at H = 519, B = 32: 132 CTAs, the CTAs of k-group w = cta / 12 (11
// groups) each load the group's 48 columns x 4 gates x 2 planes x 32 rows (24 KB of slice bytes) into the tile layout
// [gate][row half][plane][16 rows][56] and wait for them, once per step.
//   kMode 0: from [plane][gate][row][Hq] planes, 6 16-byte cp.async per (gate, plane, row): 1,536 copies;
//   kMode 1: from a k-group-blocked ring already in the tile layout, one 1-D cp.async.bulk per gate (4 x 7 KB) on an mbarrier.
constexpr int kBgHq = 528, kBgGateB = 4 * 16 * kGRowE * 2, kBgGroupB = 4 * kBgGateB;
template <int kMode>
__global__ void __launch_bounds__(kGWarps * 32, 1) bwd_group_load_kernel(const __nv_bfloat16* __restrict__ dgq, const uint8_t* __restrict__ blk,
                                                                         int reps, long long* cycles, uint32_t* sink) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ __align__(8) uint64_t bar;
  const int tid = threadIdx.x, w = blockIdx.x / 12, ks0 = 3 * w;
  const uint32_t xs = (uint32_t)__cvta_generic_to_shared(sm), b = (uint32_t)__cvta_generic_to_shared(&bar);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  uint32_t acc = 0;
  const long long t0 = clock64();
  for (int r = 0; r < reps; ++r) {
    if (kMode == 0) {
      const size_t gs = size_t(32) * kBgHq, lo = 4 * gs;
      for (int i = tid; i < 4 * 2 * 32 * 6; i += blockDim.x) {
        const int c = i % 6, row = (i / 6) % 32, pl = (i / (6 * 32)) & 1, g = i / (12 * 32);
        const uint32_t d = xs + 2 * (g * 2 * 2 * 16 * kGRowE + (row >> 4) * 2 * 16 * kGRowE + pl * 16 * kGRowE + (row & 15) * kGRowE + c * 8);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(dgq + (pl ? lo : 0) + g * gs + size_t(row) * kBgHq + ks0 * 16 + c * 8)
                     : "memory");
      }
      asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    } else {
      if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(uint32_t(kBgGroupB)) : "memory");
        for (int g = 0; g < 4; ++g)
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                       ::"r"(xs + g * kBgGateB), "l"(blk + size_t(w) * kBgGroupB + g * kBgGateB), "r"(kBgGateB), "r"(b) : "memory");
      }
      g_wait(b, uint32_t(r & 1));
    }
    __syncthreads();
    acc += reinterpret_cast<const uint32_t*>(sm)[tid];
    __syncthreads();
  }
  const long long t1 = clock64();
  if (tid == 0) { cycles[blockIdx.x] = t1 - t0; sink[blockIdx.x] = acc; }
}

static int bwd_group_load() {
  const int reps = 400, grid = 132;
  const size_t smem = size_t(kBgGroupB) + 9 * 1024;   // the group tiles + the kernel's other dynamic shared memory
  __nv_bfloat16* dgq; uint8_t* blk; long long* cyc; uint32_t* sink;
  CK(cudaMalloc(&dgq, size_t(2) * 4 * 32 * kBgHq * 2)); CK(cudaMemset(dgq, 0, size_t(2) * 4 * 32 * kBgHq * 2));
  CK(cudaMalloc(&blk, size_t(11) * kBgGroupB)); CK(cudaMemset(blk, 0, size_t(11) * kBgGroupB));
  CK(cudaMalloc(&cyc, grid * sizeof(long long))); CK(cudaMalloc(&sink, grid * 4));
  CK(cudaFuncSetAttribute(bwd_group_load_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  CK(cudaFuncSetAttribute(bwd_group_load_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  std::vector<long long> h(grid);
  for (int mode = 0; mode < 2; ++mode) {
    for (int run = 0; run < 2; ++run) {   // run 0 warms up
      if (mode == 0) bwd_group_load_kernel<0><<<grid, kGWarps * 32, smem>>>(dgq, blk, reps, cyc, sink);
      else bwd_group_load_kernel<1><<<grid, kGWarps * 32, smem>>>(dgq, blk, reps, cyc, sink);
      CK(cudaGetLastError());
      CK(cudaDeviceSynchronize());
    }
    CK(cudaMemcpy(h.data(), cyc, grid * sizeof(long long), cudaMemcpyDeviceToHost));
    long long mx = 0; for (int i = 0; i < grid; ++i) mx = h[i] > mx ? h[i] : mx;
    printf("backward group load %-28s: %d CTAs, 24.0 KB slice bytes/CTA/step: %6.0f cycles/step (max CTA)\n",
           mode == 0 ? "1536 x 16-byte cp.async" : "4 x 7 KB 1-D bulk (blocked)", grid, double(mx) / reps);
  }
  CK(cudaFree(dgq)); CK(cudaFree(blk)); CK(cudaFree(cyc)); CK(cudaFree(sink));
  return 0;
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

template <int kMode>
static cudaError_t launch_split(cudaLaunchConfig_t& cfg, size_t smem, const CUtensorMap& tm, const __nv_bfloat16* src, const uint8_t* blk,
                                int hq, int groups, int reps, long long* cyc, uint32_t* sink) {
  cudaError_t e = cudaFuncSetAttribute(gather_split_kernel<kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e == cudaSuccess) e = cudaLaunchKernelEx(&cfg, gather_split_kernel<kMode>, tm, src, blk, hq, groups, reps, cyc, sink);
  return e;
}

static int split_gather(EncodeFn enc) {
  const int hq = 528, reps = 400;
  long long* cyc; CK(cudaMalloc(&cyc, 256 * sizeof(long long)));
  uint32_t* sink; CK(cudaMalloc(&sink, 4096));
  __nv_bfloat16* src; const size_t elems = size_t(2) * 4 * 32 * hq;   // [plane][group][row][hq]
  CK(cudaMalloc(&src, elems * 2)); CK(cudaMemset(src, 0, elems * 2));
  uint8_t* blk; const size_t blk_bytes = size_t(4) * kGWarps * kGSlot;   // [group][warp][row half][plane][16][56]
  CK(cudaMalloc(&blk, blk_bytes)); CK(cudaMemset(blk, 0, blk_bytes));
  std::vector<long long> h(256);
  static const char* names[5] = {"cp.async", "TMA", "mc TMA", "mc bulk1D", "bulk1D"};
  for (int groups : {2, 4}) {
    CUtensorMap tm;
    cuuint64_t gd[4] = {cuuint64_t(hq), 32, cuuint64_t(groups), 2};
    cuuint64_t gs[3] = {cuuint64_t(hq) * 2, cuuint64_t(32) * hq * 2, cuuint64_t(groups) * 32 * hq * 2};
    cuuint32_t bx[4] = {kGRowE, 16, 1, 2}; cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, src, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("encode failed %d\n", int(r)); return 1; }
    const size_t smem = size_t(kGWarps) * 2 * kGSlot;
    const double useful = double(groups) * 2 * 32 * kGWarps * 48 * 2;   // slice bytes per CTA per step
    const double landed = useful * kGRowE / 48;                           // bytes written into each CTA's shared memory
    for (int ctas : {1, 65, 130, 132}) {
      for (int mode = 0; mode < 5; ++mode) {
        const bool pair = mode == 2 || mode == 3;
        const int n = pair ? (ctas + 1) & ~1 : ctas;
        CK(cudaMemset(cyc, 0, 256 * sizeof(long long)));
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(n); cfg.blockDim = dim3(kGWarps * 32); cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 2;
        at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = pair ? 1 : 0;
        const __nv_bfloat16* sp = src;
        if (mode == 0) CK(launch_split<0>(cfg, smem, tm, sp, blk, hq, groups, reps, cyc, sink));
        if (mode == 1) CK(launch_split<1>(cfg, smem, tm, sp, blk, hq, groups, reps, cyc, sink));
        if (mode == 2) CK(launch_split<2>(cfg, smem, tm, sp, blk, hq, groups, reps, cyc, sink));
        if (mode == 3) CK(launch_split<3>(cfg, smem, tm, sp, blk, hq, groups, reps, cyc, sink));
        if (mode == 4) CK(launch_split<4>(cfg, smem, tm, sp, blk, hq, groups, reps, cyc, sink));
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), cyc, n * sizeof(long long), cudaMemcpyDeviceToHost));
        long long mx = 0; for (int i = 0; i < n; ++i) mx = h[i] > mx ? h[i] : mx;
        const double cps = double(mx) / reps;
        printf("split gather %-9s: %3d CTAs, %5.1f KB slice bytes (%5.1f KB landed)/CTA/step: %7.0f cycles/step (max CTA), %5.1f B/clk/SM, "
               "chip %6.0f B/clk read from L2\n",
               names[mode], n, useful / 1024.0, landed / 1024.0, cps, useful / cps,
               n * (mode == 0 ? useful : pair ? landed / 2 : landed) / cps);
      }
    }
  }
  // cooperative + 2-CTA cluster launch at the kernels' footprint
  int dev = 0, sms = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  unsigned* cnt; CK(cudaMalloc(&cnt, 4));
  struct { const char* name; size_t smem; int grid; } probes[] = {
      {"forward  (130 CTAs, 208 KB)", 157696 + 46464 + 4224, 130},
      {"backward (132 CTAs, 196 KB)", 157696 + 23232 + 9216 + 6272, 132}};
  for (auto& p : probes) {
    CK(cudaFuncSetAttribute(coresident_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(p.smem)));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.grid); cfg.blockDim = dim3(kGWarps * 32); cfg.dynamicSmemBytes = p.smem;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeCooperative; at[1].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 2;
    int clusters = -1;
    cudaError_t e = cudaOccupancyMaxActiveClusters(&clusters, coresident_probe_kernel, &cfg);
    printf("%s: cudaOccupancyMaxActiveClusters(2-CTA) = %d (%s), SMs %d\n", p.name, clusters, cudaGetErrorString(e), sms);
    CK(cudaMemset(cnt, 0, 4));
    if (clusters * 2 >= p.grid) {
      e = cudaLaunchKernelEx(&cfg, coresident_probe_kernel, cnt, unsigned(p.grid));
      cudaError_t e2 = cudaDeviceSynchronize();
      printf("  cooperative + cluster {2,1,1} launch of %d CTAs: launch %s, sync %s\n", p.grid, cudaGetErrorString(e), cudaGetErrorString(e2));
      if (e != cudaSuccess) cudaGetLastError();
    } else {
      printf("  not launched: the grid would not be co-resident\n");
    }
  }
  return 0;
}

int main() {
  {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    printf("device %s, %d SMs\n", prop.name, prop.multiProcessorCount);    EncodeFn enc = nullptr; cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &q));
    if (split_gather(enc)) return 1;
    if (rs_exchange()) return 1;
    if (bwd_group_load()) return 1;
  }
  int clk = 0;
  cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  printf("sm clock (attr) %.0f MHz\n", clk / 1000.0);
  long long* cyc; CK(cudaMalloc(&cyc, 1024 * sizeof(long long)));
  float* out; CK(cudaMalloc(&out, 148 * 512 * sizeof(float)));
  uint32_t* sink; CK(cudaMalloc(&sink, 4096));
  std::vector<long long> h(1024);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  // 1. mma rate
  for (int warps : {4, 8, 16}) {
    const int iters = 2000;
    mma_rate_kernel<<<148, warps * 32>>>(out, iters, cyc);
    CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    mma_rate_kernel<<<148, warps * 32>>>(out, iters, cyc);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    CK(cudaMemcpy(h.data(), cyc, 148 * sizeof(long long), cudaMemcpyDeviceToHost));
    const double mmas = double(warps) * iters * 12;
    printf("mma.sync m16n8k16 bf16: %2d warps/SM: %.2f cycles per MMA per SM (%.1f per SMSP-MMA), %.0f flop/clk/SM, chip %.1f TFLOP/s\n", warps,
           h[0] / mmas, h[0] / mmas * 4, mmas * 4096 / h[0], 148 * mmas * 4096 / (ms * 1e-3) / 1e12);
  }
  // 2. all-gather
  const int rows = 32, hq = 576;  // 9 boxes of 64 per row
  const size_t plane = size_t(rows) * hq * 2;
  uint8_t* src; CK(cudaMalloc(&src, plane * 4 * 4)); CK(cudaMemset(src, 1, plane * 4 * 4));
  EncodeFn enc = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &q));
  CUtensorMap tm;
  { cuuint64_t gd[2] = {hq, cuuint64_t(rows) * 4}; cuuint64_t gs[1] = {hq * 2}; cuuint32_t bx[2] = {64, 32}; cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, src, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("encode failed %d\n", int(r)); return 1; } }
  const int reps = 200;
  for (int ctas : {1, 65, 130, 148}) {
    for (int planes : {2, 4}) {
      const int chunks = int(plane * planes / 16);
      CK(cudaFuncSetAttribute(gather_cpasync_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      CK(cudaFuncSetAttribute(gather_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      for (int thr : {256, 512}) {
        gather_cpasync_kernel<<<ctas, thr, plane * planes>>>(reinterpret_cast<uint4*>(src), chunks, reps, cyc, sink);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), cyc, ctas * sizeof(long long), cudaMemcpyDeviceToHost));
        long long mx = 0; for (int i = 0; i < ctas; ++i) mx = h[i] > mx ? h[i] : mx;
        printf("gather cp.async  : %3d CTAs x %d thr, %6.1f KB/step: %.0f cycles/step (max), %.1f B/clk/SM, chip %.0f B/clk\n", ctas, thr,
               plane * planes / 1024.0, double(mx) / reps, plane * planes * reps / double(mx), ctas * plane * planes * reps / double(mx));
      }
      gather_tma_kernel<<<ctas, 256, plane * planes + 2048>>>(tm, 9, planes, rows, reps, cyc, sink);
      CK(cudaDeviceSynchronize());
      CK(cudaMemcpy(h.data(), cyc, ctas * sizeof(long long), cudaMemcpyDeviceToHost));
      long long mx = 0; for (int i = 0; i < ctas; ++i) mx = h[i] > mx ? h[i] : mx;
      printf("gather TMA boxes : %3d CTAs, %6.1f KB/step: %.0f cycles/step (max), %.1f B/clk/SM, chip %.0f B/clk\n", ctas,
             plane * planes / 1024.0, double(mx) / reps, plane * planes * reps / double(mx), ctas * plane * planes * reps / double(mx));
    }
  }
  // 3. ping-pong
  uint32_t* flags; CK(cudaMalloc(&flags, 1024)); CK(cudaMemset(flags, 0, 1024));
  pingpong_kernel<<<2, 32>>>(flags, flags + 64, 2000, cyc);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h.data(), cyc, 2 * sizeof(long long), cudaMemcpyDeviceToHost));
  printf("L2 ping-pong: %.0f cycles per round trip (two store->poll hand-offs) => %.0f cycles per hand-off\n", h[0] / 2000.0, h[0] / 4000.0);
  // 4. fence
  uint32_t* fb; CK(cudaMalloc(&fb, size_t(148) * 100 * 256 * 4));
  fence_kernel<<<130, 256>>>(fb, 100, cyc);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h.data(), cyc, 130 * sizeof(long long), cudaMemcpyDeviceToHost));
  long long mxf = 0, sm = 0; for (int i = 0; i < 130; ++i) { mxf = h[i] > mxf ? h[i] : mxf; sm += h[i]; }
  printf("fence.acq_rel.gpu after 256 fresh stores/CTA, 130 CTAs: mean %.0f cycles, worst CTA %lld\n", sm / 130.0, mxf);
  return 0;
}
