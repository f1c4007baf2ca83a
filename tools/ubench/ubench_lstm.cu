// Micro-benchmarks behind the LSTM recurrence design (DESIGN.md "LSTM recurrence").
//   1. mma.sync.m16n8k16 bf16 issue rate per SM (8 / 16 warps, 12 independent accumulators)
//   2. all-gather cost: 130 CTAs each pulling the same 137 KB from L2 into shared memory (cp.async 16 B vs TMA 2D boxes)
//   3. store -> remote-poll visibility latency through L2 (one CTA stores, another spins on ld.relaxed.gpu)
//   0. (printed first) the split kernels' per-warp gather: cp.async vs TMA boxes vs 2-CTA multicast TMA, at 1 .. 132
//      CTAs, and whether a cooperative launch with 2-CTA clusters is accepted and co-resident at their footprint
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
                                                                       int hq, int groups, int reps, long long* cycles, uint32_t* sink) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ __align__(8) uint64_t bars[kGWarps][4];   // full[2], empty[2]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t rank = 0;
  if (kMode == 2) asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const uint32_t xs = (uint32_t)__cvta_generic_to_shared(sm) + w * 2 * kGSlot;
  const uint32_t full0 = (uint32_t)__cvta_generic_to_shared(&bars[w][0]), empty0 = full0 + 16;
  if (lane == 0) {
    for (int i = 0; i < 2; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full0 + 8 * i) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(empty0 + 8 * i), "r"(kMode == 2 ? 2 : 1) : "memory");
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (kMode == 2) g_cluster_sync(); else __syncthreads();
  uint32_t peer_empty0 = 0;
  if (kMode == 2) asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_empty0) : "r"(empty0), "r"(rank ^ 1u));
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
      if (kMode == 2 && h != int(rank)) continue;
      if (kMode == 2)
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
      if (kMode == 2)
        asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(peer_empty0 + 8 * slot) : "memory");
    }
    if (n + 2 < total) issue(n + 2);
  }
  long long t1 = clock64();
  if (kMode == 2) g_cluster_sync();
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

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int split_gather(EncodeFn enc) {
  const int hq = 528, reps = 400;
  long long* cyc; CK(cudaMalloc(&cyc, 256 * sizeof(long long)));
  uint32_t* sink; CK(cudaMalloc(&sink, 4096));
  __nv_bfloat16* src; const size_t elems = size_t(2) * 4 * 32 * hq;   // [plane][group][row][hq]
  CK(cudaMalloc(&src, elems * 2)); CK(cudaMemset(src, 0, elems * 2));
  std::vector<long long> h(256);
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
    for (int ctas : {1, 65, 130, 132}) {
      for (int mode = 0; mode < 3; ++mode) {
        const int n = (mode == 2) ? (ctas + 1) & ~1 : ctas;
        CK(cudaMemset(cyc, 0, 256 * sizeof(long long)));
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(n); cfg.blockDim = dim3(kGWarps * 32); cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 2;
        at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = mode == 2 ? 1 : 0;
        if (mode == 0) { CK(cudaFuncSetAttribute(gather_split_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
                         CK(cudaLaunchKernelEx(&cfg, gather_split_kernel<0>, tm, (const __nv_bfloat16*)src, hq, groups, reps, cyc, sink)); }
        if (mode == 1) { CK(cudaFuncSetAttribute(gather_split_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
                         CK(cudaLaunchKernelEx(&cfg, gather_split_kernel<1>, tm, (const __nv_bfloat16*)src, hq, groups, reps, cyc, sink)); }
        if (mode == 2) { CK(cudaFuncSetAttribute(gather_split_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
                         CK(cudaLaunchKernelEx(&cfg, gather_split_kernel<2>, tm, (const __nv_bfloat16*)src, hq, groups, reps, cyc, sink)); }
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), cyc, n * sizeof(long long), cudaMemcpyDeviceToHost));
        long long mx = 0; for (int i = 0; i < n; ++i) mx = h[i] > mx ? h[i] : mx;
        const double cps = double(mx) / reps;
        printf("split gather %-9s: %3d CTAs, %5.1f KB slice bytes/CTA/step: %7.0f cycles/step (max CTA), %5.1f B/clk/SM, chip %6.0f B/clk read from L2\n",
               mode == 0 ? "cp.async" : mode == 1 ? "TMA" : "multicast", n, useful / 1024.0, cps, useful / cps,
               n * (mode == 0 ? useful : mode == 1 ? useful * kGRowE / 48 : useful * kGRowE / 48 / 2) / cps);
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
    printf("device %s, %d SMs\n", prop.name, prop.multiProcessorCount);
    EncodeFn enc = nullptr; cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &q));
    if (split_gather(enc)) return 1;
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
