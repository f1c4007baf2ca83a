// Micro-benchmarks behind the LSTM recurrence design (DESIGN.md "LSTM recurrence").
//   1. mma.sync.m16n8k16 bf16 issue rate per SM (8 / 16 warps, 12 independent accumulators)
//   2. all-gather cost: 130 CTAs each pulling the same 137 KB from L2 into shared memory (cp.async 16 B vs TMA 2D boxes)
//   3. store -> remote-poll visibility latency through L2 (one CTA stores, another spins on ld.relaxed.gpu)
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

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
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
