// Shared device/host helpers of the wgmma kernels (gemm_tc.cu, conv_implicit.cu, conv3x3_sw.cu): mbarrier, TMA,
// wgmma descriptors, tensor-map construction.  Internal header: include inside namespace-less scope.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace tb {
namespace tcd {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;           // 64 bf16 = 128 bytes = one swizzle atom row
// warps 0-3: the consumer warpgroup (wgmma issue + epilogue, one accumulator row pair per thread), warp 4: TMA producer
constexpr int kConsumers = 128;
constexpr int kThreads = kConsumers + 32;
constexpr uint32_t kABytes = kBlockM * kBlockK * 2;  // 16 KB

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE_%=;\n"
      "bra LAB_WAIT_%=;\n"
      "LAB_DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// wgmma shared-memory matrix descriptor: start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32 | layout << 62 (1 = SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  // K-major, SWIZZLE_128B: SBO = 1024 B (8 rows x 128 B); LBO unused
  return uint64_t((saddr & 0x3FFFF) >> 4) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}
__device__ __forceinline__ uint64_t make_smem_desc_mn_lbo(uint32_t saddr, uint32_t lbo_bytes) {
  // MN-major, SWIZZLE_128B: LBO = byte distance between the 64-wide mn groups, SBO = 1024 B (next 8 k rows)
  return uint64_t((saddr & 0x3FFFF) >> 4) | (uint64_t(lbo_bytes >> 4) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t saddr) { return make_smem_desc_mn_lbo(saddr, 8192); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// barrier over the `threads` threads of one warpgroup role (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// split-bf16 planes of a float: hi = bf16(x), lo = bf16(x - hi); packed pairs for two consecutive elements
__device__ __forceinline__ void split_bf16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ __nv_bfloat16 bf16_lo_of(float x, __nv_bfloat16 hi) {
  return __float2bfloat16_rn(x - __bfloat162float(hi));
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

inline int make_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols = kBlockK) {
  EncodeTiledFn fn = encode_fn();
  TB_REQUIRE(fn, "gemm_tc: cuTensorMapEncodeTiled is not available from the driver");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (ld * 2) % 16 == 0,
             "gemm_tc: operand must be 16-byte aligned with a leading dimension that is a multiple of 8 (ld=%lld)",
             (long long)ld);
  cuuint64_t gdim[2] = {cuuint64_t(cols), cuuint64_t(rows)};
  cuuint64_t gstride[1] = {cuuint64_t(ld) * 2};
  cuuint32_t box[2] = {cuuint32_t(box_cols), cuuint32_t(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TB_REQUIRE(r == CUDA_SUCCESS, "gemm_tc: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", int(r),
             (long long)rows, (long long)cols, (long long)ld);
  return 0;
}


// General rank-`rank` bf16 tensor map (dims/strides innermost first; strides in BYTES for dims 1..rank-1,
// multiples of 16).  Dimensions may overlap in memory - that is how the implicit-GEMM convolutions express
// "patch (ox, oy) of frame n, kernel row offset e0" as plain TMA coordinates.
inline int make_map_nd(CUtensorMap* map, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                       const uint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = encode_fn();
  TB_REQUIRE(fn, "gemm_tc: cuTensorMapEncodeTiled is not available from the driver");
  TB_REQUIRE(rank >= 2 && rank <= 5 && (reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "gemm_tc: bad tensor map arguments");
  cuuint64_t gdim[5]; cuuint64_t gstride[4]; cuuint32_t bx[5]; cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) {
    TB_REQUIRE(strides_bytes[i] % 16 == 0, "gemm_tc: tensor map stride %d (%llu B) is not a multiple of 16", i,
               (unsigned long long)strides_bytes[i]);
    gstride[i] = strides_bytes[i];
  }
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim, gstride, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TB_REQUIRE(r == CUDA_SUCCESS, "gemm_tc: cuTensorMapEncodeTiled (rank %d) failed (%d)", rank, int(r));
  return 0;
}

}  // namespace tcd
}  // namespace tb
