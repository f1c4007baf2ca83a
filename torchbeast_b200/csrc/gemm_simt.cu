// Instantiations + host launcher of the fp32 SIMT GEMM (see gemm_simt.cuh).
#include "gemm_simt.cuh"

namespace tb {

// Thread = 4 consecutive columns of one output row (one 16-byte load per split when the partial rows are
// 16-byte aligned), block = 128 threads x 4 rows; no 64-bit div/mod, the split loop keeps `splits` loads in flight.
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, float* __restrict__ C, int64_t M, int64_t N,
                                     int64_t ldc, int splits, GemmEpilogue ep, int64_t ldp) {
  const int n0 = (blockIdx.x * 128 + threadIdx.x) * 4;
  if (n0 >= N) return;
  const int64_t slice = M * ldp;  // partial rows are ldp floats apart (ldp >= N: padded so the GEMM stores 16 bytes)
  const bool vec = (ldp & 3) == 0 && (reinterpret_cast<uintptr_t>(partial) & 15) == 0 && n0 + 4 <= ldp;
  const int nv = (N - n0 < 4) ? int(N - n0) : 4;
  int nd[4]; float bias[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = n0 + j;
    nd[j] = n;
    if ((ep.permP > 1 || ep.permQ > 1) && j < nv) {
      const int p = n / ep.permQ, q = n - p * ep.permQ;
      nd[j] = q * ep.permP + p;
    }
    bias[j] = (ep.bias && j < nv) ? __ldg(ep.bias + n) : 0.0f;
  }
  for (int64_t m = int64_t(blockIdx.y) * blockDim.y + threadIdx.y; m < M; m += int64_t(gridDim.y) * blockDim.y) {
    const float* p = partial + m * ldp + n0;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (vec) {
      // 16 loads in flight per thread (same summation order): with one split per SM and unroll 4 the conv1 reduce was 37 dependent
      // L2 round trips for a 4.8 MB read
#pragma unroll 16
      for (int z = 0; z < splits; ++z) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p + int64_t(z) * slice));
        v[0] += t.x; v[1] += t.y; v[2] += t.z; v[3] += t.w;
      }
    } else {
      for (int z = 0; z < splits; ++z)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < nv) v[j] += __ldg(p + int64_t(z) * slice + j);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= nv) break;
      float x = v[j] * ep.scale + bias[j];
      if (ep.relu) x = fmaxf(x, 0.0f);
      float* c = C + m * ldc + nd[j];
      *c = ep.accumulate ? (*c + x) : x;
    }
  }
}

int launch_splitk_reduce(const float* partial, float* C, int64_t M, int64_t N, int64_t ldc, int splits, const GemmEpilogue& ep,
                         int64_t ldp, cudaStream_t stream) {
  if (M == 0 || N == 0) return 0;
  const int64_t gy = (M + 3) / 4;
  dim3 grid((unsigned)((N + 511) / 512), (unsigned)(gy < 65535 ? gy : 65535));
  splitk_reduce_kernel<<<grid, dim3(128, 4), 0, stream>>>(partial, C, M, N, ldc, splits, ep, ldp);
  return check_launch("splitk_reduce_kernel");
}

template <typename AT, typename BT, bool TA, bool TB, int BM, int BN>
static void launch_tile(const GemmArgs& g, cudaStream_t stream) {
  dim3 grid((unsigned)((g.M + BM - 1) / BM), (unsigned)((g.N + BN - 1) / BN), (unsigned)g.splits);
  gemm_simt_kernel<AT, BT, TA, TB, BM, BN><<<grid, kGemmThreads, 0, stream>>>(g);
}

template <typename AT, typename BT, bool TA, bool TB>
int gemm_simt(const AT* A, const BT* B, float* C, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
              int64_t ldc, const GemmEpilogue& ep, int splits, float* splitk_scratch, cudaStream_t stream) {
  TB_REQUIRE(M >= 0 && N >= 0 && K >= 0, "gemm: negative size");
  if (M == 0 || N == 0) return 0;
  TB_REQUIRE(A && B && C, "gemm: null pointer");
  if (splits < 1) splits = 1;
  const int64_t ktiles = (K + kGemmBK - 1) / kGemmBK;
  if (splits > ktiles) splits = int(ktiles > 0 ? ktiles : 1);
  const bool via_scratch = splits > 1 || ep.permP > 1 || ep.permQ > 1;
  TB_REQUIRE(!via_scratch || splitk_scratch, "gemm: split-K / permuted output needs scratch");
  // each path applies only part of the epilogue: reject what the chosen one would drop
  TB_REQUIRE(via_scratch ? !ep.mask && !ep.addend : ep.scale == 1.0f,
             "gemm: %s epilogue with %s", via_scratch ? "split-K / permuted" : "direct",
             via_scratch ? "mask / addend (direct path only)" : "scale != 1 (split-K / permuted path only)");
  ProfScope prof(ep.tag, stream);
  GemmArgs g;
  g.A = A; g.B = B; g.C = C; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
  g.partial = via_scratch ? splitk_scratch : nullptr; g.splits = splits; g.ep = ep;
  if (N <= 32) {
    launch_tile<AT, BT, TA, TB, 128, 32>(g, stream);
  } else if (M <= 64) {
    launch_tile<AT, BT, TA, TB, 64, 64>(g, stream);
  } else {
    launch_tile<AT, BT, TA, TB, 128, 64>(g, stream);
  }
  int rc = check_launch("gemm_simt_kernel");
  if (rc) return rc;
  if (via_scratch) {
    const int64_t total = M * N;
    int64_t blocks = (total + 255) / 256;
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    rc = launch_splitk_reduce(splitk_scratch, C, M, N, ldc, splits, ep, N, stream);
  }
  return rc;
}

#define TB_INST(AT, BT, TA, TB_)                                                                          \
  template int gemm_simt<AT, BT, TA, TB_>(const AT*, const BT*, float*, int64_t, int64_t, int64_t, int64_t, \
                                          int64_t, int64_t, const GemmEpilogue&, int, float*, cudaStream_t);
TB_INST(float, float, false, true)     // forward:  act = col . W^T
TB_INST(uint8_t, float, false, true)   // forward conv1 on the uint8 patch matrix
TB_INST(float, float, false, false)    // dgrad:    dcol = dY . W
TB_INST(float, float, true, false)     // wgrad:    dW = dY^T . col
TB_INST(float, uint8_t, true, false)   // wgrad conv1
#undef TB_INST

}  // namespace tb
