// fp32 SIMT GEMM for sm_90a: the exact-arithmetic ("fp32") backend of the network path.
//
//   C[M,N] (+)= sum_k A(m,k) * B(k,n)            fp32 accumulate, fp32 FFMA
//   A(m,k) = TA ? A[k*lda + m] : A[m*lda + k]    (AT = float or uint8; uint8 is read as x/255.f,
//   B(k,n) = TB ? B[n*ldb + k] : B[k*ldb + n]     the reference's `frame.float()/255` rounding)
//
// Tiling: CTA tile BM x BN, K step 16, 256 threads, TM x TN register micro-tile, operands
// staged through shared memory stored k-major ([BK][BM+4]) so the inner product reads are
// 128-bit and conflict-free, next K tile prefetched into registers while the current one is
// consumed.  grid.z = split-K slices; with splits > 1 each slice writes its partial tile to
// `partial` ([z][M][N]) and splitk_reduce_kernel folds them in a fixed order (deterministic).
//
// This backend keeps the learner bit-comparable with the reference's fp32 CPU arithmetic
// (parity tests); the tensor-core backend (wgmma) replaces it for throughput.
#pragma once
#include "common.cuh"

namespace tb {

struct GemmEpilogue {
  const float* bias = nullptr;   // [N], added per output column
  int relu = 0;                  // max(x, 0)
  const float* mask = nullptr;   // [M, ldmask]: C = acc * (mask > 0)   (ReLU backward)
  int64_t ldmask = 0;
  int accumulate = 0;            // C += acc
  const float* addend = nullptr; // [M, ldadd]: C = acc + bias + addend (residual connection), applied last
  int64_t ldadd = 0;
  // split-K reduce only: output column permutation n = p*Q + q  ->  q*P + p (weight-grad unpack)
  int permP = 1, permQ = 1;
  float scale = 1.0f;            // (split-K reduce only) multiplies the reduced sum
  const char* tag = "gemm";    // op name reported by the profiler
};

struct GemmArgs {
  const void* A; const void* B; float* C;
  int64_t M, N, K, lda, ldb, ldc;
  float* partial;  // non-null: write raw partial tiles [z][M][N] for splitk_reduce_kernel
  int splits;
  GemmEpilogue ep;
};

template <typename T> __device__ __forceinline__ float load_as_f32(const T* p);
template <> __device__ __forceinline__ float load_as_f32<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float load_as_f32<uint8_t>(const uint8_t* p) { return float(__ldg(p)) / 255.0f; }

constexpr int kGemmBK = 16;
constexpr int kGemmThreads = 256;

template <typename AT, typename BT, bool TA, bool TB, int BM, int BN>
__global__ void __launch_bounds__(kGemmThreads) gemm_simt_kernel(GemmArgs g) {
  constexpr int BK = kGemmBK;
  constexpr int TN = BN / 16;          // 16 thread columns
  constexpr int TM = BM / 16;          // 16 thread rows
  constexpr int LA = BM * BK / kGemmThreads;
  constexpr int LB = BN * BK / kGemmThreads;
  static_assert(TM % 4 == 0 && (TN == 2 || TN % 4 == 0), "micro-tile");
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];

  const AT* __restrict__ A = reinterpret_cast<const AT*>(g.A);
  const BT* __restrict__ B = reinterpret_cast<const BT*>(g.B);
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = int64_t(blockIdx.x) * BM, n0 = int64_t(blockIdx.y) * BN;  // M tiles on grid.x (no 65535 limit)
  // K range of this split (multiple of BK except the last)
  const int64_t ktiles = (g.K + BK - 1) / BK;
  const int64_t per = (ktiles + g.splits - 1) / g.splits;
  const int64_t kbeg = int64_t(blockIdx.z) * per * BK;
  int64_t kend = kbeg + per * BK;
  if (kend > g.K) kend = g.K;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

  float ra[LA], rb[LB];
  auto load_tiles = [&](int64_t k0) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int idx = tid + i * kGemmThreads;
      int mm, kk;
      if (TA) { kk = idx / BM; mm = idx % BM; } else { mm = idx / BK; kk = idx % BK; }
      const int64_t m = m0 + mm, k = k0 + kk;
      float v = 0.0f;
      if (m < g.M && k < kend) v = load_as_f32<AT>(TA ? A + k * g.lda + m : A + m * g.lda + k);
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int idx = tid + i * kGemmThreads;
      int nn, kk;
      if (TB) { nn = idx / BK; kk = idx % BK; } else { kk = idx / BN; nn = idx % BN; }
      const int64_t n = n0 + nn, k = k0 + kk;
      float v = 0.0f;
      if (n < g.N && k < kend) v = load_as_f32<BT>(TB ? B + n * g.ldb + k : B + k * g.ldb + n);
      rb[i] = v;
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int idx = tid + i * kGemmThreads;
      int mm, kk;
      if (TA) { kk = idx / BM; mm = idx % BM; } else { mm = idx / BK; kk = idx % BK; }
      As[kk][mm] = ra[i];
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int idx = tid + i * kGemmThreads;
      int nn, kk;
      if (TB) { nn = idx / BK; kk = idx % BK; } else { kk = idx / BN; nn = idx % BN; }
      Bs[kk][nn] = rb[i];
    }
  };

  if (kbeg < kend) {
    load_tiles(kbeg);
    for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
      store_tiles();
      __syncthreads();
      if (k0 + BK < kend) load_tiles(k0 + BK);
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[TM], b[TN];
#pragma unroll
        for (int i = 0; i < TM; i += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
          a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
        }
        if constexpr (TN == 2) {
          const float2 v = *reinterpret_cast<const float2*>(&Bs[kk][tx * TN]);
          b[0] = v.x; b[1] = v.y;
        } else {
#pragma unroll
          for (int j = 0; j < TN; j += 4) {
            const float4 v = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN + j]);
            b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
          }
        }
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

  if (g.partial) {
    float* P = g.partial + int64_t(blockIdx.z) * g.M * g.N;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int64_t m = m0 + ty * TM + i;
      if (m >= g.M) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int64_t n = n0 + tx * TN + j;
        if (n < g.N) P[m * g.N + n] = acc[i][j];
      }
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t m = m0 + ty * TM + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int64_t n = n0 + tx * TN + j;
      if (n >= g.N) continue;
      float v = acc[i][j];
      if (g.ep.bias) v += g.ep.bias[n];
      if (g.ep.relu) v = fmaxf(v, 0.0f);
      if (g.ep.mask) v = (g.ep.mask[m * g.ep.ldmask + n] > 0.0f) ? v : 0.0f;
      if (g.ep.addend) v += g.ep.addend[m * g.ep.ldadd + n];
      float* c = g.C + m * g.ldc + n;
      *c = g.ep.accumulate ? (*c + v) : v;
    }
  }
}

// out[m, perm(n)] (+)= sum_z partial[z][m][n] (+bias, relu) - fixed summation order.
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, float* __restrict__ C, int64_t M, int64_t N,
                                     int64_t ldc, int splits, GemmEpilogue ep, int64_t ldp);
int launch_splitk_reduce(const float* partial, float* C, int64_t M, int64_t N, int64_t ldc, int splits, const GemmEpilogue& ep,
                         int64_t ldp, cudaStream_t stream);

// Host launcher.  `splitk_scratch` must hold splits*M*N floats when splits > 1.
template <typename AT, typename BT, bool TA, bool TB>
int gemm_simt(const AT* A, const BT* B, float* C, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
              int64_t ldc, const GemmEpilogue& ep, int splits, float* splitk_scratch, cudaStream_t stream);

}  // namespace tb
