// Shared host/device helpers for the torchbeast_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/torchbeast_b200.h"

namespace tb {

// ---- error plumbing (thread-local, see header conventions) --------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);  // cudaGetLastError + launch counter

// Optional per-op device timing (tb_profile_*): when enabled, every ProfScope records a CUDA
// event pair on the op's stream; off by default (zero overhead beyond one branch).
struct ProfScope {
  ProfScope(const char* name, cudaStream_t stream);
  ~ProfScope();
  int slot;
  cudaStream_t stream;
};

#define TB_REQUIRE(cond, ...)      \
  do {                             \
    if (!(cond)) {                 \
      ::tb::set_error(__VA_ARGS__); \
      return 1;                    \
    }                              \
  } while (0)

// forwards a non-zero status (the callee has already set the error message)
#define TB_TRY(expr)     \
  do {                   \
    int _rc = (expr);    \
    if (_rc) return _rc; \
  } while (0)

constexpr int kWarp = 32;
constexpr int kNumSMs = 132;  // H100 SXM
// workspace layout: [0] uint32 ticket counter (self-resetting), then kMaxPartialCtas per-CTA partials of up to
// kMaxPartialSums doubles each (grid_sum3: stride 4, grid_sum<N>: stride N)
constexpr int kMaxPartialCtas = 4096;
constexpr int kMaxPartialSums = 5;
constexpr size_t kWorkspaceBytes = 64 + size_t(kMaxPartialCtas) * kMaxPartialSums * sizeof(double);

template <typename F> struct M;
template <> struct M<float> {
  static __device__ __forceinline__ float exp(float x) { return expf(x); }
  static __device__ __forceinline__ float log(float x) { return logf(x); }
  static __device__ __forceinline__ float min(float a, float b) { return fminf(a, b); }
  static __device__ __forceinline__ float max(float a, float b) { return fmaxf(a, b); }
};
template <> struct M<double> {
  static __device__ __forceinline__ double exp(double x) { return ::exp(x); }
  static __device__ __forceinline__ double log(double x) { return ::log(x); }
  static __device__ __forceinline__ double min(double a, double b) { return fmin(a, b); }
  static __device__ __forceinline__ double max(double a, double b) { return fmax(a, b); }
};

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): words 0 and 1 of the output.
// Shared by the action sampler (sample.cu) and the replay slot draws (replay.cu); the uniform draws use word 0 only,
// the prioritised draws both.
__device__ __forceinline__ uint2 philox4x32_10_w01(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                   uint32_t k1) {
  constexpr uint32_t kM0 = 0xD2511F53u, kM1 = 0xCD9E8D57u, kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(kM0, c0), lo0 = kM0 * c0;
    const uint32_t hi1 = __umulhi(kM1, c2), lo1 = kM1 * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += kW0;
    k1 += kW1;
  }
  return make_uint2(c0, c1);
}
__device__ __forceinline__ uint32_t philox4x32_10_w0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                     uint32_t k1) {
  return philox4x32_10_w01(c0, c1, c2, c3, k0, k1).x;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Deterministic grid-wide sum of up to 3 doubles per thread.
// Every thread of every CTA must call this (it contains __syncthreads).  Returns true in
// exactly ONE thread of the whole grid (thread 0 of the CTA that finishes last), with the
// grid totals in tot[0..2]; partials are combined in CTA-index order so the result does not
// depend on scheduling.  `ws` is the caller's zero-initialised workspace; the ticket counter
// is reset before returning so the workspace can be reused by the next launch on the stream.
__device__ __forceinline__ bool grid_sum3(double s0, double s1, double s2, void* ws, double* tot) {
  __shared__ double sm[32][3];
  __shared__ bool is_last;
  const int tid = threadIdx.x + threadIdx.y * blockDim.x;
  const int nthreads = blockDim.x * blockDim.y;
  const int warp = tid >> 5, lane = tid & 31, nwarps = (nthreads + 31) >> 5;
  s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
  if (lane == 0) { sm[warp][0] = s0; sm[warp][1] = s1; sm[warp][2] = s2; }
  __syncthreads();
  const unsigned nblocks = gridDim.x * gridDim.y;
  const unsigned bid = blockIdx.x + blockIdx.y * gridDim.x;
  unsigned* counter = reinterpret_cast<unsigned*>(ws);
  double* partials = reinterpret_cast<double*>(reinterpret_cast<char*>(ws) + 64);
  if (tid == 0) {
    double a = 0, b = 0, c = 0;
    for (int w = 0; w < nwarps; ++w) { a += sm[w][0]; b += sm[w][1]; c += sm[w][2]; }
    if (nblocks == 1) {
      tot[0] = a; tot[1] = b; tot[2] = c;
      is_last = true;
    } else {
      partials[bid * 4 + 0] = a; partials[bid * 4 + 1] = b; partials[bid * 4 + 2] = c;
      __threadfence();
      unsigned ticket = atomicAdd(counter, 1u);
      is_last = (ticket == nblocks - 1);
    }
  }
  __syncthreads();
  if (is_last && nblocks > 1) {
    // the last CTA folds the partials with ALL its threads: thread t takes CTAs t, t + nthreads, ... and the
    // per-thread sums are combined warp by warp - a fixed pattern, independent of which CTA arrived last
    // (one thread walking hundreds of partials with dependent fp64 adds was slow in grad_sumsq_kernel)
    __threadfence();
    double x = 0, y = 0, z = 0;
    for (unsigned i = tid; i < nblocks; i += nthreads) {
      x += __ldcg(&partials[i * 4 + 0]); y += __ldcg(&partials[i * 4 + 1]); z += __ldcg(&partials[i * 4 + 2]);
    }
    x = warp_sum(x); y = warp_sum(y); z = warp_sum(z);
    __syncthreads();
    if (lane == 0) { sm[warp][0] = x; sm[warp][1] = y; sm[warp][2] = z; }
    __syncthreads();
    if (tid == 0) {
      double a = 0, b = 0, c = 0;
      for (int w = 0; w < nwarps; ++w) { a += sm[w][0]; b += sm[w][1]; c += sm[w][2]; }
      tot[0] = a; tot[1] = b; tot[2] = c;
      *counter = 0u;
    }
  }
  __syncthreads();
  return is_last && tid == 0;
}

// grid_sum3 for N doubles per thread (partials at stride N): the same summation order per value, so the first three
// totals of grid_sum<5> are bit-identical to grid_sum3's for the same inputs and grid.
template <int N>
__device__ __forceinline__ bool grid_sum(double (&s)[N], void* ws, double* tot) {
  static_assert(N >= 1 && N <= kMaxPartialSums, "grid_sum: partials do not fit the workspace");
  __shared__ double sm[32][N];
  __shared__ bool is_last;
  const int tid = threadIdx.x + threadIdx.y * blockDim.x;
  const int nthreads = blockDim.x * blockDim.y;
  const int warp = tid >> 5, lane = tid & 31, nwarps = (nthreads + 31) >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) s[k] = warp_sum(s[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) sm[warp][k] = s[k];
  }
  __syncthreads();
  const unsigned nblocks = gridDim.x * gridDim.y;
  const unsigned bid = blockIdx.x + blockIdx.y * gridDim.x;
  unsigned* counter = reinterpret_cast<unsigned*>(ws);
  double* partials = reinterpret_cast<double*>(reinterpret_cast<char*>(ws) + 64);
  if (tid == 0) {
    double a[N];
#pragma unroll
    for (int k = 0; k < N; ++k) a[k] = 0;
    for (int w = 0; w < nwarps; ++w) {
#pragma unroll
      for (int k = 0; k < N; ++k) a[k] += sm[w][k];
    }
    if (nblocks == 1) {
#pragma unroll
      for (int k = 0; k < N; ++k) tot[k] = a[k];
      is_last = true;
    } else {
#pragma unroll
      for (int k = 0; k < N; ++k) partials[bid * N + k] = a[k];
      __threadfence();
      unsigned ticket = atomicAdd(counter, 1u);
      is_last = (ticket == nblocks - 1);
    }
  }
  __syncthreads();
  if (is_last && nblocks > 1) {  // fold as grid_sum3 does
    __threadfence();
    double x[N];
#pragma unroll
    for (int k = 0; k < N; ++k) x[k] = 0;
    for (unsigned i = tid; i < nblocks; i += nthreads) {
#pragma unroll
      for (int k = 0; k < N; ++k) x[k] += __ldcg(&partials[i * N + k]);
    }
#pragma unroll
    for (int k = 0; k < N; ++k) x[k] = warp_sum(x[k]);
    __syncthreads();
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < N; ++k) sm[warp][k] = x[k];
    }
    __syncthreads();
    if (tid == 0) {
      double a[N];
#pragma unroll
      for (int k = 0; k < N; ++k) a[k] = 0;
      for (int w = 0; w < nwarps; ++w) {
#pragma unroll
        for (int k = 0; k < N; ++k) a[k] += sm[w][k];
      }
#pragma unroll
      for (int k = 0; k < N; ++k) tot[k] = a[k];
      *counter = 0u;
    }
  }
  __syncthreads();
  return is_last && tid == 0;
}

}  // namespace tb
