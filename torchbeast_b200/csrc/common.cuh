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

constexpr int kWarp = 32;
constexpr int kNumSMs = 132;  // H100 SXM
// workspace layout: [0] uint32 ticket counter (self-resetting), then kMaxPartialCtas x 4 doubles
constexpr int kMaxPartialCtas = 4096;
constexpr size_t kWorkspaceBytes = 64 + size_t(kMaxPartialCtas) * 4 * sizeof(double);

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

}  // namespace tb
