// Fused policy / baseline heads: see heads.cuh.
#include "heads.cuh"

namespace tb {

namespace {

constexpr int kMaxOut = 32;   // A + 1 outputs at most
constexpr int kSlabRows = 64; // rows per partial block of the weight-gradient reduction

// Block = 8 warps x kFwdRowsPerWarp rows each; the (A+1) x F weight matrix is staged once per block in shared memory
// (the first version re-read it through L1 for every row).  Lanes stride over F; 8 accumulators per pass.
constexpr int kFwdRowsPerWarp = 2;  // 16 rows per block: ~160 blocks at N = 2592
__global__ void heads_fwd_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ Wp,
                                 const float* __restrict__ bp, const float* __restrict__ Wb, const float* __restrict__ bb,
                                 int64_t N, int F, int A, float* __restrict__ logits, float* __restrict__ baseline) {
  extern __shared__ float wsm[];  // [(A+1)][F]
  const int O = A + 1;
  for (int i = threadIdx.x; i < O * F; i += blockDim.x) {
    const int o = i / F, f = i - o * F;
    wsm[i] = (o < A) ? __ldg(Wp + int64_t(o) * F + f) : __ldg(Wb + f);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  const int64_t row0 = (int64_t(blockIdx.x) * (blockDim.x >> 5) + wrp) * kFwdRowsPerWarp;
  for (int rr = 0; rr < kFwdRowsPerWarp; ++rr) {
    const int64_t n = row0 + rr;
    if (n >= N) return;
    const float* xr = x + n * ldx;
    for (int o0 = 0; o0 < O; o0 += 8) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int f = lane; f < F; f += 32) {
        const float xv = __ldg(xr + f);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (o0 + j < O) acc[j] = fmaf(xv, wsm[(o0 + j) * F + f], acc[j]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int o = o0 + j;
        if (o >= O) break;
        const float s = warp_sum(acc[j]);
        if (lane == 0) {
          if (o < A) logits[n * A + o] = s + __ldg(bp + o);
          else baseline[n] = s + __ldg(bb);
        }
      }
    }
  }
}

// thread per (row, feature)
__global__ void heads_dgrad_kernel(const float* __restrict__ Wp, const float* __restrict__ Wb, const float* __restrict__ dl,
                                   const float* __restrict__ db, int64_t N, int F, int A, float* __restrict__ dx, int64_t lddx) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n = blockIdx.y;
  if (f >= F) return;
  float s = __ldg(db + n) * __ldg(Wb + f);
  for (int a = 0; a < A; ++a) s = fmaf(__ldg(dl + n * A + a), __ldg(Wp + int64_t(a) * F + f), s);
  dx[n * lddx + f] = s;
}

// block (32 x 8): 32 feature columns (column F is the implicit ones column -> bias gradients) x a slab of rows;
// partial [slab][A+1][F+1]
__global__ void heads_wgrad_partial_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ dl,
                                           const float* __restrict__ db, int64_t N, int F, int A, float* __restrict__ part) {
  __shared__ float sm[8][33];
  const int f = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = int64_t(blockIdx.y) * kSlabRows;
  const int64_t r1 = (r0 + kSlabRows < N) ? r0 + kSlabRows : N;
  const int O = A + 1, F1 = F + 1;
  for (int o0 = 0; o0 < O; o0 += 8) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (f < F1) {
      for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
        const float xv = (f < F) ? __ldg(x + r * ldx + f) : 1.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int o = o0 + j;
          if (o < A) acc[j] = fmaf(__ldg(dl + r * A + o), xv, acc[j]);
          else if (o == A) acc[j] = fmaf(__ldg(db + r), xv, acc[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      __syncthreads();
      sm[threadIdx.y][threadIdx.x] = acc[j];
      __syncthreads();
      const int o = o0 + j;
      if (threadIdx.y == 0 && f < F1 && o < O) {
        float t = 0.f;
#pragma unroll
        for (int y = 0; y < 8; ++y) t += sm[y][threadIdx.x];
        part[(int64_t(blockIdx.y) * O + o) * F1 + f] = t;
      }
    }
  }
}

// fold the slabs in a fixed order and route each entry to its destination
__global__ void heads_wgrad_final_kernel(const float* __restrict__ part, int slabs, int F, int A, float* __restrict__ dWp,
                                         float* __restrict__ dbp, float* __restrict__ dWb, float* __restrict__ dbb) {
  __shared__ float sm[8][33];
  const int O = A + 1, F1 = F + 1;
  const int idx = blockIdx.x * 32 + threadIdx.x;
  const int total = O * F1;
  float t = 0.f;
  if (idx < total) {
#pragma unroll 4
    for (int s = threadIdx.y; s < slabs; s += 8) t += __ldg(part + int64_t(s) * total + idx);
  }
  sm[threadIdx.y][threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.y == 0 && idx < total) {
    float u = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) u += sm[y][threadIdx.x];
    const int o = idx / F1, f = idx - o * F1;
    if (o < A) { if (f < F) dWp[int64_t(o) * F + f] = u; else dbp[o] = u; }
    else       { if (f < F) dWb[f] = u; else dbb[0] = u; }
  }
}

}  // namespace

int heads_forward(const float* x, int64_t ldx, const float* Wp, const float* bp, const float* Wb, const float* bb, int64_t N, int F,
                  int A, float* logits, float* baseline, cudaStream_t stream) {
  TB_REQUIRE(x && Wp && bp && Wb && bb && logits && baseline, "heads_forward: null pointer");
  TB_REQUIRE(A >= 1 && A < kMaxOut && F >= 1, "heads_forward: bad sizes");
  if (N == 0) return 0;
  ProfScope prof("heads_fwd", stream);
  const size_t smem = sizeof(float) * size_t(A + 1) * F;
  TB_REQUIRE(smem <= 48 * 1024, "heads_forward: (A+1)*F too large for the shared-memory weight stage");
  const int64_t rows_per_block = 8 * kFwdRowsPerWarp;
  heads_fwd_kernel<<<(unsigned)((N + rows_per_block - 1) / rows_per_block), 256, smem, stream>>>(x, ldx, Wp, bp, Wb, bb, N, F, A,
                                                                                                logits, baseline);
  return check_launch("heads_fwd_kernel");
}

int64_t heads_scratch_floats(int64_t N, int F, int A) {
  return ((N + kSlabRows - 1) / kSlabRows) * int64_t(A + 1) * (F + 1);
}

int heads_backward(const float* x, int64_t ldx, const float* Wp, const float* Wb, const float* dlogits, const float* dbaseline,
                   int64_t N, int F, int A, float* dx, int64_t lddx, float* dWp, float* dbp, float* dWb, float* dbb, float* scratch,
                   cudaStream_t stream) {
  TB_REQUIRE(x && Wp && Wb && dlogits && dbaseline && dx && dWp && dbp && dWb && dbb && scratch, "heads_backward: null pointer");
  TB_REQUIRE(A >= 1 && A < kMaxOut && F >= 1 && N >= 1 && N < 65536 * int64_t(kSlabRows), "heads_backward: bad sizes");
  ProfScope prof("heads_bwd", stream);
  heads_dgrad_kernel<<<dim3((unsigned)((F + 127) / 128), (unsigned)N), 128, 0, stream>>>(Wp, Wb, dlogits, dbaseline, N, F, A, dx, lddx);
  int rc = check_launch("heads_dgrad_kernel");
  if (rc) return rc;
  const int slabs = int((N + kSlabRows - 1) / kSlabRows);
  heads_wgrad_partial_kernel<<<dim3((unsigned)((F + 1 + 31) / 32), (unsigned)slabs), dim3(32, 8), 0, stream>>>(
      x, ldx, dlogits, dbaseline, N, F, A, scratch);
  rc = check_launch("heads_wgrad_partial_kernel");
  if (rc) return rc;
  const int total = (A + 1) * (F + 1);
  heads_wgrad_final_kernel<<<(unsigned)((total + 31) / 32), dim3(32, 8), 0, stream>>>(scratch, slabs, F, A, dWp, dbp, dWb, dbb);
  return check_launch("heads_wgrad_final_kernel");
}

}  // namespace tb
