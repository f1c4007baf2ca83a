// Fused policy / baseline heads: see heads.cuh.
#include "heads.cuh"

namespace tb {

namespace {

constexpr int kMaxOut = 32;   // A < kMaxOut actions
constexpr int kSlabRows = 64; // rows per partial block of the weight-gradient reduction, up to kHeadsMaxSlabs blocks
constexpr int kFwdSmemFloats = 48 * 1024 / 4;  // the forward's weight stage

// Block = 8 warps x kFwdRowsPerWarp rows each; the (A+V) x F weight matrix is staged in shared memory (the first version
// re-read it through L1 for every row), in tiles of `tile` outputs when it does not fit at once (e.g. A = 18, V = 64,
// F = 519).  Lanes stride over F; 8 accumulators per pass.  Each output's sum is formed in the same order whatever the
// tiling, so V = 1 (one tile) gives the single-baseline results.
constexpr int kFwdRowsPerWarp = 2;  // 16 rows per block: ~160 blocks at N = 2592
__global__ void heads_fwd_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ Wp,
                                 const float* __restrict__ bp, const float* __restrict__ Wb, const float* __restrict__ bb,
                                 int64_t N, int F, int A, int V, int tile, float* __restrict__ logits,
                                 float* __restrict__ baseline) {
  extern __shared__ float wsm[];  // [tile][F]
  const int O = A + V;
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  const int64_t row0 = (int64_t(blockIdx.x) * (blockDim.x >> 5) + wrp) * kFwdRowsPerWarp;
  for (int ot = 0; ot < O; ot += tile) {
    const int ot1 = (ot + tile < O) ? ot + tile : O;
    if (ot > 0) __syncthreads();  // the previous tile's reads are done
    for (int i = threadIdx.x; i < (ot1 - ot) * F; i += blockDim.x) {
      const int oi = i / F, f = i - oi * F, o = ot + oi;
      wsm[i] = (o < A) ? __ldg(Wp + int64_t(o) * F + f) : __ldg(Wb + int64_t(o - A) * F + f);
    }
    __syncthreads();
    for (int rr = 0; rr < kFwdRowsPerWarp; ++rr) {
      const int64_t n = row0 + rr;
      if (n >= N) break;
      const float* xr = x + n * ldx;
      for (int o0 = ot; o0 < ot1; o0 += 8) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int f = lane; f < F; f += 32) {
          const float xv = __ldg(xr + f);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (o0 + j < ot1) acc[j] = fmaf(xv, wsm[(o0 + j - ot) * F + f], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int o = o0 + j;
          if (o >= ot1) break;
          const float s = warp_sum(acc[j]);
          if (lane == 0) {
            if (o < A) logits[n * A + o] = s + __ldg(bp + o);
            else baseline[n * V + (o - A)] = s + __ldg(bb + (o - A));
          }
        }
      }
    }
  }
}

// thread per (row, feature); rows on grid.x, which has no 65535 limit
__global__ void heads_dgrad_kernel(const float* __restrict__ Wp, const float* __restrict__ Wb, const float* __restrict__ dl,
                                   const float* __restrict__ db, int64_t N, int F, int A, int V, float* __restrict__ dx,
                                   int64_t lddx) {
  const int f = blockIdx.y * blockDim.x + threadIdx.x;
  const int64_t n = blockIdx.x;
  if (f >= F) return;
  float s = __ldg(db + n * V) * __ldg(Wb + f);
  for (int v = 1; v < V; ++v) s = fmaf(__ldg(db + n * V + v), __ldg(Wb + int64_t(v) * F + f), s);
  for (int a = 0; a < A; ++a) s = fmaf(__ldg(dl + n * A + a), __ldg(Wp + int64_t(a) * F + f), s);
  dx[n * lddx + f] = s;
}

// block (32 x 8): 32 feature columns (column F is the implicit ones column -> bias gradients) x a slab of rows;
// partial [slab][A+V][F+1].  kLong: slabs of `long_rows` rows (N > 64 * kHeadsMaxSlabs), else of kSlabRows, a
// compile-time bound the short form's loop is scheduled around.
template <bool kLong>
__global__ void heads_wgrad_partial_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ dl,
                                           const float* __restrict__ db, int64_t N, int F, int A, int V, int64_t long_rows,
                                           float* __restrict__ part) {
  __shared__ float sm[8][33];
  const int64_t rows = kLong ? long_rows : kSlabRows;
  const int f = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = int64_t(blockIdx.y) * rows;
  const int64_t r1 = (r0 + rows < N) ? r0 + rows : N;
  const int O = A + V, F1 = F + 1;
  for (int o0 = 0; o0 < O; o0 += 8) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (f < F1) {
      for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
        const float xv = (f < F) ? __ldg(x + r * ldx + f) : 1.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int o = o0 + j;
          if (o < A) acc[j] = fmaf(__ldg(dl + r * A + o), xv, acc[j]);
          else if (o < O) acc[j] = fmaf(__ldg(db + r * V + (o - A)), xv, acc[j]);
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
__global__ void heads_wgrad_final_kernel(const float* __restrict__ part, int slabs, int F, int A, int V,
                                         float* __restrict__ dWp, float* __restrict__ dbp, float* __restrict__ dWb,
                                         float* __restrict__ dbb) {
  __shared__ float sm[8][33];
  const int O = A + V, F1 = F + 1;
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
    else       { if (f < F) dWb[int64_t(o - A) * F + f] = u; else dbb[o - A] = u; }
  }
}

}  // namespace

int heads_forward(const float* x, int64_t ldx, const float* Wp, const float* bp, const float* Wb, const float* bb, int64_t N, int F,
                  int A, float* logits, float* baseline, cudaStream_t stream, int V) {
  TB_REQUIRE(x && Wp && bp && Wb && bb && logits && baseline, "heads_forward: null pointer");
  TB_REQUIRE(A >= 1 && A < kMaxOut && V >= 1 && V <= kHeadsMaxValues && F >= 1 && F <= kFwdSmemFloats,
             "heads_forward: bad sizes A=%d V=%d F=%d", A, V, F);
  if (N == 0) return 0;
  ProfScope prof("heads_fwd", stream);
  const int fit = kFwdSmemFloats / F;
  const int tile = (A + V < fit) ? A + V : fit;
  const size_t smem = sizeof(float) * size_t(tile) * F;
  const int64_t rows_per_block = 8 * kFwdRowsPerWarp;
  heads_fwd_kernel<<<(unsigned)((N + rows_per_block - 1) / rows_per_block), 256, smem, stream>>>(x, ldx, Wp, bp, Wb, bb, N, F, A,
                                                                                                V, tile, logits, baseline);
  return check_launch("heads_fwd_kernel");
}

// Rows per slab: kSlabRows while that takes at most kHeadsMaxSlabs slabs (the bits of every N <= 64 * kHeadsMaxSlabs do
// not depend on the cap), else the fewest rows that keep the slab count at the cap.
static int64_t heads_slab_rows(int64_t N) {
  const int64_t slabs = (N + kSlabRows - 1) / kSlabRows;
  return slabs <= kHeadsMaxSlabs ? kSlabRows : (N + kHeadsMaxSlabs - 1) / kHeadsMaxSlabs;
}

static int64_t heads_slabs(int64_t N) {
  const int64_t rows = heads_slab_rows(N);
  return (N + rows - 1) / rows;
}

int64_t heads_scratch_floats(int64_t N, int F, int A, int V) {
  return (N > 0 ? heads_slabs(N) : 0) * int64_t(A + V) * (F + 1);
}

int heads_backward(const float* x, int64_t ldx, const float* Wp, const float* Wb, const float* dlogits, const float* dbaseline,
                   int64_t N, int F, int A, float* dx, int64_t lddx, float* dWp, float* dbp, float* dWb, float* dbb, float* scratch,
                   cudaStream_t stream, int V) {
  TB_REQUIRE(x && Wp && Wb && dlogits && dbaseline && dx && dWp && dbp && dWb && dbb && scratch, "heads_backward: null pointer");
  TB_REQUIRE(A >= 1 && A < kMaxOut && V >= 1 && V <= kHeadsMaxValues && F >= 1 && F <= 65535 * 128 && N >= 1 &&
             N < (int64_t(1) << 31), "heads_backward: bad sizes A=%d V=%d F=%d N=%lld", A, V, F, (long long)N);
  ProfScope prof("heads_bwd", stream);
  heads_dgrad_kernel<<<dim3((unsigned)N, (unsigned)((F + 127) / 128)), 128, 0, stream>>>(Wp, Wb, dlogits, dbaseline, N, F, A, V,
                                                                                         dx, lddx);
  int rc = check_launch("heads_dgrad_kernel");
  if (rc) return rc;
  const int slabs = int(heads_slabs(N));
  const int64_t rows = heads_slab_rows(N);
  const dim3 grid((unsigned)((F + 1 + 31) / 32), (unsigned)slabs);
  if (rows == kSlabRows)
    heads_wgrad_partial_kernel<false><<<grid, dim3(32, 8), 0, stream>>>(x, ldx, dlogits, dbaseline, N, F, A, V, rows, scratch);
  else
    heads_wgrad_partial_kernel<true><<<grid, dim3(32, 8), 0, stream>>>(x, ldx, dlogits, dbaseline, N, F, A, V, rows, scratch);
  rc = check_launch("heads_wgrad_partial_kernel");
  if (rc) return rc;
  const int total = (A + V) * (F + 1);
  heads_wgrad_final_kernel<<<(unsigned)((total + 31) / 32), dim3(32, 8), 0, stream>>>(scratch, slabs, F, A, V, dWp, dbp, dWb,
                                                                                      dbb);
  return check_launch("heads_wgrad_final_kernel");
}

}  // namespace tb
