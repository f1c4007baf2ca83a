// Data-movement / pointwise kernels of the network path (see net_kernels.cuh).
// All of these are HBM-bound byte/float shuffles: coalesced 128-bit accesses, grid-stride
// loops sized in multiples of the SM count, no tensor cores.
#include "net_kernels.cuh"

#include <cuda_bf16.h>

namespace tb {

static inline unsigned grid_for(int64_t work_items, int threads) {
  int64_t blocks = (work_items + threads - 1) / threads;
  const int64_t cap = int64_t(kNumSMs) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

// ---------------------------------------------------------------------------------------
// uint8 NCHW frames -> uint8 patch matrix.  One thread moves one kernel row (KW bytes).
// ---------------------------------------------------------------------------------------
__global__ void im2col_u8_nchw_kernel(const uint8_t* __restrict__ frame, uint8_t* __restrict__ col, int64_t N, int C,
                                      int H, int W, int KH, int KW, int S, int OH, int OW, int aligned4) {
  const int64_t rows_k = int64_t(C) * KH;               // kernel rows per patch
  const int64_t total = N * OH * OW * rows_k;
  const int64_t K = rows_k * KW;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t row = i / rows_k;
    const int ck = int(i % rows_k);
    const int c = ck / KH, kh = ck % KH;
    const int64_t n = row / (OH * OW);
    const int rem = int(row % (OH * OW));
    const int oy = rem / OW, ox = rem % OW;
    const uint8_t* src = frame + ((n * C + c) * H + (oy * S + kh)) * W + ox * S;
    uint8_t* dst = col + row * K + int64_t(ck) * KW;
    if (aligned4) {
      // 4-byte aligned source (ox*S, W multiples of 4), 8-byte aligned destination
      const uint32_t lo = __ldg(reinterpret_cast<const uint32_t*>(src));
      const uint32_t hi = __ldg(reinterpret_cast<const uint32_t*>(src) + 1);
      *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
    } else {
      for (int kw = 0; kw < KW; ++kw) dst[kw] = __ldg(src + kw);
    }
  }
}

int im2col_u8_nchw(const uint8_t* frame, uint8_t* col, int64_t N, int C, int H, int W, int KH, int KW, int S,
                   cudaStream_t stream) {
  ProfScope prof("im2col_u8", stream);
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  const int64_t total = N * OH * OW * C * KH;
  if (total == 0) return 0;
  const int aligned4 = (KW == 8 && (S & 3) == 0 && (W & 3) == 0 && (reinterpret_cast<uintptr_t>(frame) & 3) == 0 &&
                        (reinterpret_cast<uintptr_t>(col) & 7) == 0);
  im2col_u8_nchw_kernel<<<grid_for(total, 256), 256, 0, stream>>>(frame, col, N, C, H, W, KH, KW, S, OH, OW, aligned4);
  return check_launch("im2col_u8_nchw_kernel");
}

// ---------------------------------------------------------------------------------------
// f32 NHWC activation -> f32 patch matrix, one float4 per thread (C % 4 == 0).
// ---------------------------------------------------------------------------------------
__global__ void im2col_f32_nhwc_kernel(const float4* __restrict__ act, float4* __restrict__ col, int64_t N, int H,
                                       int W, int C4, int KH, int KW, int S, int OH, int OW) {
  const int64_t K4 = int64_t(KH) * KW * C4;
  const int64_t total = N * OH * OW * K4;
  const int rowlen = KW * C4;  // contiguous float4s per kernel row in the source
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t row = i / K4;
    const int k4 = int(i % K4);
    const int kh = k4 / rowlen, r = k4 % rowlen;
    const int64_t n = row / (OH * OW);
    const int rem = int(row % (OH * OW));
    const int oy = rem / OW, ox = rem % OW;
    col[i] = __ldg(act + ((n * H + (oy * S + kh)) * W + ox * S) * C4 + r);
  }
}

int im2col_f32_nhwc(const float* act, float* col, int64_t N, int H, int W, int C, int KH, int KW, int S,
                    cudaStream_t stream) {
  ProfScope prof("im2col_f32", stream);
  TB_REQUIRE(C % 4 == 0, "im2col_f32_nhwc: C must be a multiple of 4");
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  const int64_t total = N * OH * OW * KH * KW * (C / 4);
  if (total == 0) return 0;
  im2col_f32_nhwc_kernel<<<grid_for(total, 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(act), reinterpret_cast<float4*>(col), N, H, W, C / 4, KH, KW, S, OH, OW);
  return check_launch("im2col_f32_nhwc_kernel");
}

// ---------------------------------------------------------------------------------------
// col2im (gather): d_act[n,iy,ix,c] = sum over (kh,kw) with oy*S+kh == iy, ox*S+kw == ix.
// ---------------------------------------------------------------------------------------
__global__ void col2im_f32_nhwc_kernel(const float4* __restrict__ dcol, const float4* __restrict__ act,
                                       float4* __restrict__ dact, int64_t N, int H, int W, int C4, int KH, int KW,
                                       int S, int OH, int OW) {
  const int64_t total = N * H * W * C4;
  const int64_t K4 = int64_t(KH) * KW * C4;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c4 = int(i % C4);
    int64_t t = i / C4;
    const int ix = int(t % W); t /= W;
    const int iy = int(t % H);
    const int64_t n = t / H;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int kh = iy % S; kh < KH; kh += S) {
      const int oy = (iy - kh) / S;
      if (iy - kh < 0) break;
      if (oy >= OH) continue;
      for (int kw = ix % S; kw < KW; kw += S) {
        const int ox = (ix - kw) / S;
        if (ix - kw < 0) break;
        if (ox >= OW) continue;
        const float4 v = __ldg(dcol + ((n * OH + oy) * OW + ox) * K4 + (kh * KW + kw) * C4 + c4);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    }
    if (act) {
      const float4 a = __ldg(act + i);
      s.x = a.x > 0.f ? s.x : 0.f; s.y = a.y > 0.f ? s.y : 0.f;
      s.z = a.z > 0.f ? s.z : 0.f; s.w = a.w > 0.f ? s.w : 0.f;
    }
    dact[i] = s;
  }
}

int col2im_f32_nhwc(const float* dcol, const float* act, float* dact, int64_t N, int H, int W, int C, int KH, int KW,
                    int S, cudaStream_t stream) {
  ProfScope prof("col2im", stream);
  TB_REQUIRE(C % 4 == 0, "col2im_f32_nhwc: C must be a multiple of 4");
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  const int64_t total = N * H * W * (C / 4);
  if (total == 0) return 0;
  col2im_f32_nhwc_kernel<<<grid_for(total, 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(dcol), reinterpret_cast<const float4*>(act), reinterpret_cast<float4*>(dact), N,
      H, W, C / 4, KH, KW, S, OH, OW);
  return check_launch("col2im_f32_nhwc_kernel");
}

// ---------------------------------------------------------------------------------------
__global__ void permute_pq_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t O, int P, int Q) {
  const int64_t total = O * P * Q;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t o = i / (int64_t(P) * Q);
    const int r = int(i % (int64_t(P) * Q));
    const int p = r / Q, q = r % Q;
    out[i] = __ldg(in + o * P * Q + int64_t(q) * P + p);
  }
}

int permute_pq(const float* in, float* out, int64_t O, int P, int Q, cudaStream_t stream) {
  ProfScope prof("weight_pack", stream);
  const int64_t total = O * P * Q;
  if (total == 0) return 0;
  permute_pq_kernel<<<grid_for(total, 256), 256, 0, stream>>>(in, out, O, P, Q);
  return check_launch("permute_pq_kernel");
}

// ---------------------------------------------------------------------------------------
// column sums: block (32 x 8) covers 32 columns x a slab of rows; slabs reduced in a second pass.
// ---------------------------------------------------------------------------------------
constexpr int kColsumSlabs = 256;

int64_t colsum_scratch_floats(int64_t ncols) { return int64_t(kColsumSlabs) * ncols; }

__global__ void colsum_partial_kernel(const float* __restrict__ X, float* __restrict__ part, int64_t M, int64_t ncols,
                                      int64_t ld, int64_t rows_per_slab) {
  __shared__ float sm[8][33];
  const int64_t n = int64_t(blockIdx.x) * 32 + threadIdx.x;
  const int64_t r0 = int64_t(blockIdx.y) * rows_per_slab;
  int64_t r1 = r0 + rows_per_slab;
  if (r1 > M) r1 = M;
  float s = 0.0f;
  if (n < ncols)
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += __ldg(X + r * ld + n);
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && n < ncols) {
    float t = 0.0f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += sm[y][threadIdx.x];
    part[int64_t(blockIdx.y) * ncols + n] = t;
  }
}

// block (32 x 8): 8 partial sums per column (slab s goes to row s % 8), folded in a fixed order.  (The first
// version walked all slabs with one thread per column: 256 dependent L2 round trips per call.)
__global__ void colsum_final_kernel(const float* __restrict__ part, float* __restrict__ out, int64_t ncols, int slabs) {
  __shared__ float sm[8][33];
  const int64_t n = int64_t(blockIdx.x) * 32 + threadIdx.x;
  float t = 0.0f;
  if (n < ncols) {
#pragma unroll 8
    for (int s = threadIdx.y; s < slabs; s += 8) t += __ldg(part + int64_t(s) * ncols + n);
  }
  sm[threadIdx.y][threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.y == 0 && n < ncols) {
    float u = 0.0f;
#pragma unroll
    for (int y = 0; y < 8; ++y) u += sm[y][threadIdx.x];
    out[n] = u;
  }
}

int colsum(const float* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, cudaStream_t stream) {
  ProfScope prof("bias_grad_colsum", stream);
  if (ncols == 0) return 0;
  TB_REQUIRE(X && out && scratch, "colsum: null pointer");
  int slabs = kColsumSlabs;
  if (M < int64_t(slabs) * 64) slabs = int((M + 63) / 64);  // >= 8 rows per thread: fewer, fuller blocks
  if (slabs < 1) slabs = 1;
  const int64_t rows_per_slab = (M + slabs - 1) / slabs;
  dim3 grid((unsigned)((ncols + 31) / 32), (unsigned)slabs);
  colsum_partial_kernel<<<grid, dim3(32, 8), 0, stream>>>(X, scratch, M, ncols, ld, rows_per_slab);
  int rc = check_launch("colsum_partial_kernel");
  if (rc) return rc;
  colsum_final_kernel<<<(unsigned)((ncols + 31) / 32), dim3(32, 8), 0, stream>>>(scratch, out, ncols, slabs);
  return check_launch("colsum_final_kernel");
}

// ---------------------------------------------------------------------------------------
__global__ void core_extras_kernel(float* __restrict__ core, int64_t ld, int64_t N, int F,
                                   const float* __restrict__ reward, const int64_t* __restrict__ last_action, int A) {
  const int64_t total = N * (A + 1);
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / (A + 1);
    const int j = int(i % (A + 1));
    float v;
    if (j == 0) v = fminf(fmaxf(reward[n], -1.0f), 1.0f);
    else v = (last_action[n] == int64_t(j - 1)) ? 1.0f : 0.0f;
    core[n * ld + F + j] = v;
  }
}

int core_extras(float* core, int64_t ld, int64_t N, int F, const float* reward, const int64_t* last_action, int A,
                cudaStream_t stream) {
  ProfScope prof("core_extras", stream);
  if (N == 0) return 0;
  // A == 0: reward column only (polybeast Net has no last-action one-hot)
  core_extras_kernel<<<grid_for(N * (A + 1), 256), 256, 0, stream>>>(core, ld, N, F, reward, last_action, A);
  return check_launch("core_extras_kernel");
}

__global__ void relu_mask_kernel(float* __restrict__ X, const float* __restrict__ Y, int64_t M, int64_t ncols,
                                 int64_t ldx, int64_t ldy) {
  const int64_t total = M * ncols;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t m = i / ncols, n = i % ncols;
    if (!(Y[m * ldy + n] > 0.0f)) X[m * ldx + n] = 0.0f;
  }
}

int relu_mask_inplace(float* X, const float* Y, int64_t M, int64_t ncols, int64_t ldx, int64_t ldy,
                      cudaStream_t stream) {
  ProfScope prof("relu_mask", stream);
  if (M * ncols == 0) return 0;
  relu_mask_kernel<<<grid_for(M * ncols, 256), 256, 0, stream>>>(X, Y, M, ncols, ldx, ldy);
  return check_launch("relu_mask_kernel");
}


// =========================================================================================
// bf16 operand staging (tensor-core backend)
// =========================================================================================
__device__ __forceinline__ void acc_bf16x8(const uint4& v, float (&s)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __bfloat1622float2(h[j]);
    s[2 * j] += f.x; s[2 * j + 1] += f.y;
  }
}

__global__ void pack_weights_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t O, int P,
                                         int Q, int64_t ld, int64_t lo_off) {
  const int64_t total = O * ld;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t o = i / ld;
    const int64_t r = i % ld;
    float v = 0.0f;
    if (r < int64_t(P) * Q) {
      const int pp = int(r / Q), q = int(r % Q);
      v = __ldg(in + o * P * Q + int64_t(q) * P + pp);
    }
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    out[i] = h;
    if (lo_off) out[lo_off + i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

int pack_weights_bf16(const float* in, void* out, int64_t O, int P, int Q, int64_t ld_out, cudaStream_t stream, int64_t lo_off) {
  ProfScope prof("weight_pack_bf16", stream);
  const int64_t total = O * ld_out;
  if (total == 0) return 0;
  pack_weights_bf16_kernel<<<grid_for(total, 256), 256, 0, stream>>>(in, static_cast<__nv_bfloat16*>(out), O, P, Q, ld_out, lo_off);
  return check_launch("pack_weights_bf16_kernel");
}

// weights [O, C, KH, KW] (fp32, reference layout) -> B operand of the implicit input-gradient GEMMs (bf16):
//   stride 1: out[c][(kh*KW + kw)*O + o]
//   stride 2: out[((py*2 + px)*C + c)][((i*(KW/2) + j)*O + o]  with kh = py + 2i, kw = px + 2j
__global__ void pack_dgrad_weights_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int O, int C,
                                               int KH, int KW, int S, int64_t lo_off) {
  const int64_t total = int64_t(O) * C * KH * KW;
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int kw = int(idx % KW), kh = int((idx / KW) % KH), c = int((idx / (int64_t(KW) * KH)) % C), o = int(idx / (int64_t(KW) * KH * C));
  const float v = in[idx];
  int64_t dst;
  if (S == 1) {
    dst = int64_t(c) * (KH * KW * O) + int64_t(kh * KW + kw) * O + o;
  } else {
    const int py = kh & 1, i = kh >> 1, px = kw & 1, j = kw >> 1;
    dst = (int64_t((py * 2 + px) * C + c)) * ((KH / 2) * (KW / 2) * O) + int64_t(i * (KW / 2) + j) * O + o;
  }
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  out[dst] = h;
  if (lo_off) out[lo_off + dst] = __float2bfloat16_rn(v - __bfloat162float(h));
}

int pack_dgrad_weights_bf16(const float* in, void* out_bf16, int O, int C, int KH, int KW, int S, cudaStream_t stream,
                            int64_t lo_off) {
  TB_REQUIRE(in && out_bf16 && (S == 1 || (S == 2 && KH % 2 == 0 && KW % 2 == 0)), "pack_dgrad_weights_bf16: bad arguments");
  ProfScope prof("weight_pack_bf16", stream);
  const int64_t total = int64_t(O) * C * KH * KW;
  pack_dgrad_weights_bf16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, static_cast<__nv_bfloat16*>(out_bf16), O,
                                                                                     C, KH, KW, S, lo_off);
  return check_launch("pack_dgrad_weights_bf16_kernel");
}

__global__ void colsum_partial_bf16_kernel(const __nv_bfloat16* __restrict__ X, float* __restrict__ part, int64_t M,
                                           int64_t ncols, int64_t ld, int64_t rows_per_slab, int64_t lo_off) {
  __shared__ float sm[8][33];
  const int64_t n = int64_t(blockIdx.x) * 32 + threadIdx.x;
  const int64_t r0 = int64_t(blockIdx.y) * rows_per_slab;
  int64_t r1 = r0 + rows_per_slab;
  if (r1 > M) r1 = M;
  float s = 0.0f;
  if (n < ncols)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      s += __bfloat162float(X[r * ld + n]);
      if (lo_off) s += __bfloat162float(X[lo_off + r * ld + n]);
    }
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && n < ncols) {
    float t = 0.0f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += sm[y][threadIdx.x];
    part[int64_t(blockIdx.y) * ncols + n] = t;
  }
}

// Dense [M, ncols] bf16 with ncols in {8,16,32,64}: every thread streams 16-byte vectors whose column
// group never changes (the grid stride is a multiple of the row length), so the kernel is a plain
// coalesced read of the whole matrix followed by a small shared-memory fold.
__global__ void colsum_dense_bf16_kernel(const uint4* __restrict__ X, float* __restrict__ part, int64_t nvec, int cg,
                                         int64_t lo_vec) {
  __shared__ float sm[256][9];
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;  // multiple of cg (cg | 256)
#pragma unroll 4
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    acc_bf16x8(__ldg(X + i), s);
    if (lo_vec) acc_bf16x8(__ldg(X + lo_vec + i), s);  // split-bf16 gradient: hi + lo planes
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[threadIdx.x][j] = s[j];
  __syncthreads();
  if (threadIdx.x < cg * 8) {
    const int g = threadIdx.x / 8, j = threadIdx.x % 8;
    float t = 0.f;
    for (int k = g; k < 256; k += cg) t += sm[k][j];
    part[int64_t(blockIdx.x) * cg * 8 + g * 8 + j] = t;
  }
}

int colsum_bf16(const void* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, cudaStream_t stream,
                int64_t lo_off) {
  ProfScope prof("bias_grad_colsum", stream);
  if (ncols == 0) return 0;
  TB_REQUIRE(X && out && scratch, "colsum_bf16: null pointer");
  if (ld == ncols && (ncols == 8 || ncols == 16 || ncols == 32 || ncols == 64) && M >= 4096 &&
      (reinterpret_cast<uintptr_t>(X) & 15) == 0 && (lo_off & 7) == 0) {
    const int cg = int(ncols / 8);
    // partials [blocks][ncols] must fit the caller's scratch (colsum_scratch_floats(>= 512) = 256 * 512 floats): 6 CTAs per SM
    // keep enough 16-byte loads in flight to stream at HBM rate
    int blocks = kNumSMs * 6;
    if (int64_t(blocks) * ncols > int64_t(kColsumSlabs) * 512) blocks = int(int64_t(kColsumSlabs) * 512 / ncols);
    colsum_dense_bf16_kernel<<<blocks, 256, 0, stream>>>(static_cast<const uint4*>(X), scratch, M * cg, cg, lo_off / 8);
    int rc = check_launch("colsum_dense_bf16_kernel");
    if (rc) return rc;
    colsum_final_kernel<<<(unsigned)((ncols + 31) / 32), dim3(32, 8), 0, stream>>>(scratch, out, ncols, blocks);
    return check_launch("colsum_final_kernel");
  }
  int slabs = kColsumSlabs;
  if (M < int64_t(slabs) * 64) slabs = int((M + 63) / 64);
  if (slabs < 1) slabs = 1;
  const int64_t rows_per_slab = (M + slabs - 1) / slabs;
  dim3 grid((unsigned)((ncols + 31) / 32), (unsigned)slabs);
  colsum_partial_bf16_kernel<<<grid, dim3(32, 8), 0, stream>>>(static_cast<const __nv_bfloat16*>(X), scratch, M, ncols, ld,
                                                                rows_per_slab, lo_off);
  int rc = check_launch("colsum_partial_bf16_kernel");
  if (rc) return rc;
  colsum_final_kernel<<<(unsigned)((ncols + 31) / 32), dim3(32, 8), 0, stream>>>(scratch, out, ncols, slabs);
  return check_launch("colsum_final_kernel");
}

}  // namespace tb
