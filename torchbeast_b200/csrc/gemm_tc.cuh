// bf16 wgmma GEMM (see gemm_tc.cu): host interface.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace tb {

struct TcEpilogue {
  float* C = nullptr; int64_t ldc = 0;               // fp32 output (nullable)
  __nv_bfloat16* C16 = nullptr; int64_t ldc16 = 0;   // bf16 output (nullable) - next GEMM's operand
  // Split-bf16 ("bf16x3") mode: every operand x is stored as TWO bf16 planes, hi = bf16(x) and lo = bf16(x - hi)
  // (16-17 significant bits together), and the product is accumulated as hi.hi + hi.lo + lo.hi in the same fp32
  // fp32 accumulator - fp32-grade results (relative error ~2^-17 per product instead of 2^-9) at 3 MMAs per k-step.
  // a_lo / b_lo: element offsets from the operand base pointers to their lo planes (both non-zero = split product,
  // both zero = plain bf16); c16_lo: element offset from C16 to the lo plane of the bf16 output (0 = hi only).
  int64_t a_lo = 0, b_lo = 0, c16_lo = 0;
  const float* bias = nullptr;                       // [N]
  float scale = 1.0f;                                // applied to the accumulator first (1/255 for uint8 frames)
  int relu = 0;
  const float* mask = nullptr; int64_t ldmask = 0;   // out = (mask > 0) ? out : 0   (ReLU backward)
  const __nv_bfloat16* mask16 = nullptr;             // same, mask stored in bf16 (uses ldmask)
  const __nv_bfloat16* addend16 = nullptr; int64_t ldadd = 0;  // out += addend (residual connection), applied last
  const float* addend32 = nullptr;                   // same, residual stored in fp32 (uses ldadd)
  int permP = 1, permQ = 1;                          // (split-K reduce only) weight-grad column un-pack
  int max_ctas = 0;                                  // > 0: cap the persistent grid (GEMMs running beside a cooperative kernel)
  const char* tag = "gemm_tc";
};

// C[M,N] = epilogue(A[M,K] . B[N,K]^T); A, B bf16 with K contiguous, lda/ldb multiples of 8,
// 16-byte aligned bases.
int gemm_tc_bf16(const void* A, const void* B, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                 const TcEpilogue& ep, cudaStream_t stream);

// General form: a_mn / b_mn mark operands whose ROW index is the reduction index
//   (a_mn: A is [K, M] row-major; b_mn: B is [K, N] row-major).  splits > 1 (or partial != nullptr)
//   writes raw fp32 partial tiles [z][M][N] to `partial` for splitk_reduce_kernel.
int gemm_tc_bf16_ex(const void* A, const void* B, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, bool a_mn,
                    bool b_mn, const TcEpilogue& ep, int splits, float* partial, cudaStream_t stream);

// Implicit-GEMM convolution forward over a bf16 NHWC activation [Nf, H, W, C] (no patch matrix): out[Nf*OH*OW, O] =
// epilogue(patches . Wp^T) with Wp [O, KH*KW*C] packed (kh, kw, c).  The activation is read through a rank-4
// tensor map with overlapping dimensions.  Requires conv_tc_implicit_applicable().
bool conv_tc_implicit_applicable(int H, int W, int C, int KH, int KW, int S, int O);
int conv_tc_fwd_implicit(const void* act_nhwc_bf16, const void* w_packed_bf16, int64_t Nf, int H, int W, int C, int KH, int KW,
                         int S, int O, const TcEpilogue& ep, cudaStream_t stream);

// Input gradient of the same convolution as a gather-form transposed convolution (no gradient patch matrix, no
// col2im): dX (ep.C16, bf16 NHWC [Nf,H,W,C], times the ReLU mask ep.mask16) from dY [Nf,OH,OW,64].  Stride 1, or
// stride 2 with a 4x4 kernel (output pixels split into 4 parity classes that share the dY boxes).  wt_bf16 comes
// from pack_dgrad_weights_bf16 (net_kernels.cuh).
bool conv_tc_dgrad_implicit_applicable(int H, int W, int C, int KH, int KW, int S, int O);
int conv_tc_dgrad_implicit(const void* dy_nhwc_bf16, const void* wt_bf16, int64_t Nf, int H, int W, int C, int KH, int KW, int S,
                           int O, const TcEpilogue& ep, cudaStream_t stream);

// Weight gradient of the same convolution, patches again read through TMA: dW (fp32, [O, KH*KW*C] un-packed by
// permP/permQ like the split-K reduce of gemm_tc_bf16_ex) = scale * dY^T . patches; dy_bf16 [Nf*OH*OW, O], O <= 64.
int conv_tc_wgrad_implicit(const void* dy_bf16, const void* act_nhwc_bf16, int64_t Nf, int H, int W, int C, int KH, int KW, int S,
                           int O, float* dW, int permP, int permQ, float scale, float* partial, int64_t partial_floats,
                           const char* tag, cudaStream_t stream, int64_t dy_lo = 0, int64_t act_lo = 0);

// lo_off != 0: also write the lo plane bf16(x - hi) at out + lo_off elements (split-bf16 operands)
int f32_to_bf16(const float* in, void* out, int64_t rows, int64_t cols, int64_t ld, int64_t ld16, cudaStream_t stream,
                int64_t lo_off = 0);

}  // namespace tb
