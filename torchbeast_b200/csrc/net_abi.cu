// C ABI of the fp32 network building blocks (SIMT GEMM, patch-matrix and pointwise kernels, fused heads, bias-gradient
// column sums) so that they can be tested in isolation against float64 references; the learner calls the same internals
// from atarinet.cu, resnet.cu and lstm.cu.  See include/torchbeast_b200.h.
#include <cuda_bf16.h>

#include "gemm_simt.cuh"
#include "heads.cuh"
#include "lstm.cuh"
#include "net_kernels.cuh"
#include "resnet_kernels.cuh"

using namespace tb;

// dtype 0 = fp32, 1 = bf16: call F<float> or F<__nv_bfloat16> on the same void pointers
#define TB_BY_DTYPE(name, dtype, call_f32, call_bf16)                \
  do {                                                              \
    TB_REQUIRE((dtype) == 0 || (dtype) == 1, name ": dtype must be 0 (f32) or 1 (bf16)"); \
    return (dtype) ? (call_bf16) : (call_f32);                      \
  } while (0)

using bf16 = __nv_bfloat16;

extern "C" {

int tb_gemm_f32(const void* A, int a_u8, const void* B, int b_u8, int ta, int tb, int64_t M, int64_t N, int64_t K, int64_t lda,
                int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, const float* mask, int64_t ldmask,
                const float* addend, int64_t ldadd, int accumulate, int permP, int permQ, float scale, int splits, float* scratch,
                void* stream) {
  GemmEpilogue ep;
  ep.bias = bias; ep.relu = relu; ep.mask = mask; ep.ldmask = ldmask; ep.accumulate = accumulate; ep.addend = addend;
  ep.ldadd = ldadd; ep.permP = permP; ep.permQ = permQ; ep.scale = scale; ep.tag = "gemm_f32";
  TB_REQUIRE(permP >= 1 && permQ >= 1 && (permP * permQ == 1 || int64_t(permP) * permQ == N),
             "tb_gemm_f32: the column permutation must cover N = permP * permQ");
  cudaStream_t st = (cudaStream_t)stream;
  const float* Af = static_cast<const float*>(A);
  const float* Bf = static_cast<const float*>(B);
  // the five instantiations the learner uses
  if (!a_u8 && !b_u8 && !ta && tb)
    return gemm_simt<float, float, false, true>(Af, Bf, C, M, N, K, lda, ldb, ldc, ep, splits, scratch, st);
  if (a_u8 && !b_u8 && !ta && tb)
    return gemm_simt<uint8_t, float, false, true>(static_cast<const uint8_t*>(A), Bf, C, M, N, K, lda, ldb, ldc, ep, splits,
                                                  scratch, st);
  if (!a_u8 && !b_u8 && !ta && !tb)
    return gemm_simt<float, float, false, false>(Af, Bf, C, M, N, K, lda, ldb, ldc, ep, splits, scratch, st);
  if (!a_u8 && !b_u8 && ta && !tb)
    return gemm_simt<float, float, true, false>(Af, Bf, C, M, N, K, lda, ldb, ldc, ep, splits, scratch, st);
  if (!a_u8 && b_u8 && ta && !tb)
    return gemm_simt<float, uint8_t, true, false>(Af, static_cast<const uint8_t*>(B), C, M, N, K, lda, ldb, ldc, ep, splits,
                                                  scratch, st);
  set_error("tb_gemm_f32: no kernel for a_u8=%d b_u8=%d ta=%d tb=%d", a_u8, b_u8, ta, tb);
  return 1;
}

int tb_gemm_f32_splits(int64_t M, int64_t N, int64_t K, int64_t scratch_floats, int64_t cap) {
  return simt_splits(M, N, K, scratch_floats, cap);
}

int64_t tb_splitk_scratch_floats(void) { return kSplitKScratchFloats; }

int tb_im2col_u8_nchw(const uint8_t* frame, uint8_t* col, int64_t N, int C, int H, int W, int KH, int KW, int S, void* stream) {
  TB_REQUIRE(frame && col, "tb_im2col_u8_nchw: null pointer");
  return im2col_u8_nchw(frame, col, N, C, H, W, KH, KW, S, (cudaStream_t)stream);
}

int tb_im2col_f32_nhwc(const float* act, float* col, int64_t N, int H, int W, int C, int KH, int KW, int S, void* stream) {
  TB_REQUIRE(act && col, "tb_im2col_f32_nhwc: null pointer");
  return im2col_f32_nhwc(act, col, N, H, W, C, KH, KW, S, (cudaStream_t)stream);
}

int tb_col2im_f32_nhwc(const float* dcol, const float* act, float* dact, int64_t N, int H, int W, int C, int KH, int KW, int S,
                       void* stream) {
  TB_REQUIRE(dcol && dact, "tb_col2im_f32_nhwc: null pointer");
  return col2im_f32_nhwc(dcol, act, dact, N, H, W, C, KH, KW, S, (cudaStream_t)stream);
}

int tb_permute_pq(const float* in, float* out, int64_t O, int P, int Q, void* stream) {
  TB_REQUIRE(in && out, "tb_permute_pq: null pointer");
  return permute_pq(in, out, O, P, Q, (cudaStream_t)stream);
}

int tb_relu_mask_f32(float* X, const float* Y, int64_t M, int64_t ncols, int64_t ldx, int64_t ldy, void* stream) {
  TB_REQUIRE(X && Y, "tb_relu_mask_f32: null pointer");
  return relu_mask_inplace(X, Y, M, ncols, ldx, ldy, (cudaStream_t)stream);
}

int tb_core_extras(float* core, int64_t ld, int64_t N, int F, const float* reward, const int64_t* last_action, int A,
                   void* stream) {
  TB_REQUIRE(core && reward && (A == 0 || last_action), "tb_core_extras: null pointer");
  return core_extras(core, ld, N, F, reward, last_action, A, (cudaStream_t)stream);
}

// ---- ResNet patch-matrix path (resnet_kernels.cuh) ----------------------------------------------------------------
int tb_im2col3x3(const void* x, void* col, int64_t N, int H, int W, int C, int64_t ldk, int relu_in, int dtype, void* stream) {
  TB_REQUIRE(x && col, "tb_im2col3x3: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_im2col3x3", dtype,
              im2col3x3(static_cast<const float*>(x), static_cast<float*>(col), N, H, W, C, ldk, relu_in, st),
              im2col3x3(static_cast<const bf16*>(x), static_cast<bf16*>(col), N, H, W, C, ldk, relu_in, st));
}

// dtype 0: uint8 patch matrix (the fp32 backend reads it as x/255), 1: bf16
int tb_im2col3x3_u8(const uint8_t* frame, void* col, int64_t N, int C, int H, int W, int64_t ldk, int dtype, void* stream) {
  TB_REQUIRE(frame && col, "tb_im2col3x3_u8: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_im2col3x3_u8", dtype, im2col3x3_u8_nchw(frame, static_cast<uint8_t*>(col), N, C, H, W, ldk, st),
              im2col3x3_u8_nchw(frame, static_cast<bf16*>(col), N, C, H, W, ldk, st));
}

int tb_col2im3x3(const void* dcol, const void* relu_src, const void* addend, void* dx, int64_t N, int H, int W, int C, int64_t ldk,
                 int dtype, void* stream) {
  TB_REQUIRE(dcol && dx, "tb_col2im3x3: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_col2im3x3", dtype,
              col2im3x3(static_cast<const float*>(dcol), static_cast<const float*>(relu_src), static_cast<const float*>(addend),
                        static_cast<float*>(dx), N, H, W, C, ldk, st),
              col2im3x3(static_cast<const bf16*>(dcol), static_cast<const bf16*>(relu_src), static_cast<const bf16*>(addend),
                        static_cast<bf16*>(dx), N, H, W, C, ldk, st));
}

int tb_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* argmax, int64_t N, int H, int W, int C, int dtype, void* stream) {
  TB_REQUIRE(x && y && argmax, "tb_maxpool3x3s2_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_maxpool3x3s2_fwd", dtype,
              maxpool3x3s2_fwd(static_cast<const float*>(x), static_cast<float*>(y), argmax, N, H, W, C, st),
              maxpool3x3s2_fwd(static_cast<const bf16*>(x), static_cast<bf16*>(y), argmax, N, H, W, C, st));
}

int tb_maxpool3x3s2_bwd(const uint8_t* argmax, const void* dy, void* dx, int64_t N, int H, int W, int C, int dtype, void* stream) {
  TB_REQUIRE(argmax && dy && dx, "tb_maxpool3x3s2_bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_maxpool3x3s2_bwd", dtype,
              maxpool3x3s2_bwd(argmax, static_cast<const float*>(dy), static_cast<float*>(dx), N, H, W, C, st),
              maxpool3x3s2_bwd(argmax, static_cast<const bf16*>(dy), static_cast<bf16*>(dx), N, H, W, C, st));
}

int tb_relu_fwd(const void* x, void* y, int64_t n, int dtype, void* stream) {
  TB_REQUIRE(x && y, "tb_relu_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_relu_fwd", dtype, relu_fwd(static_cast<const float*>(x), static_cast<float*>(y), n, st),
              relu_fwd(static_cast<const bf16*>(x), static_cast<bf16*>(y), n, st));
}

int tb_relu_bwd(const void* x, const void* dy, void* dx, int64_t n, int dtype, void* stream) {
  TB_REQUIRE(x && dy && dx, "tb_relu_bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  TB_BY_DTYPE("tb_relu_bwd", dtype,
              relu_bwd(static_cast<const float*>(x), static_cast<const float*>(dy), static_cast<float*>(dx), n, st),
              relu_bwd(static_cast<const bf16*>(x), static_cast<const bf16*>(dy), static_cast<bf16*>(dx), n, st));
}

// ---- bias-gradient column sums ---------------------------------------------------------------------------------------
int64_t tb_colsum_scratch_floats(int64_t ncols) { return colsum_scratch_floats(ncols); }

int tb_colsum_f32(const float* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, void* stream) {
  return colsum(X, out, M, ncols, ld, scratch, (cudaStream_t)stream);
}

int tb_colsum_bf16(const void* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, int64_t lo_off,
                   void* stream) {
  return colsum_bf16(X, out, M, ncols, ld, scratch, (cudaStream_t)stream, lo_off);
}

// ---- fused policy / baseline heads (heads.cuh) -----------------------------------------------------------------------
int64_t tb_heads_scratch_floats(int64_t N, int F, int A, int V) { return heads_scratch_floats(N, F, A, V); }

int tb_heads_forward(const float* x, int64_t ldx, const float* Wp, const float* bp, const float* Wb, const float* bb, int64_t N,
                     int F, int A, int V, float* logits, float* baseline, void* stream) {
  return heads_forward(x, ldx, Wp, bp, Wb, bb, N, F, A, logits, baseline, (cudaStream_t)stream, V);
}

int tb_heads_backward(const float* x, int64_t ldx, const float* Wp, const float* Wb, const float* dlogits, const float* dbaseline,
                      int64_t N, int F, int A, int V, float* dx, int64_t lddx, float* dWp, float* dbp, float* dWb, float* dbb,
                      float* scratch, void* stream) {
  return heads_backward(x, ldx, Wp, Wb, dlogits, dbaseline, N, F, A, dx, lddx, dWp, dbp, dWb, dbb, scratch, (cudaStream_t)stream,
                        V);
}

}  // extern "C"
