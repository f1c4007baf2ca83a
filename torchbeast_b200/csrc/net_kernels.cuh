// Data-movement / pointwise kernels of the network path (declarations; definitions in
// net_kernels.cu).  Internal activation layout is NHWC ([frame, y, x, channel]) so that a
// convolution patch is a few long contiguous runs and a GEMM output tile IS the next layer's
// activation; the uint8 frames arrive NCHW ([T+1,B,4,84,84], reference monobeast.py:302).
#pragma once
#include "common.cuh"

namespace tb {

// frames u8 [N,C,H,W] -> patch matrix u8 [N*OH*OW, C*KH*KW], k = (c*KH + kh)*KW + kw  (== the
// reference weight's own [out, c, kh, kw] flattening, so conv1.weight is used unpermuted).
int im2col_u8_nchw(const uint8_t* frame, uint8_t* col, int64_t N, int C, int H, int W, int KH, int KW, int S,
                   cudaStream_t stream);

// act f32 NHWC [N,H,W,C] -> patch matrix f32 [N*OH*OW, KH*KW*C], k = (kh*KW + kw)*C + c.
int im2col_f32_nhwc(const float* act, float* col, int64_t N, int H, int W, int C, int KH, int KW, int S,
                    cudaStream_t stream);

// dcol f32 [N*OH*OW, KH*KW*C] -> d_act NHWC [N,H,W,C] (gather form, deterministic), multiplied by
// the ReLU mask of the forward activation `act` (same shape) when act != nullptr.
int col2im_f32_nhwc(const float* dcol, const float* act, float* dact, int64_t N, int H, int W, int C, int KH, int KW,
                    int S, cudaStream_t stream);

// out[o, p*Q + q] = in[o, q*P + p]   (weight pack: reference [o,c,kh,kw] -> GEMM [o,(kh,kw),c])
int permute_pq(const float* in, float* out, int64_t O, int P, int Q, cudaStream_t stream);

// out[n] = sum_m X[m*ld + n], n < ncols (bias gradients); deterministic two-stage reduction.
// scratch: >= colsum_scratch_floats(ncols) floats.
int64_t colsum_scratch_floats(int64_t ncols);
int colsum(const float* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, cudaStream_t stream);

// core[n, F] = clamp(reward[n], -1, 1); core[n, F+1+j] = (last_action[n] == j)   (monobeast.py:593-597)
// seg non-NULL (a factored action space, A = its width): last_action is [N, D] and the one-hot becomes a K-hot,
// core[n, F+1+off_k+last_action[n, k]] = 1 for each component k
int core_extras(float* core, int64_t ld, int64_t N, int F, const float* reward, const int64_t* last_action, int A,
                cudaStream_t stream, const ActionSegments* seg = nullptr);
// A continuous action space of D dimensions: core[n, F] = clamp(reward[n], -1, 1); core[n, F+1+k] = last_action[n, k]
// (float32 [N, D]) as it is
int core_extras_continuous(float* core, int64_t ld, int64_t N, int F, const float* reward, const float* last_action,
                           int D, cudaStream_t stream);

// X[m, n] *= (Y[m, n] > 0) for n < ncols (ReLU backward in place on a strided view)
int relu_mask_inplace(float* X, const float* Y, int64_t M, int64_t ncols, int64_t ldx, int64_t ldy,
                      cudaStream_t stream);

// ---- bf16 operand staging for the tensor-core backend ---------------------------------------
// out_bf16[o*ld_out + p*Q + q] = in[o*P*Q + q*P + p]; columns [P*Q, ld_out) zero
// lo_off != 0 (all three below): split-bf16 - also write / read the lo plane at +lo_off elements
int pack_weights_bf16(const float* in, void* out_bf16, int64_t O, int P, int Q, int64_t ld_out, cudaStream_t stream,
                      int64_t lo_off = 0);
// weights [O,C,KH,KW] fp32 -> bf16 B operand of the implicit input-gradient GEMMs (see gemm_tc.cuh)
int pack_dgrad_weights_bf16(const float* in, void* out_bf16, int O, int C, int KH, int KW, int S, cudaStream_t stream,
                            int64_t lo_off = 0);
// colsum over a bf16 matrix (bias gradients), fp32 accumulation
int colsum_bf16(const void* X_bf16, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, cudaStream_t stream,
                int64_t lo_off = 0);

}  // namespace tb
