// Implicit-GEMM first convolution over uint8 NCHW frames (see conv_implicit.cu): host interface.
#pragma once
#include "gemm_tc.cuh"

namespace tb {

// true when the wgmma implicit-GEMM kernels cover this shape (8x8 kernel, 4 input / 32 output channels,
// W and stride multiples of 4)
bool conv_u8_implicit_applicable(int C, int H, int W, int KH, int KW, int S, int O);

// frames u8 NCHW -> bf16 NCHW (exact), the operand image of the two kernels below
int frames_u8_to_bf16(const uint8_t* frame, void* frame_bf16, int64_t count, cudaStream_t stream);
// the same image [T1*B, 4, HW] (byte-identical) from an unstacked rollout: frames u8 [T1+3, B, HW], done [T1, B]
// (restack.cuh); HW % 16 == 0
int frames_u8_unstacked_to_bf16(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW,
                                void* frame_bf16, cudaStream_t stream);

// act[N*OH*OW, 32] (bf16, ep.C16) = relu(ep.scale * patches(frame) . W^T + ep.bias); w_bf16 [32, 256] with
// k = (c*8 + kh)*8 + kw (the reference weight's own flattening).  Split-bf16: ep.b_lo = lo plane of the weights
// (the pixels are exact in bf16), ep.c16_lo = lo plane of the output.
int conv_u8_fwd_implicit(const void* frame_bf16, const void* w_bf16, int64_t N, int H, int W, int S, const TcEpilogue& ep,
                         cudaStream_t stream);

// dW[32, 256] (fp32) = scale * dY^T . patches(frame); dy_bf16 [N*OH*OW, 32]; partial: split scratch
// (>= kNumSMs*32*256 floats), reduced in fixed order
int conv_u8_wgrad_implicit(const void* dy_bf16, const void* frame_bf16, int64_t N, int H, int W, int S, float* dW, float scale,
                           float* partial, int64_t partial_floats, const char* tag, cudaStream_t stream, int64_t dy_lo = 0);

}  // namespace tb
