// 3x3 / stride 1 / pad 1 convolutions of the IMPALA ResNet as shifted-window implicit GEMMs (see conv3x3_sw.cu).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace tb {

// Zero-padded, channel-chunk-planar split-bf16 image: [Nf][C/8][(H+2)*(W+2)][8] (hi plane; lo plane at + lo_off elements).
// One (pixel, 8 channels) unit is 16 bytes, the pixels of a chunk plane are contiguous: 128 consecutive flattened padded
// pixels are 128 rows of a K-major UMMA operand without swizzle (rows 16 bytes apart), and the window of tap (kh, kw) is the
// same rows shifted by (kh*(W+2) + kw)*16 bytes - every input element reaches shared memory ONCE per tile (plus halo).
// elements of one plane including the slack the last tile's window may run into
int64_t sw_image_elems(int64_t Nf, int H, int W, int C);
// fp32 NHWC [Nf, H, W, C] (optionally through ReLU) -> padded planar hi / lo image
int sw_pad_split(const float* x, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int H, int W, int C, int relu_in, cudaStream_t stream);
// same, and also db[C] = column sums of x (bias gradient when x is dL/d(conv output)); scratch >= kNumSMs*8*C floats
int sw_pad_split_colsum(const float* x, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int H, int W, int C, float* db,
                        float* scratch, int64_t scratch_floats, cudaStream_t stream);

// nn.MaxPool2d(3, 2, 1) backward fused with the image producer: dy_pooled [Nf, OH, OW, C] fp32 + the forward's argmax taps ->
// the padded planar hi / lo image of dL/d(pool input) [Nf, H, W, C] and its column sums db[C] (never materialised in fp32)
int sw_pool_bwd_image_colsum(const uint8_t* argmax, const float* dy_pooled, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int H, int W,
                             int C, float* db, float* scratch, int64_t scratch_floats, cudaStream_t stream);

// scratch floats of sw_pad_split_colsum / sw_pool_bwd_image_colsum on an Nf x H x W image with C channels: one row of C
// per 256-thread block plus the second-level slices
int64_t sw_colsum_scratch_floats(int64_t Nf, int H, int W, int C);

// uint8 NCHW frames [Nf, 1 <= Cf <= 16, H, W] -> padded planar image with 16 channels (channels >= Cf and the whole lo plane
// are zero; pixel values 0..255 are exact in bf16): the first convolution of the net through the same kernels
int sw_frames_u8(const uint8_t* frame, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int Cf, int H, int W, cudaStream_t stream);
// the same image (Cf = 4, byte-identical) from an unstacked rollout: frames u8 [T1+3, B, H, W], done [T1, B] (restack.cuh)
int sw_frames_u8_unstacked(const uint8_t* frames, const uint8_t* done, __nv_bfloat16* out, int64_t lo_off, int64_t T1, int64_t B,
                           int H, int W, cudaStream_t stream);

// weights [O, C, 3, 3] fp32 -> the shared-memory image of the B operand (sw_weight_elems(O, C) elements; R operand rows,
// the hi rows of a block followed by its lo rows so that [w_hi | w_lo] is one 2R-row operand):
//   transpose == 0 (forward):        R = O, K = C:  [tap][C/16][2][hi R rows | lo R rows][8]
//   transpose == 1 (input gradient): R = C, K = O:  [tap][O/16][2][hi R rows | lo R rows][8] with flipped taps (W[o, c, 2-a, 2-b])
// in blocks of RB = min(R, 32) rows, each block a complete operand of that layout with R = RB (one block when R <= 32;
// R = 64: two, one per column block of the wide forward kernel)
int64_t sw_weight_elems(int O, int C);
// c_real > 0 (forward only): the weight tensor has c_real < C input channels, the rest of the operand is zero
int sw_pack_weights(const float* w, __nv_bfloat16* out, int O, int C, int transpose, cudaStream_t stream, int c_real = 0);

struct SwEpilogue {
  float scale = 1.0f;              // applied to the accumulator first (1/255 for uint8 frames)
  const float* bias = nullptr;     // [NO]
  const float* mask = nullptr;     // [M, NO] fp32: out = mask > 0 ? out : 0 (ReLU backward), applied before the addend
  const float* addend = nullptr;   // [M, NO] fp32 residual / skip gradient, applied last
  // optional: also write the result (through ReLU if emit_relu) as the complete padded planar hi / lo image of the next conv
  // (same H x W, NO channels; sw_image_elems(Nf, H, W, NO) elements per plane, lo plane at + emit_lo) - no separate
  // sw_pad_split pass over the fp32 result
  __nv_bfloat16* emit = nullptr; int64_t emit_lo = 0; int emit_relu = 0;
  // optional: column sums of the result per (tile, epilogue warp): csum[sw_csum_rows(Nf, H, W)][NO] (+ 128*NO floats of
  // scratch behind it for sw_csum_reduce) - the bias gradient of the next conv when the result is its dY
  float* csum = nullptr;
  const char* tag = "conv3x3_sw";
};
int64_t sw_csum_rows(int64_t Nf, int H, int W);
// db[C] = column sums of csum[rows][C] in a fixed order (uses csum[rows*C .. rows*C + 128*C) as scratch)
int sw_csum_reduce(float* csum, int64_t rows, int C, float* db, cudaStream_t stream);

bool sw_conv_applicable(int H, int W, int CK, int NO);
// a CK -> NO conv at H x W can be trained on these kernels: it is applicable, W >= 5 (the weight gradient's last pixel step
// of a frame must end in the zero run behind it), and its forward, its input-gradient convolution (NO -> CK) and its weight
// gradient fit the shared memory (the input window grows with W + 2); input_grad = false: a first conv, whose input
// gradient is never formed
bool sw_conv_trainable(int H, int W, int CK, int NO, bool input_grad = true);
// out fp32 [Nf*H*W, NO] = epilogue(conv3x3(image) with the packed weights); CK = channels of the image (16 / 32 / 64),
// NO = output channels (16 / 32 / 64; a pair with a 64-channel side runs on sw_conv_fwd_wide_kernel)
int sw_conv_fwd(const __nv_bfloat16* img, int64_t img_lo, const __nv_bfloat16* wk, float* out, int64_t Nf, int H, int W, int CK, int NO,
                const SwEpilogue& ep, cudaStream_t stream);

// weight gradient dW[O, C, 3, 3] (fp32, reference layout) = sum over pixels dY (x) windows(x): dyimg = padded planar image of
// dL/d(conv output) (O channels), ximg = padded planar image of the conv's input (C channels); partial: split scratch
// c_real > 0: dW is [O, c_real, 3, 3] (the image's channels >= c_real are padding); scale multiplies the result
int sw_conv_wgrad(const __nv_bfloat16* dyimg, int64_t dy_lo, const __nv_bfloat16* ximg, int64_t x_lo, float* dW, int64_t Nf, int H,
                  int W, int C, int O, float* partial, int64_t partial_floats, const char* tag, cudaStream_t stream,
                  float scale = 1.0f, int c_real = 0);

}  // namespace tb
