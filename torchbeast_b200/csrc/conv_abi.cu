// C ABI of the convolution building blocks (bf16 and split-bf16 tensor-core backends) so that they can be
// tested in isolation against torch.nn.functional.conv2d; the learner calls the same internals from
// atarinet.cu and resnet.cu.  See include/torchbeast_b200.h.
#include "conv3x3_sw.cuh"
#include "conv_implicit.cuh"
#include "gemm_tc.cuh"
#include "net_kernels.cuh"
#include "resnet_kernels.cuh"

using namespace tb;

extern "C" {

int tb_conv_nhwc_bf16_fwd(const void* act_bf16, const float* weight, const float* bias, int64_t Nf, int H, int W, int C, int KH,
                          int KW, int S, int O, int relu, void* out_bf16, void* pack_scratch_bf16, void* stream) {
  TB_REQUIRE(act_bf16 && weight && bias && out_bf16 && pack_scratch_bf16, "tb_conv_nhwc_bf16_fwd: null pointer");
  TB_REQUIRE(conv_tc_implicit_applicable(H, W, C, KH, KW, S, O), "tb_conv_nhwc_bf16_fwd: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t K = int64_t(KH) * KW * C;
  int rc = pack_weights_bf16(weight, pack_scratch_bf16, O, KH * KW, C, K, st);
  if (rc) return rc;
  TcEpilogue te;
  te.C16 = static_cast<__nv_bfloat16*>(out_bf16); te.ldc16 = O; te.bias = bias; te.relu = relu; te.tag = "conv_fwd";
  return conv_tc_fwd_implicit(act_bf16, pack_scratch_bf16, Nf, H, W, C, KH, KW, S, O, te, st);
}

int tb_conv_nhwc_bf16_dgrad(const void* dy_bf16, const float* weight, const void* act_bf16, int64_t Nf, int H, int W, int C, int KH,
                            int KW, int S, int O, void* dx_bf16, void* pack_scratch_bf16, void* stream) {
  TB_REQUIRE(dy_bf16 && weight && dx_bf16 && pack_scratch_bf16, "tb_conv_nhwc_bf16_dgrad: null pointer");
  TB_REQUIRE(conv_tc_dgrad_implicit_applicable(H, W, C, KH, KW, S, O), "tb_conv_nhwc_bf16_dgrad: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = pack_dgrad_weights_bf16(weight, pack_scratch_bf16, O, C, KH, KW, S, st);
  if (rc) return rc;
  TcEpilogue te;
  te.C16 = static_cast<__nv_bfloat16*>(dx_bf16); te.ldc16 = C;
  te.mask16 = static_cast<const __nv_bfloat16*>(act_bf16); te.ldmask = C; te.tag = "conv_dgrad";
  return conv_tc_dgrad_implicit(dy_bf16, pack_scratch_bf16, Nf, H, W, C, KH, KW, S, O, te, st);
}

int tb_conv_nhwc_bf16_wgrad(const void* dy_bf16, const void* act_bf16, int64_t Nf, int H, int W, int C, int KH, int KW, int S, int O,
                            float* dweight, float* partial, int64_t partial_floats, void* stream) {
  TB_REQUIRE(conv_tc_implicit_applicable(H, W, C, KH, KW, S, O) && O <= 64, "tb_conv_nhwc_bf16_wgrad: unsupported shape");
  return conv_tc_wgrad_implicit(dy_bf16, act_bf16, Nf, H, W, C, KH, KW, S, O, dweight, KH * KW, C, 1.0f, partial, partial_floats,
                                "conv_wgrad", (cudaStream_t)stream);
}

int tb_conv1_u8_fwd(const uint8_t* frame, const float* weight, const float* bias, int64_t N, int H, int W, int S, int relu,
                    void* out_bf16, void* image_bf16, void* pack_scratch_bf16, void* stream) {
  TB_REQUIRE(frame && weight && bias && out_bf16 && image_bf16 && pack_scratch_bf16, "tb_conv1_u8_fwd: null pointer");
  TB_REQUIRE(conv_u8_implicit_applicable(4, H, W, 8, 8, S, 32), "tb_conv1_u8_fwd: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = pack_weights_bf16(weight, pack_scratch_bf16, 32, 1, 256, 256, st);  // reference flattening (c, kh, kw) kept
  if (rc) return rc;
  rc = frames_u8_to_bf16(frame, image_bf16, N * 4 * H * W, st);
  if (rc) return rc;
  TcEpilogue te;
  te.C16 = static_cast<__nv_bfloat16*>(out_bf16); te.ldc16 = 32; te.bias = bias; te.scale = 1.0f / 255.0f; te.relu = relu;
  te.tag = "conv1_fwd";
  return conv_u8_fwd_implicit(image_bf16, pack_scratch_bf16, N, H, W, S, te, st);
}

int tb_conv1_u8_wgrad(const void* dy_bf16, const void* image_bf16, int64_t N, int H, int W, int S, float* dweight, float* partial,
                      int64_t partial_floats, void* stream) {
  TB_REQUIRE(conv_u8_implicit_applicable(4, H, W, 8, 8, S, 32), "tb_conv1_u8_wgrad: unsupported shape");
  return conv_u8_wgrad_implicit(dy_bf16, image_bf16, N, H, W, S, dweight, 1.0f / 255.0f, partial, partial_floats, "conv1_wgrad",
                                (cudaStream_t)stream);
}

// ---- split-bf16 (bf16x3) forms: every bf16 operand is a hi plane with its lo plane *_lo elements further; the packed
// weights are written as hi plane [0, O*KH*KW*C) and lo plane right behind it
int tb_conv_nhwc_bf16x3_fwd(const void* act_bf16, int64_t act_lo, const float* weight, const float* bias, int64_t Nf, int H, int W,
                            int C, int KH, int KW, int S, int O, int relu, void* out_bf16, int64_t out_lo, void* pack_scratch_bf16,
                            void* stream) {
  TB_REQUIRE(act_bf16 && weight && bias && out_bf16 && pack_scratch_bf16, "tb_conv_nhwc_bf16x3_fwd: null pointer");
  TB_REQUIRE(act_lo > 0 && out_lo > 0, "tb_conv_nhwc_bf16x3_fwd: the input and output need lo planes");
  TB_REQUIRE(conv_tc_implicit_applicable(H, W, C, KH, KW, S, O), "tb_conv_nhwc_bf16x3_fwd: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t K = int64_t(KH) * KW * C;
  int rc = pack_weights_bf16(weight, pack_scratch_bf16, O, KH * KW, C, K, st, int64_t(O) * K);
  if (rc) return rc;
  TcEpilogue te;
  te.C16 = static_cast<__nv_bfloat16*>(out_bf16); te.ldc16 = O; te.c16_lo = out_lo; te.bias = bias; te.relu = relu;
  te.a_lo = act_lo; te.b_lo = int64_t(O) * K; te.tag = "conv_fwd";
  return conv_tc_fwd_implicit(act_bf16, pack_scratch_bf16, Nf, H, W, C, KH, KW, S, O, te, st);
}

int tb_conv_nhwc_bf16x3_dgrad(const void* dy_bf16, int64_t dy_lo, const float* weight, const void* act_bf16, int64_t Nf, int H,
                              int W, int C, int KH, int KW, int S, int O, void* dx_bf16, int64_t dx_lo, void* pack_scratch_bf16,
                              void* stream) {
  TB_REQUIRE(dy_bf16 && weight && dx_bf16 && pack_scratch_bf16, "tb_conv_nhwc_bf16x3_dgrad: null pointer");
  TB_REQUIRE(dy_lo > 0 && dx_lo > 0, "tb_conv_nhwc_bf16x3_dgrad: dY and dX need lo planes");
  TB_REQUIRE(conv_tc_dgrad_implicit_applicable(H, W, C, KH, KW, S, O), "tb_conv_nhwc_bf16x3_dgrad: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t wl = int64_t(O) * C * KH * KW;
  int rc = pack_dgrad_weights_bf16(weight, pack_scratch_bf16, O, C, KH, KW, S, st, wl);
  if (rc) return rc;
  TcEpilogue te;
  te.C16 = static_cast<__nv_bfloat16*>(dx_bf16); te.ldc16 = C; te.c16_lo = dx_lo;
  te.mask16 = static_cast<const __nv_bfloat16*>(act_bf16); te.ldmask = C;   // the ReLU mask reads the hi plane
  te.a_lo = dy_lo; te.b_lo = wl; te.tag = "conv_dgrad";
  return conv_tc_dgrad_implicit(dy_bf16, pack_scratch_bf16, Nf, H, W, C, KH, KW, S, O, te, st);
}

int tb_conv_nhwc_bf16x3_wgrad(const void* dy_bf16, int64_t dy_lo, const void* act_bf16, int64_t act_lo, int64_t Nf, int H, int W,
                              int C, int KH, int KW, int S, int O, float* dweight, float* partial, int64_t partial_floats,
                              void* stream) {
  TB_REQUIRE(dy_lo > 0 && act_lo > 0, "tb_conv_nhwc_bf16x3_wgrad: dY and the activation need lo planes");
  TB_REQUIRE(conv_tc_implicit_applicable(H, W, C, KH, KW, S, O) && O <= 64, "tb_conv_nhwc_bf16x3_wgrad: unsupported shape");
  return conv_tc_wgrad_implicit(dy_bf16, act_bf16, Nf, H, W, C, KH, KW, S, O, dweight, KH * KW, C, 1.0f, partial, partial_floats,
                                "conv_wgrad", (cudaStream_t)stream, dy_lo, act_lo);
}

// conv1 on split weights: the pixels are exact in bf16, so only the weights and the output have lo planes
int tb_conv1_u8_bf16x3_fwd(const uint8_t* frame, const float* weight, const float* bias, int64_t N, int H, int W, int S, int relu,
                           void* out_bf16, int64_t out_lo, void* image_bf16, void* pack_scratch_bf16, void* stream) {
  TB_REQUIRE(frame && weight && bias && out_bf16 && image_bf16 && pack_scratch_bf16, "tb_conv1_u8_bf16x3_fwd: null pointer");
  TB_REQUIRE(out_lo > 0, "tb_conv1_u8_bf16x3_fwd: the output needs a lo plane");
  TB_REQUIRE(conv_u8_implicit_applicable(4, H, W, 8, 8, S, 32), "tb_conv1_u8_bf16x3_fwd: unsupported shape");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = pack_weights_bf16(weight, pack_scratch_bf16, 32, 1, 256, 256, st, 32 * 256);
  if (rc) return rc;
  rc = frames_u8_to_bf16(frame, image_bf16, N * 4 * H * W, st);
  if (rc) return rc;
  TcEpilogue te;
  te.C16 = static_cast<__nv_bfloat16*>(out_bf16); te.ldc16 = 32; te.c16_lo = out_lo; te.bias = bias; te.scale = 1.0f / 255.0f;
  te.relu = relu; te.b_lo = 32 * 256; te.tag = "conv1_fwd";
  return conv_u8_fwd_implicit(image_bf16, pack_scratch_bf16, N, H, W, S, te, st);
}

int tb_conv1_u8_bf16x3_wgrad(const void* dy_bf16, int64_t dy_lo, const void* image_bf16, int64_t N, int H, int W, int S,
                             float* dweight, float* partial, int64_t partial_floats, void* stream) {
  TB_REQUIRE(dy_lo > 0, "tb_conv1_u8_bf16x3_wgrad: dY needs a lo plane");
  TB_REQUIRE(conv_u8_implicit_applicable(4, H, W, 8, 8, S, 32), "tb_conv1_u8_bf16x3_wgrad: unsupported shape");
  return conv_u8_wgrad_implicit(dy_bf16, image_bf16, N, H, W, S, dweight, 1.0f / 255.0f, partial, partial_floats, "conv1_wgrad",
                                (cudaStream_t)stream, dy_lo);
}

// ---- ResNet shifted-window convolutions (conv3x3_sw.cuh) and the producers of their images -----------------------
int64_t tb_sw_image_elems(int64_t Nf, int H, int W, int C) { return sw_image_elems(Nf, H, W, C); }
int64_t tb_sw_colsum_scratch_floats(int64_t Nf, int H, int W, int C) { return sw_colsum_scratch_floats(Nf, H, W, C); }
int64_t tb_sw_weight_elems(int O, int C) { return sw_weight_elems(O, C); }
int64_t tb_sw_csum_rows(int64_t Nf, int H, int W) { return sw_csum_rows(Nf, H, W); }

int tb_sw_pad_split_f32(const float* x, void* out, int64_t lo_off, int64_t Nf, int H, int W, int C, int relu_in, float* db,
                        float* scratch, int64_t scratch_floats, void* stream) {
  TB_REQUIRE(x && out && lo_off > 0, "tb_sw_pad_split_f32: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out);
  if (!db) return sw_pad_split(x, o, lo_off, Nf, H, W, C, relu_in, st);
  TB_REQUIRE(!relu_in && scratch, "tb_sw_pad_split_f32: the column-sum form takes no ReLU and needs scratch");
  return sw_pad_split_colsum(x, o, lo_off, Nf, H, W, C, db, scratch, scratch_floats, st);
}

int tb_sw_frames_u8(const uint8_t* frame, void* out, int64_t lo_off, int64_t Nf, int Cf, int H, int W, void* stream) {
  TB_REQUIRE(frame && out && lo_off > 0, "tb_sw_frames_u8: null pointer");
  return sw_frames_u8(frame, static_cast<__nv_bfloat16*>(out), lo_off, Nf, Cf, H, W, (cudaStream_t)stream);
}

int tb_sw_pack_weights(const float* weight, void* out, int O, int C, int transpose, int c_real, void* stream) {
  TB_REQUIRE(weight && out, "tb_sw_pack_weights: null pointer");
  return sw_pack_weights(weight, static_cast<__nv_bfloat16*>(out), O, C, transpose, (cudaStream_t)stream, c_real);
}

int tb_sw_conv_fwd(const void* img, int64_t img_lo, const void* wk, float* out, int64_t Nf, int H, int W, int CK, int NO,
                   float scale, const float* bias, const float* mask, const float* addend, void* emit, int64_t emit_lo,
                   int emit_relu, float* csum, void* stream) {
  SwEpilogue ep;
  ep.scale = scale; ep.bias = bias; ep.mask = mask; ep.addend = addend;
  ep.emit = static_cast<__nv_bfloat16*>(emit); ep.emit_lo = emit_lo; ep.emit_relu = emit_relu; ep.csum = csum;
  return sw_conv_fwd(static_cast<const __nv_bfloat16*>(img), img_lo, static_cast<const __nv_bfloat16*>(wk), out, Nf, H, W, CK, NO,
                     ep, (cudaStream_t)stream);
}

int tb_sw_csum_reduce(float* csum, int64_t rows, int C, float* db, void* stream) {
  TB_REQUIRE(csum && db, "tb_sw_csum_reduce: null pointer");
  return sw_csum_reduce(csum, rows, C, db, (cudaStream_t)stream);
}

int tb_sw_conv_wgrad(const void* dyimg, int64_t dy_lo, const void* ximg, int64_t x_lo, float* dweight, int64_t Nf, int H, int W,
                     int C, int O, float scale, int c_real, float* partial, int64_t partial_floats, void* stream) {
  return sw_conv_wgrad(static_cast<const __nv_bfloat16*>(dyimg), dy_lo, static_cast<const __nv_bfloat16*>(ximg), x_lo, dweight, Nf,
                       H, W, C, O, partial, partial_floats, "conv3x3_sw_wgrad", (cudaStream_t)stream, scale, c_real);
}

int tb_sw_pool_bwd_image_colsum(const uint8_t* argmax, const float* dy_pooled, void* out, int64_t lo_off, int64_t Nf, int H, int W,
                                int C, float* db, float* scratch, int64_t scratch_floats, void* stream) {
  TB_REQUIRE(argmax && dy_pooled && out && db && scratch && lo_off > 0, "tb_sw_pool_bwd_image_colsum: null pointer");
  return sw_pool_bwd_image_colsum(argmax, dy_pooled, static_cast<__nv_bfloat16*>(out), lo_off, Nf, H, W, C, db, scratch,
                                  scratch_floats, (cudaStream_t)stream);
}

int tb_maxpool3x3s2_fwd_f32(const float* x, float* y, uint8_t* argmax, int64_t N, int H, int W, int C, void* stream) {
  TB_REQUIRE(x && y && argmax, "tb_maxpool3x3s2_fwd_f32: null pointer");
  return maxpool3x3s2_fwd<float>(x, y, argmax, N, H, W, C, (cudaStream_t)stream);
}

}  // extern "C"
