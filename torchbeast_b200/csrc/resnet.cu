// IMPALA "deep" ResNet (polybeast_learner.Net) forward / backward for the learner, behind the C ABI.
//
// Replaces /root/reference/torchbeast/polybeast_learner.py:214-266 (Net.forward) and its autograd graph:
//   for ch in (16, 32, 32):  x = maxpool3x3/2(conv3x3(x));  x += conv(relu(conv(relu(x))));  x += conv(relu(conv(relu(x))))
//   x = relu(x) -> fc 3872->256 -> relu -> cat[x, clip(reward)] -> [LSTM(257->256)] -> policy / baseline
// Same construction as atarinet.cu: NHWC activations, every conv a patch-matrix GEMM through the shared
// GEMM backends (fp32 SIMT for parity, bf16 wgmma for throughput - the activation element type T
// follows the backend), residual adds fused into the GEMM epilogue, ReLU-on-read fused into the patch
// gather, ReLU masks and skip-gradients fused into the gather-form col2im, weights/gradients in ONE
// flat buffer in state_dict order.  Patch matrices are recomputed in the backward pass (a gather is
// cheaper than keeping 15 of them resident).
#include <type_traits>

#include "gemm_simt.cuh"
#include "gemm_tc.cuh"
#include "heads.cuh"
#include "lstm.cuh"
#include "net_kernels.cuh"
#include "resnet_kernels.cuh"
#include "conv3x3_sw.cuh"

namespace tb {

namespace {

constexpr int kSections = 3;
constexpr int kSecCh[kSections] = {16, 32, 32};
constexpr int kSecCin[kSections] = {4, 16, 32};
constexpr int kSecS[kSections] = {84, 42, 21};     // spatial size of the section's feat conv
constexpr int kSecSo[kSections] = {42, 21, 11};    // after the max-pool
constexpr int kFcIn = 32 * 11 * 11;                // 3872
constexpr int kFcOut = 256;
constexpr int kLstmH = 256;
constexpr int64_t kScratchFloats = int64_t(8) << 20;

struct ConvP { int64_t w, b; };
struct ResParams {
  ConvP feat[kSections], blk[kSections][4];  // blk: r1a, r1b, r2a, r2b
  int64_t fc_w, fc_b, lstm[4], policy_w, policy_b, baseline_w, baseline_b, total;
  int core_in, core_out;
};

ResParams res_params(int A, int use_lstm) {
  ResParams p;
  int64_t o = 0;
  auto take = [&](int64_t n) { int64_t r = o; o += n; return r; };
  for (int i = 0; i < kSections; ++i) { p.feat[i].w = take(int64_t(kSecCh[i]) * kSecCin[i] * 9); p.feat[i].b = take(kSecCh[i]); }
  for (int blk = 0; blk < 2; ++blk)     // resnet1.{0,1,2}.{1,3} then resnet2.{0,1,2}.{1,3}
    for (int i = 0; i < kSections; ++i)
      for (int j = 0; j < 2; ++j) {
        p.blk[i][blk * 2 + j].w = take(int64_t(kSecCh[i]) * kSecCh[i] * 9);
        p.blk[i][blk * 2 + j].b = take(kSecCh[i]);
      }
  p.fc_w = take(int64_t(kFcOut) * kFcIn); p.fc_b = take(kFcOut);
  p.core_in = kFcOut + 1;
  p.core_out = use_lstm ? kLstmH : p.core_in;
  for (int k = 0; k < 4; ++k) p.lstm[k] = -1;
  if (use_lstm) {
    p.lstm[0] = take(int64_t(4) * kLstmH * p.core_in); p.lstm[1] = take(int64_t(4) * kLstmH * kLstmH);
    p.lstm[2] = take(4 * kLstmH); p.lstm[3] = take(4 * kLstmH);
  }
  p.policy_w = take(int64_t(A) * p.core_out); p.policy_b = take(A);
  p.baseline_w = take(p.core_out); p.baseline_b = take(1);
  p.total = o;
  return p;
}

template <typename T> struct Sec { T *P, *X0, *Y1, *X1, *Y2, *X2; uint8_t* arg; };

template <typename T>
struct ResWs {
  Sec<T> s[kSections];
  T *fcin, *dfc, *dfcin, *g[3], *col, *dcol;
  T *wfeat[kSections], *wblk[kSections][4], *wfc;
  float *core_in, *core_out, *dcore_out, *dcore_in, *splitk, *colsum_scratch;
  int64_t splitk_floats = 0;   // >= kScratchFloats; the split backend's per-tile column-sum partials grow with the frame count
  // split-bf16 backend (precision 2): activations stay fp32; only the GEMM operands are bf16 hi / lo planes
  // (lo plane = hi pointer + the *_lo element offset)
  __nv_bfloat16 *fcb = nullptr, *dfcb = nullptr, *wb_fc = nullptr;
  int64_t fcb_lo = 0, dfcb_lo = 0, wb_fc_lo = 0;
  // every 3x3 conv is a shifted-window implicit GEMM (conv3x3_sw.cuh): the conv's input as a zero-padded
  // channel-chunk-planar split-bf16 image, kept for the weight gradient; the images of dY (ping-pong); weights in the
  // kernels' shared-memory layout (wi: forward, wd: flipped / transposed for the input-gradient convolution)
  __nv_bfloat16 *wd_feat[kSections] = {nullptr, nullptr, nullptr}, *wd_blk[kSections][4] = {};
  int64_t wd_feat_lo[kSections] = {0, 0, 0}, wd_blk_lo[kSections][4] = {};
  __nv_bfloat16 *xp_feat[kSections] = {nullptr, nullptr, nullptr}, *xp_blk[kSections][4] = {}, *dyp = nullptr, *dyp2 = nullptr;
  int64_t xp_feat_lo[kSections] = {0, 0, 0}, xp_blk_lo[kSections][4] = {}, dyp_lo = 0, dyp2_lo = 0;
  __nv_bfloat16 *wi_feat[kSections] = {nullptr, nullptr, nullptr}, *wi_blk[kSections][4] = {};
  int64_t wi_feat_lo[kSections] = {0, 0, 0}, wi_blk_lo[kSections][4] = {};
  LstmWs lstm;
  size_t bytes;
};

inline int64_t ldk_of(int cin, bool bf16) { const int64_t k = int64_t(cin) * 9; return bf16 ? ((k + 7) & ~int64_t(7)) : k; }

template <typename T>
ResWs<T> res_ws(void* base, int64_t N, int64_t T1, int64_t B, int A, int use_lstm, bool split = false) {
  constexpr bool kBf16 = !std::is_same<T, float>::value;
  ResWs<T> w;
  size_t off = 0;
  auto take = [&](size_t nbytes) { void* p = base ? static_cast<char*>(base) + off : nullptr; off += (nbytes + 255) & ~size_t(255); return p; };
  auto takeT = [&](int64_t n) { return static_cast<T*>(take(size_t(n) * sizeof(T))); };
  auto takef = [&](int64_t n) { return static_cast<float*>(take(size_t(n) * sizeof(float))); };
  const ResParams pp = res_params(A, use_lstm);
  int64_t maxact = 0;
  for (int i = 0; i < kSections; ++i) {
    const int64_t big = N * kSecS[i] * kSecS[i] * kSecCh[i], small = N * kSecSo[i] * kSecSo[i] * kSecCh[i];
    w.s[i].P = takeT(big); w.s[i].X0 = takeT(small); w.s[i].Y1 = takeT(small); w.s[i].X1 = takeT(small);
    w.s[i].Y2 = takeT(small); w.s[i].X2 = takeT(small);
    w.s[i].arg = static_cast<uint8_t*>(take(size_t(small)));
    if (big > maxact) maxact = big;
  }
  w.fcin = takeT(N * kFcIn); w.dfc = takeT(N * kFcOut); w.dfcin = takeT(N * kFcIn);
  for (int k = 0; k < 3; ++k) w.g[k] = takeT(maxact);
  int64_t maxcol = 0;
  for (int i = 0; i < kSections; ++i) {
    const int64_t a = N * kSecS[i] * kSecS[i] * ldk_of(kSecCin[i], kBf16), b = N * kSecSo[i] * kSecSo[i] * ldk_of(kSecCh[i], kBf16);
    if (a > maxcol) maxcol = a;
    if (b > maxcol) maxcol = b;
  }
  w.col = split ? nullptr : takeT(maxcol);   // (the split backend's convolutions gather their own operands)
  w.dcol = split ? nullptr : takeT(maxcol);
  if (split) {
    auto takeh = [&](int64_t n, int64_t& lo) {
      lo = (n + 127) & ~int64_t(127);
      return static_cast<__nv_bfloat16*>(take(size_t(2) * lo * sizeof(__nv_bfloat16)));
    };
    w.fcb = takeh(N * kFcIn, w.fcb_lo);
    w.dfcb = takeh(N * kFcOut, w.dfcb_lo);
    w.wb_fc = takeh(int64_t(kFcOut) * kFcIn, w.wb_fc_lo);
    for (int i = 0; i < kSections; ++i) {
      if (i > 0) w.wd_feat[i] = takeh(int64_t(kSecCin[i]) * 9 * kSecCh[i], w.wd_feat_lo[i]);
      for (int j = 0; j < 4; ++j) w.wd_blk[i][j] = takeh(int64_t(kSecCh[i]) * 9 * kSecCh[i], w.wd_blk_lo[i][j]);
    }
    int64_t maxp = 0;
    for (int i = 0; i < kSections; ++i) {
      {   // (the 4 frame channels of the first conv are padded to 16)
        const int cin16 = kSecCin[i] < 16 ? 16 : kSecCin[i];
        w.xp_feat[i] = takeh(sw_image_elems(N, kSecS[i], kSecS[i], cin16), w.xp_feat_lo[i]);
        w.wi_feat[i] = takeh(sw_weight_elems(kSecCh[i], cin16) / 2, w.wi_feat_lo[i]);
        const int64_t e = sw_image_elems(N, kSecS[i], kSecS[i], kSecCh[i]);
        if (e > maxp) maxp = e;
      }
      for (int j = 0; j < 4; ++j) {
        w.xp_blk[i][j] = takeh(sw_image_elems(N, kSecSo[i], kSecSo[i], kSecCh[i]), w.xp_blk_lo[i][j]);
        w.wi_blk[i][j] = takeh(sw_weight_elems(kSecCh[i], kSecCh[i]) / 2, w.wi_blk_lo[i][j]);
      }
      const int64_t e = sw_image_elems(N, kSecSo[i], kSecSo[i], kSecCh[i]);
      if (e > maxp) maxp = e;
    }
    w.dyp = takeh(maxp, w.dyp_lo);     // dY images ping-pong: a conv's input-gradient epilogue writes the next conv's dY image
    w.dyp2 = takeh(maxp, w.dyp2_lo);
  }
  for (int i = 0; i < kSections; ++i) {
    w.wfeat[i] = takeT(int64_t(kSecCh[i]) * ldk_of(kSecCin[i], kBf16));
    for (int j = 0; j < 4; ++j) w.wblk[i][j] = takeT(int64_t(kSecCh[i]) * ldk_of(kSecCh[i], kBf16));
  }
  w.wfc = takeT(int64_t(kFcOut) * kFcIn);
  w.core_in = takef(N * pp.core_in);
  w.core_out = use_lstm ? takef(N * pp.core_out) : w.core_in;
  w.dcore_out = takef(N * (pp.core_in > pp.core_out ? pp.core_in : pp.core_out));
  w.dcore_in = use_lstm ? takef(N * pp.core_in) : w.dcore_out;
  // split-K partials need kScratchFloats; the split backend's fixed-order column-sum partials need up to ~1000 floats per frame
  // (one row of C floats per 128-pixel block / per tile and epilogue warp of the largest image)
  w.splitk_floats = kScratchFloats;
  if (split && N * 1056 + 8192 > w.splitk_floats) w.splitk_floats = N * 1056 + 8192;
  w.splitk = takef(w.splitk_floats);
  w.colsum_scratch = takef(colsum_scratch_floats(4 * kLstmH));
  if (use_lstm) {
    const int lprec = split ? 2 : (kBf16 ? 1 : 0);
    const size_t lb = lstm_ws_bytes(T1, B, pp.core_in, kLstmH, 1, lprec);
    w.lstm = lstm_ws(take(lb), T1, B, pp.core_in, kLstmH, 1, lprec);
  } else {
    w.lstm = LstmWs();
  }
  w.bytes = off;
  return w;
}

#define TB_TRY(expr)        \
  do {                      \
    int _rc = (expr);       \
    if (_rc) return _rc;    \
  } while (0)

int splits_simt(int64_t M, int64_t N, int64_t K) {
  const int64_t bm = (N <= 32) ? 128 : (M <= 64 ? 64 : 128), bn = (N <= 32) ? 32 : 64;
  const int64_t tiles = ((M + bm - 1) / bm) * ((N + bn - 1) / bn);
  int64_t s = (2 * kNumSMs + tiles - 1) / tiles;
  const int64_t kt = (K + kGemmBK - 1) / kGemmBK;
  if (s > kt / 4) s = kt / 4;
  if (s * M * N > kScratchFloats) s = kScratchFloats / (M * N);
  if (s > 128) s = 128;
  return int(s < 1 ? 1 : s);
}
int splits_tc(int64_t M, int64_t N, int64_t K) {
  const int64_t bn = N <= 64 ? 64 : 128;
  const int64_t tiles = ((M + 127) / 128) * ((N + bn - 1) / bn);
  int64_t s = (2 * kNumSMs + tiles - 1) / tiles;
  const int64_t kb = (K + 63) / 64;
  if (s > kb / 4) s = kb / 4;
  const int64_t Np = (N + 31) & ~int64_t(31);  // partial rows are padded to 32 floats (gemm_tc.cu)
  if (s * M * Np > kScratchFloats) s = kScratchFloats / (M * Np);
  if (s > kNumSMs) s = kNumSMs;
  return int(s < 1 ? 1 : s);
}

// ---- backend-generic GEMM wrappers ------------------------------------------------------------
// forward: out[M,cout] = scale * col[M,K] . W[cout,K]^T + bias (+relu) (+addend)
int conv_fwd(const float* col, const float* W, float* out, int64_t M, int cout, int64_t K, int64_t ldk, const float* bias,
             int relu, const float* addend, float /*scale*/, int64_t ldc, const char* tag, cudaStream_t st) {
  GemmEpilogue ep; ep.bias = bias; ep.relu = relu; ep.addend = addend; ep.ldadd = cout; ep.tag = tag;
  return gemm_simt<float, float, false, true>(col, W, out, M, cout, K, ldk, ldk, ldc, ep, 1, nullptr, st);
}
int conv_fwd_u8(const uint8_t* col, const float* W, float* out, int64_t M, int cout, int64_t K, int64_t ldk, const float* bias,
                const char* tag, cudaStream_t st) {
  GemmEpilogue ep; ep.bias = bias; ep.tag = tag;
  return gemm_simt<uint8_t, float, false, true>(col, W, out, M, cout, K, ldk, ldk, cout, ep, 1, nullptr, st);
}
int conv_fwd(const __nv_bfloat16* col, const __nv_bfloat16* W, __nv_bfloat16* out, int64_t M, int cout, int64_t K, int64_t ldk,
             const float* bias, int relu, const __nv_bfloat16* addend, float scale, int64_t ldc, const char* tag, cudaStream_t st) {
  TcEpilogue te; te.C16 = out; te.ldc16 = ldc; te.bias = bias; te.relu = relu; te.addend16 = addend; te.ldadd = cout;
  te.scale = scale; te.tag = tag;
  return gemm_tc_bf16(col, W, M, cout, K, ldk, ldk, te, st);
}
// dgrad: dcol[M,K] = dY[M,cout] . W[cout,K]
int conv_dgrad(const float* dY, const float* W, float* dcol, int64_t M, int cout, int64_t K, int64_t ldk, const char* tag,
               cudaStream_t st) {
  GemmEpilogue ep; ep.tag = tag;
  return gemm_simt<float, float, false, false>(dY, W, dcol, M, K, cout, cout, ldk, ldk, ep, 1, nullptr, st);
}
int conv_dgrad(const __nv_bfloat16* dY, const __nv_bfloat16* W, __nv_bfloat16* dcol, int64_t M, int cout, int64_t K, int64_t ldk,
               const char* tag, cudaStream_t st) {
  TcEpilogue te; te.C16 = dcol; te.ldc16 = ldk; te.tag = tag;
  return gemm_tc_bf16_ex(dY, W, M, K, cout, cout, ldk, false, true, te, 1, nullptr, st);
}
// wgrad: dW[cout,K] (fp32, un-packed by the split-K reduce) = scale * dY[M,cout]^T . col[M,K]
int conv_wgrad(const float* dY, const void* col, bool col_u8, float* dW, int64_t M, int cout, int64_t K, int64_t ldk, int permP,
               int permQ, float /*scale: the u8 operand is read as x/255*/, float* scratch, const char* tag, cudaStream_t st) {
  GemmEpilogue ep; ep.permP = permP; ep.permQ = permQ; ep.tag = tag;
  const int s = splits_simt(cout, K, M);
  if (col_u8)
    return gemm_simt<float, uint8_t, true, false>(dY, static_cast<const uint8_t*>(col), dW, cout, K, M, cout, ldk, K, ep, s, scratch, st);
  return gemm_simt<float, float, true, false>(dY, static_cast<const float*>(col), dW, cout, K, M, cout, ldk, K, ep, s, scratch, st);
}
int conv_wgrad(const __nv_bfloat16* dY, const void* col, bool, float* dW, int64_t M, int cout, int64_t K, int64_t ldk, int permP,
               int permQ, float scale, float* scratch, const char* tag, cudaStream_t st) {
  TcEpilogue te; te.C = dW; te.ldc = K; te.permP = permP; te.permQ = permQ; te.scale = scale; te.tag = tag;
  return gemm_tc_bf16_ex(dY, col, cout, K, M, cout, ldk, true, true, te, splits_tc(cout, K, M), scratch, st);
}
int pack_w(const float* in, float* out, int64_t O, int P, int Q, int64_t, cudaStream_t st) { return permute_pq(in, out, O, P, Q, st); }
int pack_w(const float* in, __nv_bfloat16* out, int64_t O, int P, int Q, int64_t ld, cudaStream_t st) {
  return pack_weights_bf16(in, out, O, P, Q, ld, st);
}
// fc forward into the fp32 core buffer
int fc_fwd(const float* x, const float* W, float* core, int64_t N, int64_t ldc, const float* bias, cudaStream_t st) {
  GemmEpilogue ep; ep.bias = bias; ep.relu = 1; ep.tag = "fc_fwd";
  return gemm_simt<float, float, false, true>(x, W, core, N, kFcOut, kFcIn, kFcIn, kFcIn, ldc, ep, 1, nullptr, st);
}
int fc_fwd(const __nv_bfloat16* x, const __nv_bfloat16* W, float* core, int64_t N, int64_t ldc, const float* bias, cudaStream_t st) {
  TcEpilogue te; te.C = core; te.ldc = ldc; te.bias = bias; te.relu = 1; te.tag = "fc_fwd";
  return gemm_tc_bf16(x, W, N, kFcOut, kFcIn, kFcIn, kFcIn, te, st);
}

template <typename T>
struct Impl {
  static constexpr bool kBf16 = !std::is_same<T, float>::value;
  using ColFirst = typename std::conditional<kBf16, __nv_bfloat16, uint8_t>::type;

  static int forward(const uint8_t* frame, const float* reward, const float* notdone, const float* h0, const float* c0,
                     const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace, float* policy_logits,
                     float* baseline, float* hN, float* cN, cudaStream_t st) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(A, use_lstm);
    ResWs<T> w = res_ws<T>(workspace, N, T1, B, A, use_lstm);
    // weight pack: [o, c, kh, kw] -> [o, (kh,kw), c]; first conv keeps (c,kh,kw); fc: [o, c, (h,w)] -> [o, (h,w), c]
    TB_TRY(pack_w(P + pp.feat[0].w, w.wfeat[0], kSecCh[0], 1, 36, ldk_of(4, kBf16), st));
    for (int i = 0; i < kSections; ++i) {
      if (i > 0) TB_TRY(pack_w(P + pp.feat[i].w, w.wfeat[i], kSecCh[i], 9, kSecCin[i], ldk_of(kSecCin[i], kBf16), st));
      for (int j = 0; j < 4; ++j) TB_TRY(pack_w(P + pp.blk[i][j].w, w.wblk[i][j], kSecCh[i], 9, kSecCh[i], ldk_of(kSecCh[i], kBf16), st));
    }
    TB_TRY(pack_w(P + pp.fc_w, w.wfc, kFcOut, 121, 32, kFcIn, st));
    const T* xin = nullptr;
    for (int i = 0; i < kSections; ++i) {
      const int S = kSecS[i], So = kSecSo[i], ch = kSecCh[i], cin = kSecCin[i];
      const int64_t M = N * S * S, Mo = N * So * So;
      const int64_t ldk_in = ldk_of(cin, kBf16), ldk = ldk_of(ch, kBf16);
      if (i == 0) {
        TB_TRY(im2col3x3_u8_nchw<ColFirst>(frame, reinterpret_cast<ColFirst*>(w.col), N, 4, S, S, ldk_in, st));
        if constexpr (kBf16) {
          TB_TRY(conv_fwd(w.col, w.wfeat[0], w.s[0].P, M, ch, 36, ldk_in, P + pp.feat[0].b, 0, nullptr, 1.0f / 255.0f, ch, "feat_conv_fwd", st));
        } else {
          TB_TRY(conv_fwd_u8(reinterpret_cast<const uint8_t*>(w.col), w.wfeat[0], w.s[0].P, M, ch, 36, ldk_in, P + pp.feat[0].b,
                             "feat_conv_fwd", st));
        }
      } else {
        TB_TRY(im2col3x3<T>(xin, w.col, N, S, S, cin, ldk_in, 0, st));
        TB_TRY(conv_fwd(w.col, w.wfeat[i], w.s[i].P, M, ch, int64_t(cin) * 9, ldk_in, P + pp.feat[i].b, 0, nullptr, 1.0f, ch,
                        "feat_conv_fwd", st));
      }
      TB_TRY(maxpool3x3s2_fwd<T>(w.s[i].P, w.s[i].X0, w.s[i].arg, N, S, S, ch, st));
      const T* ins[4] = {w.s[i].X0, w.s[i].Y1, w.s[i].X1, w.s[i].Y2};
      T* outs[4] = {w.s[i].Y1, w.s[i].X1, w.s[i].Y2, w.s[i].X2};
      const T* adds[4] = {nullptr, w.s[i].X0, nullptr, w.s[i].X1};
      for (int j = 0; j < 4; ++j) {
        TB_TRY(im2col3x3<T>(ins[j], w.col, N, So, So, ch, ldk, 1, st));
        TB_TRY(conv_fwd(w.col, w.wblk[i][j], outs[j], Mo, ch, int64_t(ch) * 9, ldk, P + pp.blk[i][j].b, 0, adds[j], 1.0f, ch,
                        "res_conv_fwd", st));
      }
      xin = w.s[i].X2;
    }
    TB_TRY(relu_fwd<T>(w.s[2].X2, w.fcin, N * kFcIn, st));
    TB_TRY(fc_fwd(w.fcin, w.wfc, w.core_in, N, pp.core_in, P + pp.fc_b, st));
    TB_TRY(core_extras(w.core_in, pp.core_in, N, kFcOut, reward, nullptr, 0, st));
    if (use_lstm) {
      LstmParams lp;
      lp.w_ih[0] = P + pp.lstm[0]; lp.w_hh[0] = P + pp.lstm[1]; lp.b_ih[0] = P + pp.lstm[2]; lp.b_hh[0] = P + pp.lstm[3];
      lp.w_ih[1] = lp.w_hh[1] = lp.b_ih[1] = lp.b_hh[1] = nullptr;
      TB_TRY(lstm_forward(w.core_in, notdone, h0, c0, lp, T1, B, pp.core_in, kLstmH, 1, w.lstm, w.core_out, hN, cN, w.splitk,
                          kBf16 ? 1 : 0, st));
    }
    TB_TRY(heads_forward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.policy_b, P + pp.baseline_w, P + pp.baseline_b, N,
                         pp.core_out, A, policy_logits, baseline, st));
    return 0;
  }

  // one 3x3 conv backward: bias grad, weight grad (patch matrix recomputed from the stored input), and - if dx - the
  // input gradient dx = col2im(dY . W) * (relu_in ? x > 0 : 1) + addend
  static int conv_bwd(const T* x, bool relu_in, const T* dY, const T* Wp, float* dW, float* db, T* dx, const T* addend, int64_t N,
                      int S, int cin, int cout, ResWs<T>& w, cudaStream_t st) {
    const int64_t M = N * S * S, K = int64_t(cin) * 9, ldk = ldk_of(cin, kBf16);
    TB_TRY(colsum_t<T>(dY, db, M, cout, cout, w.colsum_scratch, st));
    TB_TRY(im2col3x3<T>(x, w.col, N, S, S, cin, ldk, relu_in ? 1 : 0, st));
    TB_TRY(conv_wgrad(dY, w.col, false, dW, M, cout, K, ldk, 9, cin, 1.0f, w.splitk, "res_conv_wgrad", st));
    if (dx) {
      TB_TRY(conv_dgrad(dY, Wp, w.dcol, M, cout, K, ldk, "res_conv_dgrad", st));
      TB_TRY(col2im3x3<T>(w.dcol, relu_in ? x : nullptr, addend, dx, N, S, S, cin, ldk, st));
    }
    return 0;
  }

  static int backward(const uint8_t* frame, const float* grad_logits, const float* grad_baseline, const float* notdone,
                      const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace, float* G, cudaStream_t st) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(A, use_lstm);
    ResWs<T> w = res_ws<T>(workspace, N, T1, B, A, use_lstm);
    // heads
    TB_TRY(heads_backward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.baseline_w, grad_logits, grad_baseline, N, pp.core_out,
                          A, w.dcore_out, pp.core_out, G + pp.policy_w, G + pp.policy_b, G + pp.baseline_w, G + pp.baseline_b,
                          w.splitk, st));
    if (use_lstm) {
      LstmParams lp; LstmGrads lg;
      lp.w_ih[0] = P + pp.lstm[0]; lp.w_hh[0] = P + pp.lstm[1]; lp.b_ih[0] = P + pp.lstm[2]; lp.b_hh[0] = P + pp.lstm[3];
      lg.w_ih[0] = G + pp.lstm[0]; lg.w_hh[0] = G + pp.lstm[1]; lg.b_ih[0] = G + pp.lstm[2]; lg.b_hh[0] = G + pp.lstm[3];
      lp.w_ih[1] = lp.w_hh[1] = lp.b_ih[1] = lp.b_hh[1] = nullptr;
      lg.w_ih[1] = lg.w_hh[1] = lg.b_ih[1] = lg.b_hh[1] = nullptr;
      TB_TRY(lstm_backward(w.dcore_out, w.core_in, notdone, lp, lg, T1, B, pp.core_in, kLstmH, 1, w.lstm, w.dcore_in, w.splitk,
                           w.colsum_scratch, kBf16 ? 1 : 0, st));
    }
    // fc
    TB_TRY(relu_mask_inplace(w.dcore_in, w.core_in, N, kFcOut, pp.core_in, pp.core_in, st));
    TB_TRY(colsum(w.dcore_in, G + pp.fc_b, N, kFcOut, pp.core_in, w.colsum_scratch, st));
    TB_TRY(convert_from_f32<T>(w.dcore_in, w.dfc, N, kFcOut, pp.core_in, kFcOut, st));
    TB_TRY(conv_wgrad(w.dfc, w.fcin, false, G + pp.fc_w, N, kFcOut, kFcIn, kFcIn, 121, 32, 1.0f, w.splitk, "fc_wgrad", st));
    TB_TRY(conv_dgrad(w.dfc, w.wfc, w.dfcin, N, kFcOut, kFcIn, kFcIn, "fc_dgrad", st));
    T* g0 = w.g[0]; T* g1 = w.g[1]; T* g2 = w.g[2];
    TB_TRY(relu_bwd<T>(w.s[2].X2, w.dfcin, g0, N * kFcIn, st));  // dL/dX2 of the last section
    for (int i = kSections - 1; i >= 0; --i) {
      const int S = kSecS[i], So = kSecSo[i], ch = kSecCh[i], cin = kSecCin[i];
      Sec<T>& s = w.s[i];
      // block 2: X2 = X1 + conv_b(relu(Y2)), Y2 = conv_a(relu(X1))
      TB_TRY(conv_bwd(s.Y2, true, g0, w.wblk[i][3], G + pp.blk[i][3].w, G + pp.blk[i][3].b, g1, nullptr, N, So, ch, ch, w, st));
      TB_TRY(conv_bwd(s.X1, true, g1, w.wblk[i][2], G + pp.blk[i][2].w, G + pp.blk[i][2].b, g2, g0, N, So, ch, ch, w, st));
      // block 1: X1 = X0 + conv_b(relu(Y1)), Y1 = conv_a(relu(X0))
      TB_TRY(conv_bwd(s.Y1, true, g2, w.wblk[i][1], G + pp.blk[i][1].w, G + pp.blk[i][1].b, g0, nullptr, N, So, ch, ch, w, st));
      TB_TRY(conv_bwd(s.X0, true, g0, w.wblk[i][0], G + pp.blk[i][0].w, G + pp.blk[i][0].b, g1, g2, N, So, ch, ch, w, st));
      TB_TRY(maxpool3x3s2_bwd<T>(s.arg, g1, g2, N, S, S, ch, st));   // g2 = dL/dP
      const int64_t M = N * S * S;
      if (i == 0) {
        const int64_t ldk_in = ldk_of(4, kBf16);
        TB_TRY(colsum_t<T>(g2, G + pp.feat[0].b, M, ch, ch, w.colsum_scratch, st));
        TB_TRY(im2col3x3_u8_nchw<ColFirst>(frame, reinterpret_cast<ColFirst*>(w.col), N, 4, S, S, ldk_in, st));
        TB_TRY(conv_wgrad(g2, w.col, !kBf16, G + pp.feat[0].w, M, ch, 36, ldk_in, 1, 1, 1.0f / 255.0f, w.splitk, "feat_conv_wgrad", st));
      } else {
        TB_TRY(conv_bwd(w.s[i - 1].X2, false, g2, w.wfeat[i], G + pp.feat[i].w, G + pp.feat[i].b, g0, nullptr, N, S, cin, ch, w, st));
      }
    }
    return 0;
  }
};


// ---- split-bf16 backend (precision 2) ----------------------------------------------------------------------
// The fp32 data flow of Impl<float> (fp32 NHWC activations, fp32 gradients, the same pool / ReLU kernels) with every
// contraction on the tensor cores in split-bf16: the 3x3 convolutions are shifted-window implicit GEMMs over hi / lo
// bf16 images, the fc GEMM reads hi / lo planes, products are hi.hi + hi.lo + lo.hi in fp32 (~2^-17 relative per
// product: fp32-grade, holds the 1e-4 parity contract that plain bf16 operands do not).
struct SplitImpl {
  using W = ResWs<float>;
  static int gemm_fwd(const __nv_bfloat16* a, int64_t a_lo, const __nv_bfloat16* b, int64_t b_lo, float* out, int64_t M, int cout,
                      int64_t K, int64_t ldk, const float* bias, const float* addend, float scale, int relu, int64_t ldc,
                      const char* tag, cudaStream_t st) {
    TcEpilogue te; te.C = out; te.ldc = ldc; te.bias = bias; te.relu = relu; te.addend32 = addend; te.ldadd = cout; te.scale = scale;
    te.a_lo = a_lo; te.b_lo = b_lo; te.tag = tag;
    return gemm_tc_bf16(a, b, M, cout, K, ldk, ldk, te, st);
  }
  // dW[cout, K] (fp32, un-packed by the split-K reduce) = scale * dY^T . col
  static int gemm_wgrad(const __nv_bfloat16* dy, int64_t dy_lo, const __nv_bfloat16* col, int64_t col_lo, float* dW, int64_t M,
                        int cout, int64_t K, int64_t ldk, int permP, int permQ, float scale, float* scratch, const char* tag,
                        cudaStream_t st) {
    TcEpilogue te; te.C = dW; te.ldc = K; te.permP = permP; te.permQ = permQ; te.scale = scale; te.a_lo = dy_lo; te.b_lo = col_lo;
    te.tag = tag;
    return gemm_tc_bf16_ex(dy, col, cout, K, M, cout, ldk, true, true, te, splits_tc(cout, K, M), scratch, st);
  }
  // shifted-window implicit GEMM: x fp32 NHWC -> padded planar split-bf16 image xp (kept for the weight gradient) -> out fp32
  // x == nullptr: the previous conv's epilogue already wrote this conv's input image into xp.  emit: the NEXT conv's input
  // image (this conv's output, through ReLU if emit_relu), written by the epilogue.
  static int conv_impl(const float* x, int relu_in, __nv_bfloat16* xp, int64_t xp_lo, const float* Wsrc, __nv_bfloat16* wi, int64_t wi_lo,
                       float* out, int64_t N, int S, int cin, int cout, const float* bias, const float* addend, __nv_bfloat16* emit,
                       int64_t emit_lo, int emit_relu, const char* tag, cudaStream_t st) {
    TB_TRY(sw_pack_weights(Wsrc, wi, cout, cin, 0, st));
    if (x) TB_TRY(sw_pad_split(x, xp, xp_lo, N, S, S, cin, relu_in, st));
    SwEpilogue ep; ep.bias = bias; ep.addend = addend; ep.emit = emit; ep.emit_lo = emit_lo; ep.emit_relu = emit_relu; ep.tag = tag;
    return sw_conv_fwd(xp, xp_lo, wi, out, N, S, S, cin, cout, ep, st);
  }

  static int forward(const uint8_t* frame, const float* reward, const float* notdone, const float* h0, const float* c0,
                     const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace, float* policy_logits,
                     float* baseline, float* hN, float* cN, cudaStream_t st) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(A, use_lstm);
    W w = res_ws<float>(workspace, N, T1, B, A, use_lstm, true);
    TB_TRY(pack_weights_bf16(P + pp.fc_w, w.wb_fc, kFcOut, 121, 32, kFcIn, st, w.wb_fc_lo));
    for (int i = 0; i < kSections; ++i) {
      const int S = kSecS[i], So = kSecSo[i], ch = kSecCh[i], cin = kSecCin[i];
      if (i == 0) {
        // the first conv through the same kernels: frame pixels (exact in bf16) as a 16-channel image, 1/255 in the epilogue
        TB_TRY(sw_pack_weights(P + pp.feat[0].w, w.wi_feat[0], ch, 16, 0, st, 4));
        TB_TRY(sw_frames_u8(frame, w.xp_feat[0], w.xp_feat_lo[0], N, 4, S, S, st));
        SwEpilogue ep; ep.scale = 1.0f / 255.0f; ep.bias = P + pp.feat[0].b; ep.tag = "feat_conv_fwd";
        TB_TRY(sw_conv_fwd(w.xp_feat[0], w.xp_feat_lo[0], w.wi_feat[0], w.s[0].P, N, S, S, 16, ch, ep, st));
      } else {
        // (its input image was written by the epilogue of the previous section's last conv)
        TB_TRY(conv_impl(nullptr, 0, w.xp_feat[i], w.xp_feat_lo[i], P + pp.feat[i].w, w.wi_feat[i], w.wi_feat_lo[i], w.s[i].P, N, S, cin, ch,
                         P + pp.feat[i].b, nullptr, nullptr, 0, 0, "feat_conv_fwd", st));
      }
      TB_TRY(maxpool3x3s2_fwd<float>(w.s[i].P, w.s[i].X0, w.s[i].arg, N, S, S, ch, st));
      float* outs[4] = {w.s[i].Y1, w.s[i].X1, w.s[i].Y2, w.s[i].X2};
      const float* adds[4] = {nullptr, w.s[i].X0, nullptr, w.s[i].X1};
      for (int j = 0; j < 4; ++j) {
        // conv j's epilogue writes relu(output) as conv j+1's input image; the section's last conv writes the next
        // section's feat-conv input (no ReLU there)
        __nv_bfloat16* emit = j < 3 ? w.xp_blk[i][j + 1] : (i + 1 < kSections ? w.xp_feat[i + 1] : nullptr);
        const int64_t emit_lo = j < 3 ? w.xp_blk_lo[i][j + 1] : (i + 1 < kSections ? w.xp_feat_lo[i + 1] : 0);
        TB_TRY(conv_impl(j == 0 ? w.s[i].X0 : nullptr, 1, w.xp_blk[i][j], w.xp_blk_lo[i][j], P + pp.blk[i][j].w, w.wi_blk[i][j],
                         w.wi_blk_lo[i][j], outs[j], N, So, ch, ch, P + pp.blk[i][j].b, adds[j], emit, emit_lo, j < 3 ? 1 : 0,
                         "res_conv_fwd", st));
      }
    }
    TB_TRY(relu_fwd<float>(w.s[2].X2, w.fcin, N * kFcIn, st));
    TB_TRY(f32_to_bf16(w.fcin, w.fcb, N, kFcIn, kFcIn, kFcIn, st, w.fcb_lo));
    TB_TRY(gemm_fwd(w.fcb, w.fcb_lo, w.wb_fc, w.wb_fc_lo, w.core_in, N, kFcOut, kFcIn, kFcIn, P + pp.fc_b, nullptr, 1.0f, 1,
                    pp.core_in, "fc_fwd", st));
    TB_TRY(core_extras(w.core_in, pp.core_in, N, kFcOut, reward, nullptr, 0, st));
    if (use_lstm) {
      LstmParams lp;
      lp.w_ih[0] = P + pp.lstm[0]; lp.w_hh[0] = P + pp.lstm[1]; lp.b_ih[0] = P + pp.lstm[2]; lp.b_hh[0] = P + pp.lstm[3];
      lp.w_ih[1] = lp.w_hh[1] = lp.b_ih[1] = lp.b_hh[1] = nullptr;
      TB_TRY(lstm_forward(w.core_in, notdone, h0, c0, lp, T1, B, pp.core_in, kLstmH, 1, w.lstm, w.core_out, hN, cN, w.splitk, 2, st));
    }
    TB_TRY(heads_forward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.policy_b, P + pp.baseline_w, P + pp.baseline_b, N,
                         pp.core_out, A, policy_logits, baseline, st));
    return 0;
  }

  // one 3x3 conv backward on the shifted-window kernels: dY -> padded planar image (+ bias gradient in the same pass);
  // weight gradient from that image and the input image kept by the forward pass; input gradient = the SAME convolution
  // kernel over the dY image with flipped / transposed weights, ReLU mask and skip gradient in its epilogue
  static int conv_bwd_impl(const float* x, bool relu_in, const float* dY, __nv_bfloat16* dyimg, int64_t dyimg_lo, const float* Wsrc,
                           const __nv_bfloat16* xp, int64_t xp_lo, __nv_bfloat16* wd, int64_t wd_lo, float* dW, float* db, float* dx,
                           const float* addend, __nv_bfloat16* emit, int64_t emit_lo, float* emit_db, int64_t N, int S, int cin, int cout,
                           W& w, const char* wtag, cudaStream_t st) {
    // dY == nullptr: dyimg (and db) were already produced by the previous kernel's epilogue / the fused max-pool backward
    if (dY) TB_TRY(sw_pad_split_colsum(dY, dyimg, dyimg_lo, N, S, S, cout, db, w.splitk, w.splitk_floats, st));
    TB_TRY(sw_conv_wgrad(dyimg, dyimg_lo, xp, xp_lo, dW, N, S, S, cin, cout, w.splitk, w.splitk_floats, wtag, st));
    if (dx) {
      TB_TRY(sw_pack_weights(Wsrc, wd, cout, cin, 1, st));
      SwEpilogue ep; ep.mask = relu_in ? x : nullptr; ep.addend = addend; ep.tag = "res_conv_dgrad";
      // emit: dx is the dY of the conv that runs next in this backward pass - its image and (through the column sums) its
      // bias gradient come out of this epilogue
      const int64_t rows = sw_csum_rows(N, S, S);
      if (emit) {
        TB_REQUIRE((rows + 128) * cin <= w.splitk_floats, "resnet: column-sum scratch too small");
        ep.emit = emit; ep.emit_lo = emit_lo; ep.csum = w.splitk;
      }
      TB_TRY(sw_conv_fwd(dyimg, dyimg_lo, wd, dx, N, S, S, cout, cin, ep, st));
      if (emit) TB_TRY(sw_csum_reduce(w.splitk, rows, cin, emit_db, st));
    }
    return 0;
  }

  static int backward(const uint8_t* frame, const float* grad_logits, const float* grad_baseline, const float* notdone,
                      const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace, float* G, cudaStream_t st) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(A, use_lstm);
    W w = res_ws<float>(workspace, N, T1, B, A, use_lstm, true);
    TB_TRY(heads_backward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.baseline_w, grad_logits, grad_baseline, N, pp.core_out,
                          A, w.dcore_out, pp.core_out, G + pp.policy_w, G + pp.policy_b, G + pp.baseline_w, G + pp.baseline_b,
                          w.splitk, st));
    if (use_lstm) {
      LstmParams lp; LstmGrads lg;
      lp.w_ih[0] = P + pp.lstm[0]; lp.w_hh[0] = P + pp.lstm[1]; lp.b_ih[0] = P + pp.lstm[2]; lp.b_hh[0] = P + pp.lstm[3];
      lg.w_ih[0] = G + pp.lstm[0]; lg.w_hh[0] = G + pp.lstm[1]; lg.b_ih[0] = G + pp.lstm[2]; lg.b_hh[0] = G + pp.lstm[3];
      lp.w_ih[1] = lp.w_hh[1] = lp.b_ih[1] = lp.b_hh[1] = nullptr;
      lg.w_ih[1] = lg.w_hh[1] = lg.b_ih[1] = lg.b_hh[1] = nullptr;
      TB_TRY(lstm_backward(w.dcore_out, w.core_in, notdone, lp, lg, T1, B, pp.core_in, kLstmH, 1, w.lstm, w.dcore_in, w.splitk,
                           w.colsum_scratch, 2, st));
    }
    TB_TRY(relu_mask_inplace(w.dcore_in, w.core_in, N, kFcOut, pp.core_in, pp.core_in, st));
    TB_TRY(colsum(w.dcore_in, G + pp.fc_b, N, kFcOut, pp.core_in, w.colsum_scratch, st));
    TB_TRY(f32_to_bf16(w.dcore_in, w.dfcb, N, kFcOut, pp.core_in, kFcOut, st, w.dfcb_lo));
    // (fcb still holds relu(X2) as hi / lo planes from the forward pass)
    TB_TRY(gemm_wgrad(w.dfcb, w.dfcb_lo, w.fcb, w.fcb_lo, G + pp.fc_w, N, kFcOut, kFcIn, kFcIn, 121, 32, 1.0f, w.splitk, "fc_wgrad", st));
    {
      TcEpilogue te; te.C = w.dfcin; te.ldc = kFcIn; te.a_lo = w.dfcb_lo; te.b_lo = w.wb_fc_lo; te.tag = "fc_dgrad";
      TB_TRY(gemm_tc_bf16_ex(w.dfcb, w.wb_fc, N, kFcIn, kFcOut, kFcOut, kFcIn, false, true, te, 1, nullptr, st));
    }
    float* g0 = w.g[0]; float* g1 = w.g[1]; float* g2 = w.g[2];
    TB_TRY(relu_bwd<float>(w.s[2].X2, w.dfcin, g0, N * kFcIn, st));
    __nv_bfloat16* dyi[2] = {w.dyp, w.dyp2};   // dY images: dyi[dsel] is the one the next kernel reads
    const int64_t dyi_lo[2] = {w.dyp_lo, w.dyp2_lo};
    int dsel = 0;
    for (int i = kSections - 1; i >= 0; --i) {
      const int S = kSecS[i], So = kSecSo[i], ch = kSecCh[i], cin = kSecCin[i];
      Sec<float>& s = w.s[i];
      const float* xs[4] = {s.X0, s.Y1, s.X1, s.Y2};
      const float* dys[4] = {g0, g2, g1, g0};       // dL/d(conv output) of r1a, r1b, r2a, r2b
      float* dxs[4] = {g1, g0, g2, g1};
      const float* skip[4] = {g2, nullptr, g0, nullptr};
      for (int j = 3; j >= 0; --j) {
        // the dY image of conv j: written by the previous kernel's epilogue, except for the very first conv of the pass
        const bool ready = !(i == kSections - 1 && j == 3);
        __nv_bfloat16* cur = dyi[dsel]; const int64_t cur_lo = dyi_lo[dsel];
        __nv_bfloat16* nxt = j > 0 ? dyi[dsel ^ 1] : nullptr;   // conv j's dx is conv j-1's dY (j = 0: feeds the max-pool backward)
        TB_TRY(conv_bwd_impl(xs[j], true, ready ? nullptr : dys[j], cur, cur_lo, P + pp.blk[i][j].w, w.xp_blk[i][j], w.xp_blk_lo[i][j],
                             w.wd_blk[i][j], w.wd_blk_lo[i][j], G + pp.blk[i][j].w, G + pp.blk[i][j].b, dxs[j], skip[j], nxt,
                             dyi_lo[dsel ^ 1], j > 0 ? G + pp.blk[i][j - 1].b : nullptr, N, So, ch, ch, w, "res_conv_wgrad", st));
        if (nxt) dsel ^= 1;
      }
      // dL/dP (the feat conv's output gradient) is consumed only as that conv's dY image + bias gradient: the max-pool
      // backward gathers straight into the image (never materialised in fp32)
      TB_TRY(sw_pool_bwd_image_colsum(s.arg, g1, dyi[dsel], dyi_lo[dsel], N, S, S, ch, G + pp.feat[i].b, w.splitk, w.splitk_floats, st));
      if (i == 0) {
        TB_TRY(sw_conv_wgrad(dyi[dsel], dyi_lo[dsel], w.xp_feat[0], w.xp_feat_lo[0], G + pp.feat[0].w, N, S, S, 16, ch, w.splitk,
                             w.splitk_floats, "feat_conv_wgrad", st, 1.0f / 255.0f, 4));
      } else {
        // its dx = dL/dX2 of section i-1 = the dY of that section's last conv: emitted as the image + bias gradient that
        // conv's backward starts from
        TB_TRY(conv_bwd_impl(w.s[i - 1].X2, false, nullptr, dyi[dsel], dyi_lo[dsel], P + pp.feat[i].w, w.xp_feat[i], w.xp_feat_lo[i],
                             w.wd_feat[i], w.wd_feat_lo[i], G + pp.feat[i].w, G + pp.feat[i].b, g0, nullptr, dyi[dsel ^ 1], dyi_lo[dsel ^ 1],
                             G + pp.blk[i - 1][3].b, N, S, cin, ch, w, "res_conv_wgrad", st));
        dsel ^= 1;
      }
    }
    return 0;
  }
};

}  // namespace
}  // namespace tb

using namespace tb;

extern "C" {

int64_t tb_resnet_param_count(int num_actions, int use_lstm) { return res_params(num_actions, use_lstm).total; }

size_t tb_resnet_workspace_bytes(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision) {
  if (precision == 2) return res_ws<float>(nullptr, T1 * B, T1, B, num_actions, use_lstm, true).bytes;
  return precision ? res_ws<__nv_bfloat16>(nullptr, T1 * B, T1, B, num_actions, use_lstm).bytes
                   : res_ws<float>(nullptr, T1 * B, T1, B, num_actions, use_lstm).bytes;
}

int tb_resnet_forward(const uint8_t* frame, const float* reward, const float* notdone, const float* h0, const float* c0,
                      const float* params, int64_t T1, int64_t B, int num_actions, int use_lstm, int precision, void* workspace,
                      float* policy_logits, float* baseline, float* hN, float* cN, void* stream) {
  TB_REQUIRE(T1 >= 1 && B >= 1 && num_actions >= 1, "resnet_forward: bad sizes");
  TB_REQUIRE(frame && reward && params && workspace && policy_logits && baseline, "resnet_forward: null pointer");
  TB_REQUIRE(!use_lstm || (notdone && h0 && c0 && hN && cN), "resnet_forward: LSTM needs notdone/h0/c0/hN/cN");
  TB_REQUIRE(precision >= 0 && precision <= 2, "resnet_forward: precision must be 0 (fp32), 1 (bf16) or 2 (split-bf16)");
  if (precision == 2)
    return SplitImpl::forward(frame, reward, notdone, h0, c0, params, T1, B, num_actions, use_lstm, workspace, policy_logits,
                              baseline, hN, cN, (cudaStream_t)stream);
  if (precision)
    return Impl<__nv_bfloat16>::forward(frame, reward, notdone, h0, c0, params, T1, B, num_actions, use_lstm, workspace,
                                        policy_logits, baseline, hN, cN, (cudaStream_t)stream);
  return Impl<float>::forward(frame, reward, notdone, h0, c0, params, T1, B, num_actions, use_lstm, workspace, policy_logits,
                              baseline, hN, cN, (cudaStream_t)stream);
}

int tb_resnet_backward(const uint8_t* frame, const float* grad_logits, const float* grad_baseline, const float* notdone,
                       const float* params, int64_t T1, int64_t B, int num_actions, int use_lstm, int precision,
                       void* workspace, float* grads, void* stream) {
  TB_REQUIRE(T1 >= 1 && B >= 1 && num_actions >= 1, "resnet_backward: bad sizes");
  TB_REQUIRE(frame && grad_logits && grad_baseline && params && workspace && grads, "resnet_backward: null pointer");
  TB_REQUIRE(!use_lstm || notdone, "resnet_backward: LSTM needs notdone");
  TB_REQUIRE(precision >= 0 && precision <= 2, "resnet_backward: precision must be 0, 1 or 2");
  if (precision == 2)
    return SplitImpl::backward(frame, grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm, workspace,
                               grads, (cudaStream_t)stream);
  if (precision)
    return Impl<__nv_bfloat16>::backward(frame, grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm,
                                         workspace, grads, (cudaStream_t)stream);
  return Impl<float>::backward(frame, grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm, workspace,
                               grads, (cudaStream_t)stream);
}

}  // extern "C"
