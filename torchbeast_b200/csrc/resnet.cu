// IMPALA "deep" ResNet (polybeast_learner.Net) forward / backward for the learner, behind the C ABI.
//
// Replaces /root/reference/torchbeast/polybeast_learner.py:214-266 (Net.forward) and its autograd graph:
//   for ch in (16, 32, 32):  x = maxpool3x3/2(conv3x3(x));  x += conv(relu(conv(relu(x))));  x += conv(relu(conv(relu(x))))
//   x = relu(x) -> fc 3872->256 -> relu -> cat[x, clip(reward)] -> [LSTM(257->256)] -> policy / baseline
// (3872 = 32 * 11 * 11 for u8 [4, 84, 84] frames; the entry points take other observation shapes, see ResGeom)
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
#include "restack.cuh"

namespace tb {

namespace {

constexpr int kSections = 3;
constexpr int kDefaultCh[kSections] = {16, 32, 32};   // the IMPALA paper's widths
constexpr int kFcOut = 256;
constexpr int kLstmH = 256;
constexpr int64_t kScratchFloats = int64_t(8) << 20;

// Supported observations u8 [C, H, W] (tb_resnet_obs_range): C frame channels (the first conv's input image has 16); H
// large enough that the last section's pooled output is still 3 rows high (17 -> 9 -> 5 -> 3, the smallest image the
// shifted-window kernels take); W large enough that it is still 5 wide (33 -> 17 -> 9 -> 5: narrower rows would let the
// weight gradient's last pixel step of a frame run past the zero run behind it, see sw_conv_trainable); both at most the
// widest row the kernels take (W + 2 <= 128 padded pixels), H bounded the same way
constexpr int kObsMaxC = 16;
constexpr int kObsMinH = 17;
constexpr int kObsMinW = 33;
constexpr int kObsMaxHW = 126;

// Section widths (tb_resnet_supported): each of 16, 32 or 64 channels, in any combination.  The shifted-window
// kernels take 16 / 32 / 64 channels on either side of a conv; 64-channel convs run at W <= 63 (any 64-wide section after
// the first, or the residual blocks of a 64-wide first section) or 16 -> 64 at W <= 126 (the first conv), which all fit.
constexpr int kWidths[3] = {16, 32, 64};

// Net geometry: section i has ch[i] channels; its feat conv runs at H[i] x W[i] (H[0] x W[0] = the frame), its max-pool
// (3, 2, 1) leaves ceil(H[i] / 2) x ceil(W[i] / 2) = H[i+1] x W[i+1]; the fc reads the last section's ch[2] x H[3] x W[3]
// output
struct ResGeom {
  int C, H[kSections + 1], W[kSections + 1], ch[kSections];
  int cin(int i) const { return i == 0 ? C : ch[i - 1]; }
  int fc_hw() const { return H[kSections] * W[kSections]; }
  int fc_in() const { return ch[kSections - 1] * fc_hw(); }
};

ResGeom res_geom(int C, int H, int W, const int* ch) {
  ResGeom g;
  g.C = C; g.H[0] = H; g.W[0] = W;
  for (int i = 0; i < kSections; ++i) { g.H[i + 1] = (g.H[i] + 1) / 2; g.W[i + 1] = (g.W[i] + 1) / 2; g.ch[i] = ch[i]; }
  return g;
}

// 0, or 1 with tb_last_error set: the range above, the widths, and on the split-bf16 backend every conv of the geometry
// on the shifted-window kernels (the other backends' im2col / GEMM kernels take any size)
int res_geom_check(int C, int H, int W, const int* ch, int precision, const char* who) {
  TB_REQUIRE(C >= 1 && C <= kObsMaxC, "%s: observation channels %d outside [1, %d]", who, C, kObsMaxC);
  TB_REQUIRE(H >= kObsMinH && H <= kObsMaxHW && W >= kObsMinW && W <= kObsMaxHW,
             "%s: observation %d x %d outside [%d, %d] x [%d, %d]", who, H, W, kObsMinH, kObsMaxHW, kObsMinW, kObsMaxHW);
  for (int i = 0; i < kSections; ++i)
    TB_REQUIRE(ch[i] == kWidths[0] || ch[i] == kWidths[1] || ch[i] == kWidths[2],
               "%s: section %d has %d channels; each section takes 16, 32 or 64", who, i, ch[i]);
  TB_REQUIRE(precision >= 0 && precision <= 2, "%s: precision must be 0 (fp32), 1 (bf16) or 2 (split-bf16)", who);
  if (precision == 2) {
    const ResGeom g = res_geom(C, H, W, ch);
    for (int i = 0; i < kSections; ++i) {
      const int c = g.ch[i], cin = i == 0 ? 16 : g.cin(i);
      // (the first conv's input gradient is never formed)
      TB_REQUIRE(sw_conv_trainable(g.H[i], g.W[i], cin, c, i > 0) && sw_conv_trainable(g.H[i + 1], g.W[i + 1], c, c),
                 "%s: section %d (%d x %d) does not fit the shifted-window conv kernels", who, i, g.H[i], g.W[i]);
    }
  }
  return 0;
}

struct ConvP { int64_t w, b; };
struct ResParams {
  ConvP feat[kSections], blk[kSections][4];  // blk: r1a, r1b, r2a, r2b
  int64_t fc_w, fc_b, lstm[4], policy_w, policy_b, baseline_w, baseline_b, total;
  int core_in, core_out;
};

ResParams res_params(const ResGeom& g, int A, int use_lstm, int V = 1) {  // V: value outputs
  ResParams p;
  int64_t o = 0;
  auto take = [&](int64_t n) { int64_t r = o; o += n; return r; };
  for (int i = 0; i < kSections; ++i) { p.feat[i].w = take(int64_t(g.ch[i]) * g.cin(i) * 9); p.feat[i].b = take(g.ch[i]); }
  for (int blk = 0; blk < 2; ++blk)     // resnet1.{0,1,2}.{1,3} then resnet2.{0,1,2}.{1,3}
    for (int i = 0; i < kSections; ++i)
      for (int j = 0; j < 2; ++j) {
        p.blk[i][blk * 2 + j].w = take(int64_t(g.ch[i]) * g.ch[i] * 9);
        p.blk[i][blk * 2 + j].b = take(g.ch[i]);
      }
  p.fc_w = take(int64_t(kFcOut) * g.fc_in()); p.fc_b = take(kFcOut);
  p.core_in = kFcOut + 1;
  p.core_out = use_lstm ? kLstmH : p.core_in;
  for (int k = 0; k < 4; ++k) p.lstm[k] = -1;
  if (use_lstm) {
    p.lstm[0] = take(int64_t(4) * kLstmH * p.core_in); p.lstm[1] = take(int64_t(4) * kLstmH * kLstmH);
    p.lstm[2] = take(4 * kLstmH); p.lstm[3] = take(4 * kLstmH);
  }
  p.policy_w = take(int64_t(A) * p.core_out); p.policy_b = take(A);
  p.baseline_w = take(int64_t(V) * p.core_out); p.baseline_b = take(V);
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
ResWs<T> res_ws(const ResGeom& g, void* base, int64_t N, int64_t T1, int64_t B, int A, int use_lstm, bool split = false) {
  constexpr bool kBf16 = !std::is_same<T, float>::value;
  ResWs<T> w;
  size_t off = 0;
  auto take = [&](size_t nbytes) { void* p = base ? static_cast<char*>(base) + off : nullptr; off += (nbytes + 255) & ~size_t(255); return p; };
  auto takeT = [&](int64_t n) { return static_cast<T*>(take(size_t(n) * sizeof(T))); };
  auto takef = [&](int64_t n) { return static_cast<float*>(take(size_t(n) * sizeof(float))); };
  const ResParams pp = res_params(g, A, use_lstm);
  const int64_t fc_in = g.fc_in();
  int64_t maxact = 0;
  for (int i = 0; i < kSections; ++i) {
    const int64_t big = N * g.H[i] * g.W[i] * g.ch[i], small = N * g.H[i + 1] * g.W[i + 1] * g.ch[i];
    w.s[i].P = takeT(big); w.s[i].X0 = takeT(small); w.s[i].Y1 = takeT(small); w.s[i].X1 = takeT(small);
    w.s[i].Y2 = takeT(small); w.s[i].X2 = takeT(small);
    w.s[i].arg = static_cast<uint8_t*>(take(size_t(small)));
    if (big > maxact) maxact = big;
  }
  w.fcin = takeT(N * fc_in); w.dfc = takeT(N * kFcOut); w.dfcin = takeT(N * fc_in);
  for (int k = 0; k < 3; ++k) w.g[k] = takeT(maxact);
  int64_t maxcol = 0;
  for (int i = 0; i < kSections; ++i) {
    const int64_t a = N * g.H[i] * g.W[i] * ldk_of(g.cin(i), kBf16), b = N * g.H[i + 1] * g.W[i + 1] * ldk_of(g.ch[i], kBf16);
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
    w.fcb = takeh(N * fc_in, w.fcb_lo);
    w.dfcb = takeh(N * kFcOut, w.dfcb_lo);
    w.wb_fc = takeh(int64_t(kFcOut) * fc_in, w.wb_fc_lo);
    for (int i = 0; i < kSections; ++i) {
      if (i > 0) w.wd_feat[i] = takeh(int64_t(g.cin(i)) * 9 * g.ch[i], w.wd_feat_lo[i]);
      for (int j = 0; j < 4; ++j) w.wd_blk[i][j] = takeh(int64_t(g.ch[i]) * 9 * g.ch[i], w.wd_blk_lo[i][j]);
    }
    int64_t maxp = 0;
    for (int i = 0; i < kSections; ++i) {
      {   // (the frame channels of the first conv are padded to 16)
        const int cin16 = i == 0 ? 16 : g.cin(i);
        w.xp_feat[i] = takeh(sw_image_elems(N, g.H[i], g.W[i], cin16), w.xp_feat_lo[i]);
        w.wi_feat[i] = takeh(sw_weight_elems(g.ch[i], cin16) / 2, w.wi_feat_lo[i]);
        const int64_t e = sw_image_elems(N, g.H[i], g.W[i], g.ch[i]);
        if (e > maxp) maxp = e;
      }
      for (int j = 0; j < 4; ++j) {
        w.xp_blk[i][j] = takeh(sw_image_elems(N, g.H[i + 1], g.W[i + 1], g.ch[i]), w.xp_blk_lo[i][j]);
        w.wi_blk[i][j] = takeh(sw_weight_elems(g.ch[i], g.ch[i]) / 2, w.wi_blk_lo[i][j]);
      }
      const int64_t e = sw_image_elems(N, g.H[i + 1], g.W[i + 1], g.ch[i]);
      if (e > maxp) maxp = e;
    }
    w.dyp = takeh(maxp, w.dyp_lo);     // dY images ping-pong: a conv's input-gradient epilogue writes the next conv's dY image
    w.dyp2 = takeh(maxp, w.dyp2_lo);
  }
  for (int i = 0; i < kSections; ++i) {
    w.wfeat[i] = takeT(int64_t(g.ch[i]) * ldk_of(g.cin(i), kBf16));
    for (int j = 0; j < 4; ++j) w.wblk[i][j] = takeT(int64_t(g.ch[i]) * ldk_of(g.ch[i], kBf16));
  }
  w.wfc = takeT(int64_t(kFcOut) * fc_in);
  w.core_in = takef(N * pp.core_in);
  w.core_out = use_lstm ? takef(N * pp.core_out) : w.core_in;
  w.dcore_out = takef(N * (pp.core_in > pp.core_out ? pp.core_in : pp.core_out));
  w.dcore_in = use_lstm ? takef(N * pp.core_in) : w.dcore_out;
  // split-K partials need kScratchFloats; the split backend's fixed-order column-sum partials need a row of C floats per
  // block of the pad-split / max-pool-backward passes and per (tile, epilogue warp) of a dgrad conv that emits the next dY
  // image and its bias gradient, plus the second-level slices - about 1000 floats per frame at 84 x 84
  w.splitk_floats = kScratchFloats;
  auto need = [&](int64_t f) { if (f > w.splitk_floats) w.splitk_floats = f; };
  // the heads' weight-gradient partials (the backward checks them against this size), for any number of value outputs
  need(heads_scratch_floats(N, pp.core_out, A, kHeadsMaxValues));
  if (split) {
    for (int i = 0; i < kSections; ++i) {
      const int ch = g.ch[i];
      need(sw_colsum_scratch_floats(N, g.H[i], g.W[i], ch));           // max-pool backward -> the feat conv's dY image
      need(sw_colsum_scratch_floats(N, g.H[i + 1], g.W[i + 1], ch));   // pad-split of a residual conv's dY
      need((sw_csum_rows(N, g.H[i + 1], g.W[i + 1]) + 128) * ch);      // residual dgrad emits the previous conv's dY
      if (i > 0) need((sw_csum_rows(N, g.H[i], g.W[i]) + 128) * g.cin(i));   // feat dgrad emits section i-1's last dY
      // the weight gradients' per-CTA partials (at most kNumSMs CTAs, sw_conv_wgrad)
      need(int64_t(kNumSMs) * ch * 9 * (i == 0 ? 16 : g.cin(i)));
      need(int64_t(kNumSMs) * ch * 9 * ch);
    }
  }
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
  const int s = simt_splits(cout, K, M, kScratchFloats, 128);
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
int fc_fwd(const float* x, const float* W, float* core, int64_t N, int64_t K, int64_t ldc, const float* bias, cudaStream_t st) {
  GemmEpilogue ep; ep.bias = bias; ep.relu = 1; ep.tag = "fc_fwd";
  return gemm_simt<float, float, false, true>(x, W, core, N, kFcOut, K, K, K, ldc, ep, 1, nullptr, st);
}
int fc_fwd(const __nv_bfloat16* x, const __nv_bfloat16* W, float* core, int64_t N, int64_t K, int64_t ldc, const float* bias,
           cudaStream_t st) {
  TcEpilogue te; te.C = core; te.ldc = ldc; te.bias = bias; te.relu = 1; te.tag = "fc_fwd";
  return gemm_tc_bf16(x, W, N, kFcOut, K, K, K, te, st);
}

template <typename T>
struct Impl {
  static constexpr bool kBf16 = !std::is_same<T, float>::value;
  using ColFirst = typename std::conditional<kBf16, __nv_bfloat16, uint8_t>::type;

  static int forward(const ResGeom& g, const uint8_t* frame, const float* reward, const float* notdone, const float* h0,
                     const float* c0, const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace,
                     float* policy_logits, float* baseline, float* hN, float* cN, cudaStream_t st, int V = 1) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(g, A, use_lstm, V);
    ResWs<T> w = res_ws<T>(g, workspace, N, T1, B, A, use_lstm);
    const int64_t fc_in = g.fc_in(), k_first = int64_t(g.C) * 9;
    // weight pack: [o, c, kh, kw] -> [o, (kh,kw), c]; first conv keeps (c,kh,kw); fc: [o, c, (h,w)] -> [o, (h,w), c]
    TB_TRY(pack_w(P + pp.feat[0].w, w.wfeat[0], g.ch[0], 1, int(k_first), ldk_of(g.C, kBf16), st));
    for (int i = 0; i < kSections; ++i) {
      if (i > 0) TB_TRY(pack_w(P + pp.feat[i].w, w.wfeat[i], g.ch[i], 9, g.cin(i), ldk_of(g.cin(i), kBf16), st));
      for (int j = 0; j < 4; ++j) TB_TRY(pack_w(P + pp.blk[i][j].w, w.wblk[i][j], g.ch[i], 9, g.ch[i], ldk_of(g.ch[i], kBf16), st));
    }
    TB_TRY(pack_w(P + pp.fc_w, w.wfc, kFcOut, g.fc_hw(), g.ch[kSections - 1], fc_in, st));
    const T* xin = nullptr;
    for (int i = 0; i < kSections; ++i) {
      const int H = g.H[i], W = g.W[i], Ho = g.H[i + 1], Wo = g.W[i + 1], ch = g.ch[i], cin = g.cin(i);
      const int64_t M = N * H * W, Mo = N * Ho * Wo;
      const int64_t ldk_in = ldk_of(cin, kBf16), ldk = ldk_of(ch, kBf16);
      if (i == 0) {
        TB_TRY(im2col3x3_u8_nchw<ColFirst>(frame, reinterpret_cast<ColFirst*>(w.col), N, g.C, H, W, ldk_in, st));
        if constexpr (kBf16) {
          TB_TRY(conv_fwd(w.col, w.wfeat[0], w.s[0].P, M, ch, k_first, ldk_in, P + pp.feat[0].b, 0, nullptr, 1.0f / 255.0f, ch,
                          "feat_conv_fwd", st));
        } else {
          TB_TRY(conv_fwd_u8(reinterpret_cast<const uint8_t*>(w.col), w.wfeat[0], w.s[0].P, M, ch, k_first, ldk_in, P + pp.feat[0].b,
                             "feat_conv_fwd", st));
        }
      } else {
        TB_TRY(im2col3x3<T>(xin, w.col, N, H, W, cin, ldk_in, 0, st));
        TB_TRY(conv_fwd(w.col, w.wfeat[i], w.s[i].P, M, ch, int64_t(cin) * 9, ldk_in, P + pp.feat[i].b, 0, nullptr, 1.0f, ch,
                        "feat_conv_fwd", st));
      }
      TB_TRY(maxpool3x3s2_fwd<T>(w.s[i].P, w.s[i].X0, w.s[i].arg, N, H, W, ch, st));
      const T* ins[4] = {w.s[i].X0, w.s[i].Y1, w.s[i].X1, w.s[i].Y2};
      T* outs[4] = {w.s[i].Y1, w.s[i].X1, w.s[i].Y2, w.s[i].X2};
      const T* adds[4] = {nullptr, w.s[i].X0, nullptr, w.s[i].X1};
      for (int j = 0; j < 4; ++j) {
        TB_TRY(im2col3x3<T>(ins[j], w.col, N, Ho, Wo, ch, ldk, 1, st));
        TB_TRY(conv_fwd(w.col, w.wblk[i][j], outs[j], Mo, ch, int64_t(ch) * 9, ldk, P + pp.blk[i][j].b, 0, adds[j], 1.0f, ch,
                        "res_conv_fwd", st));
      }
      xin = w.s[i].X2;
    }
    TB_TRY(relu_fwd<T>(w.s[2].X2, w.fcin, N * fc_in, st));
    TB_TRY(fc_fwd(w.fcin, w.wfc, w.core_in, N, fc_in, pp.core_in, P + pp.fc_b, st));
    TB_TRY(core_extras(w.core_in, pp.core_in, N, kFcOut, reward, nullptr, 0, st));
    if (use_lstm) {
      LstmParams lp;
      lp.w_ih[0] = P + pp.lstm[0]; lp.w_hh[0] = P + pp.lstm[1]; lp.b_ih[0] = P + pp.lstm[2]; lp.b_hh[0] = P + pp.lstm[3];
      lp.w_ih[1] = lp.w_hh[1] = lp.b_ih[1] = lp.b_hh[1] = nullptr;
      TB_TRY(lstm_forward(w.core_in, notdone, h0, c0, lp, T1, B, pp.core_in, kLstmH, 1, w.lstm, w.core_out, hN, cN, kBf16 ? 1 : 0,
                          st));
    }
    TB_TRY(heads_forward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.policy_b, P + pp.baseline_w, P + pp.baseline_b, N,
                         pp.core_out, A, policy_logits, baseline, st, V));
    return 0;
  }

  // one 3x3 conv backward: bias grad, weight grad (patch matrix recomputed from the stored input), and - if dx - the
  // input gradient dx = col2im(dY . W) * (relu_in ? x > 0 : 1) + addend
  static int conv_bwd(const T* x, bool relu_in, const T* dY, const T* Wp, float* dW, float* db, T* dx, const T* addend, int64_t N,
                      int H, int W, int cin, int cout, ResWs<T>& w, cudaStream_t st) {
    const int64_t M = N * H * W, K = int64_t(cin) * 9, ldk = ldk_of(cin, kBf16);
    TB_TRY(colsum_t<T>(dY, db, M, cout, cout, w.colsum_scratch, st));
    TB_TRY(im2col3x3<T>(x, w.col, N, H, W, cin, ldk, relu_in ? 1 : 0, st));
    TB_TRY(conv_wgrad(dY, w.col, false, dW, M, cout, K, ldk, 9, cin, 1.0f, w.splitk, "res_conv_wgrad", st));
    if (dx) {
      TB_TRY(conv_dgrad(dY, Wp, w.dcol, M, cout, K, ldk, "res_conv_dgrad", st));
      TB_TRY(col2im3x3<T>(w.dcol, relu_in ? x : nullptr, addend, dx, N, H, W, cin, ldk, st));
    }
    return 0;
  }

  static int backward(const ResGeom& g, const uint8_t* frame, const float* grad_logits, const float* grad_baseline,
                      const float* notdone, const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace, float* G,
                      cudaStream_t st, int V = 1) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(g, A, use_lstm, V);
    ResWs<T> w = res_ws<T>(g, workspace, N, T1, B, A, use_lstm);
    const int64_t fc_in = g.fc_in();
    // heads
    TB_REQUIRE(heads_scratch_floats(N, pp.core_out, A, V) <= w.splitk_floats, "resnet_backward: heads scratch too small");
    TB_TRY(heads_backward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.baseline_w, grad_logits, grad_baseline, N, pp.core_out,
                          A, w.dcore_out, pp.core_out, G + pp.policy_w, G + pp.policy_b, G + pp.baseline_w, G + pp.baseline_b,
                          w.splitk, st, V));
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
    TB_TRY(conv_wgrad(w.dfc, w.fcin, false, G + pp.fc_w, N, kFcOut, fc_in, fc_in, g.fc_hw(), g.ch[kSections - 1], 1.0f, w.splitk, "fc_wgrad", st));
    TB_TRY(conv_dgrad(w.dfc, w.wfc, w.dfcin, N, kFcOut, fc_in, fc_in, "fc_dgrad", st));
    T* g0 = w.g[0]; T* g1 = w.g[1]; T* g2 = w.g[2];
    TB_TRY(relu_bwd<T>(w.s[2].X2, w.dfcin, g0, N * fc_in, st));  // dL/dX2 of the last section
    for (int i = kSections - 1; i >= 0; --i) {
      const int H = g.H[i], W = g.W[i], Ho = g.H[i + 1], Wo = g.W[i + 1], ch = g.ch[i], cin = g.cin(i);
      Sec<T>& s = w.s[i];
      // block 2: X2 = X1 + conv_b(relu(Y2)), Y2 = conv_a(relu(X1))
      TB_TRY(conv_bwd(s.Y2, true, g0, w.wblk[i][3], G + pp.blk[i][3].w, G + pp.blk[i][3].b, g1, nullptr, N, Ho, Wo, ch, ch, w, st));
      TB_TRY(conv_bwd(s.X1, true, g1, w.wblk[i][2], G + pp.blk[i][2].w, G + pp.blk[i][2].b, g2, g0, N, Ho, Wo, ch, ch, w, st));
      // block 1: X1 = X0 + conv_b(relu(Y1)), Y1 = conv_a(relu(X0))
      TB_TRY(conv_bwd(s.Y1, true, g2, w.wblk[i][1], G + pp.blk[i][1].w, G + pp.blk[i][1].b, g0, nullptr, N, Ho, Wo, ch, ch, w, st));
      TB_TRY(conv_bwd(s.X0, true, g0, w.wblk[i][0], G + pp.blk[i][0].w, G + pp.blk[i][0].b, g1, g2, N, Ho, Wo, ch, ch, w, st));
      TB_TRY(maxpool3x3s2_bwd<T>(s.arg, g1, g2, N, H, W, ch, st));   // g2 = dL/dP
      const int64_t M = N * H * W;
      if (i == 0) {
        const int64_t ldk_in = ldk_of(g.C, kBf16);
        TB_TRY(colsum_t<T>(g2, G + pp.feat[0].b, M, ch, ch, w.colsum_scratch, st));
        TB_TRY(im2col3x3_u8_nchw<ColFirst>(frame, reinterpret_cast<ColFirst*>(w.col), N, g.C, H, W, ldk_in, st));
        TB_TRY(conv_wgrad(g2, w.col, !kBf16, G + pp.feat[0].w, M, ch, int64_t(g.C) * 9, ldk_in, 1, 1, 1.0f / 255.0f, w.splitk,
                          "feat_conv_wgrad", st));
      } else {
        TB_TRY(conv_bwd(w.s[i - 1].X2, false, g2, w.wfeat[i], G + pp.feat[i].w, G + pp.feat[i].b, g0, nullptr, N, H, W, cin, ch, w, st));
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
                       float* out, int64_t N, int H, int Wd, int cin, int cout, const float* bias, const float* addend,
                       __nv_bfloat16* emit, int64_t emit_lo, int emit_relu, const char* tag, cudaStream_t st) {
    TB_TRY(sw_pack_weights(Wsrc, wi, cout, cin, 0, st));
    if (x) TB_TRY(sw_pad_split(x, xp, xp_lo, N, H, Wd, cin, relu_in, st));
    SwEpilogue ep; ep.bias = bias; ep.addend = addend; ep.emit = emit; ep.emit_lo = emit_lo; ep.emit_relu = emit_relu; ep.tag = tag;
    return sw_conv_fwd(xp, xp_lo, wi, out, N, H, Wd, cin, cout, ep, st);
  }

  // done == nullptr: frame is stacked u8 [T1,B,C,H,W]; otherwise an unstacked rollout u8 [T1+3,B,84,84] (g = (4, 84, 84)),
  // restacked by the pass that writes the first conv's input image
  static int forward(const ResGeom& g, const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                     const float* h0, const float* c0, const float* P, int64_t T1, int64_t B, int A, int use_lstm, void* workspace,
                     float* policy_logits, float* baseline, float* hN, float* cN, cudaStream_t st, int V = 1) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(g, A, use_lstm, V);
    W w = res_ws<float>(g, workspace, N, T1, B, A, use_lstm, true);
    const int64_t fc_in = g.fc_in();
    TB_TRY(pack_weights_bf16(P + pp.fc_w, w.wb_fc, kFcOut, g.fc_hw(), g.ch[kSections - 1], fc_in, st, w.wb_fc_lo));
    for (int i = 0; i < kSections; ++i) {
      const int H = g.H[i], Wd = g.W[i], Ho = g.H[i + 1], Wo = g.W[i + 1], ch = g.ch[i], cin = g.cin(i);
      if (i == 0) {
        // the first conv through the same kernels: frame pixels (exact in bf16) as a 16-channel image, 1/255 in the epilogue
        TB_TRY(sw_pack_weights(P + pp.feat[0].w, w.wi_feat[0], ch, 16, 0, st, g.C));
        if (done)
          TB_TRY(sw_frames_u8_unstacked(frame, done, w.xp_feat[0], w.xp_feat_lo[0], T1, B, H, Wd, st));
        else
          TB_TRY(sw_frames_u8(frame, w.xp_feat[0], w.xp_feat_lo[0], N, g.C, H, Wd, st));
        SwEpilogue ep; ep.scale = 1.0f / 255.0f; ep.bias = P + pp.feat[0].b; ep.tag = "feat_conv_fwd";
        TB_TRY(sw_conv_fwd(w.xp_feat[0], w.xp_feat_lo[0], w.wi_feat[0], w.s[0].P, N, H, Wd, 16, ch, ep, st));
      } else {
        // (its input image was written by the epilogue of the previous section's last conv)
        TB_TRY(conv_impl(nullptr, 0, w.xp_feat[i], w.xp_feat_lo[i], P + pp.feat[i].w, w.wi_feat[i], w.wi_feat_lo[i], w.s[i].P, N, H, Wd,
                         cin, ch, P + pp.feat[i].b, nullptr, nullptr, 0, 0, "feat_conv_fwd", st));
      }
      TB_TRY(maxpool3x3s2_fwd<float>(w.s[i].P, w.s[i].X0, w.s[i].arg, N, H, Wd, ch, st));
      float* outs[4] = {w.s[i].Y1, w.s[i].X1, w.s[i].Y2, w.s[i].X2};
      const float* adds[4] = {nullptr, w.s[i].X0, nullptr, w.s[i].X1};
      for (int j = 0; j < 4; ++j) {
        // conv j's epilogue writes relu(output) as conv j+1's input image; the section's last conv writes the next
        // section's feat-conv input (no ReLU there)
        __nv_bfloat16* emit = j < 3 ? w.xp_blk[i][j + 1] : (i + 1 < kSections ? w.xp_feat[i + 1] : nullptr);
        const int64_t emit_lo = j < 3 ? w.xp_blk_lo[i][j + 1] : (i + 1 < kSections ? w.xp_feat_lo[i + 1] : 0);
        TB_TRY(conv_impl(j == 0 ? w.s[i].X0 : nullptr, 1, w.xp_blk[i][j], w.xp_blk_lo[i][j], P + pp.blk[i][j].w, w.wi_blk[i][j],
                         w.wi_blk_lo[i][j], outs[j], N, Ho, Wo, ch, ch, P + pp.blk[i][j].b, adds[j], emit, emit_lo, j < 3 ? 1 : 0,
                         "res_conv_fwd", st));
      }
    }
    TB_TRY(relu_fwd<float>(w.s[2].X2, w.fcin, N * fc_in, st));
    TB_TRY(f32_to_bf16(w.fcin, w.fcb, N, fc_in, fc_in, fc_in, st, w.fcb_lo));
    TB_TRY(gemm_fwd(w.fcb, w.fcb_lo, w.wb_fc, w.wb_fc_lo, w.core_in, N, kFcOut, fc_in, fc_in, P + pp.fc_b, nullptr, 1.0f, 1,
                    pp.core_in, "fc_fwd", st));
    TB_TRY(core_extras(w.core_in, pp.core_in, N, kFcOut, reward, nullptr, 0, st));
    if (use_lstm) {
      LstmParams lp;
      lp.w_ih[0] = P + pp.lstm[0]; lp.w_hh[0] = P + pp.lstm[1]; lp.b_ih[0] = P + pp.lstm[2]; lp.b_hh[0] = P + pp.lstm[3];
      lp.w_ih[1] = lp.w_hh[1] = lp.b_ih[1] = lp.b_hh[1] = nullptr;
      TB_TRY(lstm_forward(w.core_in, notdone, h0, c0, lp, T1, B, pp.core_in, kLstmH, 1, w.lstm, w.core_out, hN, cN, 2, st));
    }
    TB_TRY(heads_forward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.policy_b, P + pp.baseline_w, P + pp.baseline_b, N,
                         pp.core_out, A, policy_logits, baseline, st, V));
    return 0;
  }

  // one 3x3 conv backward on the shifted-window kernels: dY -> padded planar image (+ bias gradient in the same pass);
  // weight gradient from that image and the input image kept by the forward pass; input gradient = the SAME convolution
  // kernel over the dY image with flipped / transposed weights, ReLU mask and skip gradient in its epilogue
  static int conv_bwd_impl(const float* x, bool relu_in, const float* dY, __nv_bfloat16* dyimg, int64_t dyimg_lo, const float* Wsrc,
                           const __nv_bfloat16* xp, int64_t xp_lo, __nv_bfloat16* wd, int64_t wd_lo, float* dW, float* db, float* dx,
                           const float* addend, __nv_bfloat16* emit, int64_t emit_lo, float* emit_db, int64_t N, int H, int Wd, int cin,
                           int cout, W& w, const char* wtag, cudaStream_t st) {
    // dY == nullptr: dyimg (and db) were already produced by the previous kernel's epilogue / the fused max-pool backward
    if (dY) TB_TRY(sw_pad_split_colsum(dY, dyimg, dyimg_lo, N, H, Wd, cout, db, w.splitk, w.splitk_floats, st));
    TB_TRY(sw_conv_wgrad(dyimg, dyimg_lo, xp, xp_lo, dW, N, H, Wd, cin, cout, w.splitk, w.splitk_floats, wtag, st));
    if (dx) {
      TB_TRY(sw_pack_weights(Wsrc, wd, cout, cin, 1, st));
      SwEpilogue ep; ep.mask = relu_in ? x : nullptr; ep.addend = addend; ep.tag = "res_conv_dgrad";
      // emit: dx is the dY of the conv that runs next in this backward pass - its image and (through the column sums) its
      // bias gradient come out of this epilogue
      const int64_t rows = sw_csum_rows(N, H, Wd);
      if (emit) {
        TB_REQUIRE((rows + 128) * cin <= w.splitk_floats, "resnet: column-sum scratch too small");
        ep.emit = emit; ep.emit_lo = emit_lo; ep.csum = w.splitk;
      }
      TB_TRY(sw_conv_fwd(dyimg, dyimg_lo, wd, dx, N, H, Wd, cout, cin, ep, st));
      if (emit) TB_TRY(sw_csum_reduce(w.splitk, rows, cin, emit_db, st));
    }
    return 0;
  }

  // reads no frames: the first conv's weight gradient uses the input image the forward left in the workspace
  static int backward(const ResGeom& g, const float* grad_logits, const float* grad_baseline, const float* notdone, const float* P,
                      int64_t T1, int64_t B, int A, int use_lstm, void* workspace, float* G, cudaStream_t st, int V = 1) {
    const int64_t N = T1 * B;
    const ResParams pp = res_params(g, A, use_lstm, V);
    W w = res_ws<float>(g, workspace, N, T1, B, A, use_lstm, true);
    const int64_t fc_in = g.fc_in();
    TB_REQUIRE(heads_scratch_floats(N, pp.core_out, A, V) <= w.splitk_floats, "resnet_backward: heads scratch too small");
    TB_TRY(heads_backward(w.core_out, pp.core_out, P + pp.policy_w, P + pp.baseline_w, grad_logits, grad_baseline, N, pp.core_out,
                          A, w.dcore_out, pp.core_out, G + pp.policy_w, G + pp.policy_b, G + pp.baseline_w, G + pp.baseline_b,
                          w.splitk, st, V));
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
    TB_TRY(gemm_wgrad(w.dfcb, w.dfcb_lo, w.fcb, w.fcb_lo, G + pp.fc_w, N, kFcOut, fc_in, fc_in, g.fc_hw(), g.ch[kSections - 1], 1.0f, w.splitk,
                      "fc_wgrad", st));
    {
      TcEpilogue te; te.C = w.dfcin; te.ldc = fc_in; te.a_lo = w.dfcb_lo; te.b_lo = w.wb_fc_lo; te.tag = "fc_dgrad";
      TB_TRY(gemm_tc_bf16_ex(w.dfcb, w.wb_fc, N, fc_in, kFcOut, kFcOut, fc_in, false, true, te, 1, nullptr, st));
    }
    float* g0 = w.g[0]; float* g1 = w.g[1]; float* g2 = w.g[2];
    TB_TRY(relu_bwd<float>(w.s[2].X2, w.dfcin, g0, N * fc_in, st));
    __nv_bfloat16* dyi[2] = {w.dyp, w.dyp2};   // dY images: dyi[dsel] is the one the next kernel reads
    const int64_t dyi_lo[2] = {w.dyp_lo, w.dyp2_lo};
    int dsel = 0;
    for (int i = kSections - 1; i >= 0; --i) {
      const int H = g.H[i], Wd = g.W[i], Ho = g.H[i + 1], Wo = g.W[i + 1], ch = g.ch[i], cin = g.cin(i);
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
                             dyi_lo[dsel ^ 1], j > 0 ? G + pp.blk[i][j - 1].b : nullptr, N, Ho, Wo, ch, ch, w, "res_conv_wgrad", st));
        if (nxt) dsel ^= 1;
      }
      // dL/dP (the feat conv's output gradient) is consumed only as that conv's dY image + bias gradient: the max-pool
      // backward gathers straight into the image (never materialised in fp32)
      TB_TRY(sw_pool_bwd_image_colsum(s.arg, g1, dyi[dsel], dyi_lo[dsel], N, H, Wd, ch, G + pp.feat[i].b, w.splitk, w.splitk_floats, st));
      if (i == 0) {
        TB_TRY(sw_conv_wgrad(dyi[dsel], dyi_lo[dsel], w.xp_feat[0], w.xp_feat_lo[0], G + pp.feat[0].w, N, H, Wd, 16, ch, w.splitk,
                             w.splitk_floats, "feat_conv_wgrad", st, 1.0f / 255.0f, g.C));
      } else {
        // its dx = dL/dX2 of section i-1 = the dY of that section's last conv: emitted as the image + bias gradient that
        // conv's backward starts from
        TB_TRY(conv_bwd_impl(w.s[i - 1].X2, false, nullptr, dyi[dsel], dyi_lo[dsel], P + pp.feat[i].w, w.xp_feat[i], w.xp_feat_lo[i],
                             w.wd_feat[i], w.wd_feat_lo[i], G + pp.feat[i].w, G + pp.feat[i].b, g0, nullptr, dyi[dsel ^ 1], dyi_lo[dsel ^ 1],
                             G + pp.blk[i - 1][3].b, N, H, Wd, cin, ch, w, "res_conv_wgrad", st));
        dsel ^= 1;
      }
    }
    return 0;
  }
};

size_t res_ws_bytes(const ResGeom& g, int64_t T1, int64_t B, int A, int use_lstm, int precision) {
  if (precision == 2) return res_ws<float>(g, nullptr, T1 * B, T1, B, A, use_lstm, true).bytes;
  return precision ? res_ws<__nv_bfloat16>(g, nullptr, T1 * B, T1, B, A, use_lstm).bytes
                   : res_ws<float>(g, nullptr, T1 * B, T1, B, A, use_lstm).bytes;
}

}  // namespace
}  // namespace tb

using namespace tb;

extern "C" {

int tb_resnet_obs_range(int* range) {
  TB_REQUIRE(range, "resnet_obs_range: null pointer");
  const int r[6] = {1, kObsMaxC, kObsMinH, kObsMaxHW, kObsMinW, kObsMaxHW};
  for (int i = 0; i < 6; ++i) range[i] = r[i];
  return 0;
}

int tb_resnet_widths(int* widths) {
  TB_REQUIRE(widths, "resnet_widths: null pointer");
  for (int i = 0; i < 3; ++i) widths[i] = kWidths[i];
  return 0;
}

int tb_resnet_supported(int C, int H, int W, int ch0, int ch1, int ch2, int precision) {
  const int ch[kSections] = {ch0, ch1, ch2};
  return res_geom_check(C, H, W, ch, precision, "resnet_supported") == 0 ? 1 : 0;
}

int64_t tb_resnet_param_count(int C, int H, int W, int ch0, int ch1, int ch2, int num_actions, int num_values, int use_lstm) {
  const int ch[kSections] = {ch0, ch1, ch2};
  if (res_geom_check(C, H, W, ch, 0, "resnet_param_count")) return -1;
  return res_params(res_geom(C, H, W, ch), num_actions, use_lstm, num_values).total;
}

size_t tb_resnet_workspace_bytes(int C, int H, int W, int ch0, int ch1, int ch2, int64_t T1, int64_t B, int num_actions,
                                 int use_lstm, int precision) {
  const int ch[kSections] = {ch0, ch1, ch2};
  if (res_geom_check(C, H, W, ch, precision, "resnet_workspace_bytes")) return 0;
  return res_ws_bytes(res_geom(C, H, W, ch), T1, B, num_actions, use_lstm, precision);
}

int tb_resnet_forward(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone, const float* h0,
                      const float* c0, const float* params, int C, int H, int W, int ch0, int ch1, int ch2, int64_t T1,
                      int64_t B, int num_actions, int num_values, int use_lstm, int precision, void* workspace,
                      void* stacked_scratch, float* policy_logits, float* baseline, float* hN, float* cN, void* stream) {
  TB_REQUIRE(num_values >= 1 && num_values <= kHeadsMaxValues, "resnet_forward: num_values %d outside [1, %d]", num_values,
             kHeadsMaxValues);
  TB_REQUIRE(T1 >= 1 && B >= 1 && num_actions >= 1, "resnet_forward: bad sizes");
  TB_REQUIRE(frame && reward && params && workspace && policy_logits && baseline, "resnet_forward: null pointer");
  TB_REQUIRE(!use_lstm || (notdone && h0 && c0 && hN && cN), "resnet_forward: LSTM needs notdone/h0/c0/hN/cN");
  TB_REQUIRE(precision >= 0 && precision <= 2, "resnet_forward: precision must be 0 (fp32), 1 (bf16) or 2 (split-bf16)");
  TB_REQUIRE(!done || (C == 4 && H == 84 && W == 84 && ch0 == kDefaultCh[0] && ch1 == kDefaultCh[1] && ch2 == kDefaultCh[2]),
             "resnet_forward: unstacked frames (done != NULL) need the (4, 84, 84) observation and the default widths "
             "(16, 32, 32), got (%d, %d, %d) and (%d, %d, %d)", C, H, W, ch0, ch1, ch2);
  const int ch[kSections] = {ch0, ch1, ch2};
  TB_TRY(res_geom_check(C, H, W, ch, precision, "resnet_forward"));
  const ResGeom g = res_geom(C, H, W, ch);
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == 2)  // unstacked frames: the restack is fused into the first conv's image pass
    return SplitImpl::forward(g, frame, done, reward, notdone, h0, c0, params, T1, B, num_actions, use_lstm, workspace,
                              policy_logits, baseline, hN, cN, st, num_values);
  if (done) {
    TB_REQUIRE(stacked_scratch, "resnet_forward: the fp32 / bf16 backends need stacked_scratch "
                                "(tb_unstacked_scratch_bytes bytes)");
    uint8_t* stacked = static_cast<uint8_t*>(stacked_scratch);
    TB_TRY(restack_frames_u8(frame, done, T1, B, 84 * 84, stacked, st));
    frame = stacked;
  }
  if (precision)
    return Impl<__nv_bfloat16>::forward(g, frame, reward, notdone, h0, c0, params, T1, B, num_actions, use_lstm, workspace,
                                        policy_logits, baseline, hN, cN, st, num_values);
  return Impl<float>::forward(g, frame, reward, notdone, h0, c0, params, T1, B, num_actions, use_lstm, workspace, policy_logits,
                              baseline, hN, cN, st, num_values);
}

int tb_resnet_backward(const uint8_t* frame, const float* grad_logits, const float* grad_baseline, const float* notdone,
                       const float* params, int C, int H, int W, int ch0, int ch1, int ch2, int64_t T1, int64_t B,
                       int num_actions, int num_values, int use_lstm, int precision, void* workspace, float* grads,
                       void* stream) {
  TB_REQUIRE(num_values >= 1 && num_values <= kHeadsMaxValues, "resnet_backward: num_values %d outside [1, %d]", num_values,
             kHeadsMaxValues);
  TB_REQUIRE(T1 >= 1 && B >= 1 && num_actions >= 1, "resnet_backward: bad sizes");
  // the split-bf16 backend reads the first conv's input image from the workspace, the others re-read the frame
  TB_REQUIRE((frame || precision == 2) && grad_logits && grad_baseline && params && workspace && grads,
             "resnet_backward: null pointer");
  TB_REQUIRE(!use_lstm || notdone, "resnet_backward: LSTM needs notdone");
  TB_REQUIRE(precision >= 0 && precision <= 2, "resnet_backward: precision must be 0, 1 or 2");
  const int ch[kSections] = {ch0, ch1, ch2};
  TB_TRY(res_geom_check(C, H, W, ch, precision, "resnet_backward"));
  const ResGeom g = res_geom(C, H, W, ch);
  if (precision == 2)
    return SplitImpl::backward(g, grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm, workspace, grads,
                               (cudaStream_t)stream, num_values);
  if (precision)
    return Impl<__nv_bfloat16>::backward(g, frame, grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm,
                                         workspace, grads, (cudaStream_t)stream, num_values);
  return Impl<float>::backward(g, frame, grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm, workspace,
                               grads, (cudaStream_t)stream, num_values);
}

}  // extern "C"
