// AtariNet forward / backward for the IMPALA learner (sm_90a), behind the C ABI.
//
// Replaces /root/reference/torchbeast/monobeast.py:582-632 (AtariNet.forward) and the autograd
// graph torch builds behind it:   u8 frame -> /255 -> conv 8x8/4 -> conv 4x4/2 -> conv 3x3/1 ->
// fc 3136->512 -> cat[x, clip(reward), onehot(last_action)] -> [2-layer LSTM] -> policy/baseline.
//
// Structure: every dense contraction (3 convs as patch-matrix GEMMs, fc, heads, LSTM projections;
// forward, dgrad and wgrad) goes through ONE GEMM interface (gemm_simt.cuh today, the wgmma
// backend next); activations live in NHWC so that a GEMM's [rows, channels] output is the next
// layer's input with no transpose; weights stay in the reference's state_dict layout in one flat
// buffer and are re-packed per step into GEMM order (tiny); weight gradients are un-packed into
// the same flat layout by the split-K reduction so a flat optimizer / all-reduce can run on them.
#include "gemm_simt.cuh"
#include "conv_implicit.cuh"
#include "gemm_tc.cuh"
#include "heads.cuh"
#include "lstm.cuh"
#include "net_kernels.cuh"
#include "restack.cuh"

namespace tb {

// ---------------------------------------------------------------------------------------
// geometry + parameter / workspace layout
// ---------------------------------------------------------------------------------------
struct AtariGeom {
  static constexpr int C0 = 4, H0 = 84, W0 = 84;
  static constexpr int C1 = 32, K1 = 8, S1 = 4, H1 = 20, W1 = 20;  // conv1
  static constexpr int C2 = 64, K2 = 4, S2 = 2, H2 = 9, W2 = 9;    // conv2
  static constexpr int C3 = 64, K3 = 3, S3 = 1, H3 = 7, W3 = 7;    // conv3
  static constexpr int FC_IN = C3 * H3 * W3;                       // 3136
  static constexpr int FC_OUT = 512;
  static constexpr int KD1 = C0 * K1 * K1;  // 256
  static constexpr int KD2 = K2 * K2 * C1;  // 512
  static constexpr int KD3 = K3 * K3 * C2;  // 576
};

// The tensor-core trunk runs every convolution as an implicit GEMM (no patch matrices); the fixed geometry must satisfy
// all five kernels' shape predicates.
static bool implicit_geometry_ok() {
  using G = AtariGeom;
  static const bool ok = conv_u8_implicit_applicable(G::C0, G::H0, G::W0, G::K1, G::K1, G::S1, G::C1) &&
                         conv_tc_implicit_applicable(G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, G::C2) &&
                         conv_tc_implicit_applicable(G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, G::C3) &&
                         conv_tc_dgrad_implicit_applicable(G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, G::C2) &&
                         conv_tc_dgrad_implicit_applicable(G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, G::C3);
  return ok;
}

struct AtariParams {  // offsets (in floats) into the flat parameter / gradient buffers
  int64_t conv1_w, conv1_b, conv2_w, conv2_b, conv3_w, conv3_b, fc_w, fc_b;
  int64_t lstm[2][4];  // per layer: w_ih, w_hh, b_ih, b_hh
  int64_t policy_w, policy_b, baseline_w, baseline_b, total;
  int core;  // 512 + 1 + A (a continuous space: 512 + 1 + D)
};

// V: value outputs.  Dc > 0: a continuous action space of Dc dimensions, whose core takes Dc last-action columns while
// the policy layer stays A = 2 Dc wide; 0: the core takes A columns.
static AtariParams atari_params(int A, int use_lstm, int V = 1, int Dc = 0) {
  using G = AtariGeom;
  AtariParams p;
  int64_t o = 0;
  auto take = [&](int64_t n) { int64_t r = o; o += n; return r; };
  p.core = G::FC_OUT + 1 + (Dc ? Dc : A);
  p.conv1_w = take(int64_t(G::C1) * G::KD1); p.conv1_b = take(G::C1);
  p.conv2_w = take(int64_t(G::C2) * G::KD2); p.conv2_b = take(G::C2);
  p.conv3_w = take(int64_t(G::C3) * G::KD3); p.conv3_b = take(G::C3);
  p.fc_w = take(int64_t(G::FC_OUT) * G::FC_IN); p.fc_b = take(G::FC_OUT);
  for (int l = 0; l < 2; ++l)
    for (int k = 0; k < 4; ++k) p.lstm[l][k] = -1;
  if (use_lstm) {
    const int64_t H = p.core;
    for (int l = 0; l < 2; ++l) {
      p.lstm[l][0] = take(4 * H * H); p.lstm[l][1] = take(4 * H * H);
      p.lstm[l][2] = take(4 * H); p.lstm[l][3] = take(4 * H);
    }
  }
  p.policy_w = take(int64_t(A) * p.core); p.policy_b = take(A);
  p.baseline_w = take(int64_t(V) * p.core); p.baseline_b = take(V);
  p.total = o;
  return p;
}

// bf16 operand buffer of the tensor-core backends; lo != 0 (precision 2, split-bf16): element offset of the lo plane
struct HB {
  void* p = nullptr; int64_t lo = 0;
  operator void*() const { return p; }
  __nv_bfloat16* h() const { return static_cast<__nv_bfloat16*>(p); }
};

struct AtariWs {  // bump-carved view of the caller's workspace
  uint8_t* col1; float *act1, *col2, *act2, *col3, *act3, *core_in, *core_out;
  float *w2p, *w3p, *wfcp;
  float *dcore_out, *dcore_in, *dact3, *dcol3, *dact2, *dcol2, *dact1;
  float *splitk, *colsum_scratch;
  // tensor-core backends (precision 1: bf16, precision 2: split-bf16 hi/lo planes): operands / activations
  HB frameb, act1b, act2b, act3b, w1b, w2b, w3b, wfcb;
  HB dfcb, dact3b, w3tb, dact2b, w2tb, dact1b;
  LstmWs lstm;
  size_t bytes;
};

static AtariWs atari_ws(void* base, int64_t N, int64_t T1, int64_t B, int A, int use_lstm, int precision, int Dc = 0) {
  using G = AtariGeom;
  AtariWs w;
  size_t off = 0;
  auto take = [&](size_t nbytes) {
    void* p = base ? static_cast<char*>(base) + off : nullptr;
    off += (nbytes + 255) & ~size_t(255);
    return p;
  };
  const AtariParams pp = atari_params(A, use_lstm, 1, Dc);
  const int64_t M1 = N * G::H1 * G::W1, M2 = N * G::H2 * G::W2, M3 = N * G::H3 * G::W3;
  auto takef = [&](int64_t n) { return static_cast<float*>(take(size_t(n) * sizeof(float))); };
  const bool split = precision == 2;
  auto takeh = [&](int64_t n, bool planes = true) {  // bf16 (+ the lo plane right behind it in split mode)
    HB b;
    const size_t plane = (size_t(n) * 2 + 255) & ~size_t(255);
    b.p = take(planes && split ? 2 * plane : plane);
    b.lo = planes && split ? int64_t(plane / 2) : 0;
    return b;
  };
  w = AtariWs();
  w.core_in = takef(N * pp.core);
  w.core_out = use_lstm ? takef(N * pp.core) : w.core_in;
  w.dcore_out = takef(N * pp.core);
  w.dcore_in = use_lstm ? takef(N * pp.core) : w.dcore_out;
  if (!precision) {
    w.col1 = static_cast<uint8_t*>(take(size_t(M1) * G::KD1));
    w.act1 = takef(M1 * G::C1); w.col2 = takef(M2 * G::KD2); w.act2 = takef(M2 * G::C2);
    w.col3 = takef(M3 * G::KD3); w.act3 = takef(N * G::FC_IN);
    w.w2p = takef(int64_t(G::C2) * G::KD2); w.w3p = takef(int64_t(G::C3) * G::KD3);
    w.wfcp = takef(int64_t(G::FC_OUT) * G::FC_IN);
    w.dact3 = takef(N * G::FC_IN); w.dcol3 = takef(M3 * G::KD3); w.dact2 = takef(M2 * G::C2);
    w.dcol2 = takef(M2 * G::KD2); w.dact1 = takef(M1 * G::C1);
  } else {
    // frameb: the bf16 frame image conv1 gathers from (integers <= 255: exact in bf16, no lo plane); w2tb/w3tb: the
    // transposed weight packs of the input-gradient convolutions
    w.frameb = takeh(N * G::C0 * G::H0 * G::W0, false); w.act1b = takeh(M1 * G::C1);
    w.act2b = takeh(M2 * G::C2); w.act3b = takeh(N * G::FC_IN);
    w.w1b = takeh(int64_t(G::C1) * G::KD1); w.w2b = takeh(int64_t(G::C2) * G::KD2); w.w3b = takeh(int64_t(G::C3) * G::KD3);
    w.wfcb = takeh(int64_t(G::FC_OUT) * G::FC_IN);
    w.dfcb = takeh(N * G::FC_OUT); w.dact3b = takeh(N * G::FC_IN);
    w.w3tb = takeh(int64_t(G::C2) * G::KD3);
    w.dact2b = takeh(M2 * G::C2); w.w2tb = takeh(int64_t(4) * G::C1 * G::KD2);
    w.dact1b = takeh(M1 * G::C1);
  }
  w.splitk = takef(kSplitKScratchFloats);
  w.colsum_scratch = takef(colsum_scratch_floats(4 * int64_t(pp.core) > 512 ? 4 * int64_t(pp.core) : 512));
  if (use_lstm) {
    size_t lbytes = lstm_ws_bytes(T1, B, pp.core, pp.core, 2, precision);
    w.lstm = lstm_ws(take(lbytes), T1, B, pp.core, pp.core, 2, precision);
  } else {
    w.lstm = LstmWs();
  }
  w.bytes = off;
  return w;
}

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
// done == nullptr: frame is stacked u8 [T1,B,4,84,84]; otherwise frame is an unstacked rollout u8 [T1+3,B,84,84] whose stacks
// the tensor-core backends rebuild in their frame-image pass (the fp32 backend is handed restacked frames by its caller).
// seg non-NULL: a factored action space, last_action [T1,B,D] enters the core as a K-hot (core_extras).
// clast_action non-NULL (last_action then NULL): a continuous space of A / 2 dimensions, whose float32 [T1,B,A/2] last
// actions enter the core as they are (core_extras_continuous).
static int atarinet_forward(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                            const int64_t* last_action, const float* h0, const float* c0, const float* P,
                            int64_t T1, int64_t B, int A, int use_lstm, int precision, void* workspace,
                            float* policy_logits, float* baseline, float* hN, float* cN, cudaStream_t st, int V = 1,
                            const ActionSegments* seg = nullptr, const float* clast_action = nullptr) {
  using G = AtariGeom;
  const int64_t N = T1 * B;
  const int Dc = clast_action ? A / 2 : 0;
  const AtariParams pp = atari_params(A, use_lstm, V, Dc);
  AtariWs w = atari_ws(workspace, N, T1, B, A, use_lstm, precision, Dc);
  const int64_t M1 = N * G::H1 * G::W1, M2 = N * G::H2 * G::W2, M3 = N * G::H3 * G::W3;
  GemmEpilogue ep;
  if (precision) {
    // ---- tensor-core trunk: wgmma GEMMs, bf16 (precision 1) or split-bf16 hi/lo (precision 2) activations, fp32 accumulation
    TB_REQUIRE(implicit_geometry_ok(), "atarinet_forward: the trunk geometry does not fit the implicit-GEMM convolutions");
    TB_TRY(pack_weights_bf16(P + pp.conv1_w, w.w1b, G::C1, 1, G::KD1, G::KD1, st, w.w1b.lo));
    TB_TRY(pack_weights_bf16(P + pp.conv2_w, w.w2b, G::C2, G::K2 * G::K2, G::C1, G::KD2, st, w.w2b.lo));
    TB_TRY(pack_weights_bf16(P + pp.conv3_w, w.w3b, G::C3, G::K3 * G::K3, G::C2, G::KD3, st, w.w3b.lo));
    TB_TRY(pack_weights_bf16(P + pp.fc_w, w.wfcb, G::FC_OUT, G::H3 * G::W3, G::C3, G::FC_IN, st, w.wfcb.lo));
    TcEpilogue te;
    te = TcEpilogue(); te.C16 = w.act1b.h(); te.ldc16 = G::C1; te.c16_lo = w.act1b.lo; te.bias = P + pp.conv1_b;
    te.scale = 1.0f / 255.0f; te.relu = 1; te.tag = "conv1_fwd";
    // implicit GEMM: frames -> bf16 image once (kept in frameb for the backward), producer warps gather the
    // patches from it into the UMMA smem layout
    te.b_lo = w.w1b.lo;  // the pixels are exact in bf16: only the weights have a lo plane
    if (done)
      TB_TRY(frames_u8_unstacked_to_bf16(frame, done, T1, B, int64_t(G::H0) * G::W0, w.frameb, st));
    else
      TB_TRY(frames_u8_to_bf16(frame, w.frameb, N * G::C0 * G::H0 * G::W0, st));
    TB_TRY(conv_u8_fwd_implicit(w.frameb, w.w1b, N, G::H0, G::W0, G::S1, te, st));
    // conv2 / conv3: implicit GEMM - TMA gathers the patches from the NHWC activation (rank-4 map with
    // overlapping dimensions)
    te = TcEpilogue(); te.C16 = w.act2b.h(); te.ldc16 = G::C2; te.c16_lo = w.act2b.lo; te.bias = P + pp.conv2_b;
    te.relu = 1; te.tag = "conv2_fwd"; te.a_lo = w.act1b.lo; te.b_lo = w.w2b.lo;
    TB_TRY(conv_tc_fwd_implicit(w.act1b, w.w2b, N, G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, G::C2, te, st));
    te = TcEpilogue(); te.C16 = w.act3b.h(); te.ldc16 = G::C3; te.c16_lo = w.act3b.lo; te.bias = P + pp.conv3_b;
    te.relu = 1; te.tag = "conv3_fwd"; te.a_lo = w.act2b.lo; te.b_lo = w.w3b.lo;
    TB_TRY(conv_tc_fwd_implicit(w.act2b, w.w3b, N, G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, G::C3, te, st));
    te = TcEpilogue(); te.C = w.core_in; te.ldc = pp.core; te.bias = P + pp.fc_b; te.relu = 1; te.tag = "fc_fwd";
    te.a_lo = w.act3b.lo; te.b_lo = w.wfcb.lo;
    TB_TRY(gemm_tc_bf16(w.act3b, w.wfcb, N, G::FC_OUT, G::FC_IN, G::FC_IN, G::FC_IN, te, st));
  } else {
  // weight pack: [o, c, kh, kw] -> [o, (kh,kw), c];  fc: [o, c, (h,w)] -> [o, (h,w), c]
  TB_TRY(permute_pq(P + pp.conv2_w, w.w2p, G::C2, G::K2 * G::K2, G::C1, st));
  TB_TRY(permute_pq(P + pp.conv3_w, w.w3p, G::C3, G::K3 * G::K3, G::C2, st));
  TB_TRY(permute_pq(P + pp.fc_w, w.wfcp, G::FC_OUT, G::H3 * G::W3, G::C3, st));
  // conv1 (uint8 patch matrix; x/255 applied when the operand is read)
  TB_TRY(im2col_u8_nchw(frame, w.col1, N, G::C0, G::H0, G::W0, G::K1, G::K1, G::S1, st));
  ep = GemmEpilogue(); ep.bias = P + pp.conv1_b; ep.relu = 1; ep.tag = "conv1_fwd";
  TB_TRY((gemm_simt<uint8_t, float, false, true>(w.col1, P + pp.conv1_w, w.act1, M1, G::C1, G::KD1, G::KD1, G::KD1,
                                                  G::C1, ep, 1, nullptr, st)));
  // conv2
  TB_TRY(im2col_f32_nhwc(w.act1, w.col2, N, G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, st));
  ep = GemmEpilogue(); ep.bias = P + pp.conv2_b; ep.relu = 1; ep.tag = "conv2_fwd";
  TB_TRY((gemm_simt<float, float, false, true>(w.col2, w.w2p, w.act2, M2, G::C2, G::KD2, G::KD2, G::KD2, G::C2, ep, 1,
                                                nullptr, st)));
  // conv3
  TB_TRY(im2col_f32_nhwc(w.act2, w.col3, N, G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, st));
  ep = GemmEpilogue(); ep.bias = P + pp.conv3_b; ep.relu = 1; ep.tag = "conv3_fwd";
  TB_TRY((gemm_simt<float, float, false, true>(w.col3, w.w3p, w.act3, M3, G::C3, G::KD3, G::KD3, G::KD3, G::C3, ep, 1,
                                                nullptr, st)));
  // fc -> first 512 columns of the core input; then reward / one-hot columns
  ep = GemmEpilogue(); ep.bias = P + pp.fc_b; ep.relu = 1; ep.tag = "fc_fwd";
  TB_TRY((gemm_simt<float, float, false, true>(w.act3, w.wfcp, w.core_in, N, G::FC_OUT, G::FC_IN, G::FC_IN, G::FC_IN,
                                                pp.core, ep, 1, nullptr, st)));
  }
  if (clast_action)
    TB_TRY(core_extras_continuous(w.core_in, pp.core, N, G::FC_OUT, reward, clast_action, Dc, st));
  else
    TB_TRY(core_extras(w.core_in, pp.core, N, G::FC_OUT, reward, last_action, A, st, seg));
  if (use_lstm) {
    LstmParams lp;
    for (int l = 0; l < 2; ++l) {
      lp.w_ih[l] = P + pp.lstm[l][0]; lp.w_hh[l] = P + pp.lstm[l][1];
      lp.b_ih[l] = P + pp.lstm[l][2]; lp.b_hh[l] = P + pp.lstm[l][3];
    }
    TB_TRY(lstm_forward(w.core_in, notdone, h0, c0, lp, T1, B, pp.core, pp.core, 2, w.lstm, w.core_out, hN, cN, precision,
                        st));
  }
  // heads (fused skinny kernel: one pass over core_out for all A+1 outputs)
  TB_TRY(heads_forward(w.core_out, pp.core, P + pp.policy_w, P + pp.policy_b, P + pp.baseline_w, P + pp.baseline_b, N, pp.core,
                       A, policy_logits, baseline, st, V));
  return 0;
}

// ---------------------------------------------------------------------------------------
// backward: consumes the activations the forward left in the workspace
// ---------------------------------------------------------------------------------------
static int wgrad(const float* dY, int64_t ldy, const void* X, bool x_is_u8, int64_t ldx, float* dW, int64_t rows,
                 int64_t nout, int64_t kin, int permP, int permQ, AtariWs& w, cudaStream_t st, const char* tag) {
  // dW[nout, kin] = dY[rows, nout]^T . X[rows, kin]
  GemmEpilogue ep;
  ep.permP = permP; ep.permQ = permQ; ep.tag = tag;
  const int splits = simt_splits(nout, kin, rows, kSplitKScratchFloats, 128);
  if (x_is_u8)
    return gemm_simt<float, uint8_t, true, false>(dY, static_cast<const uint8_t*>(X), dW, nout, kin, rows, ldy, ldx,
                                                   kin, ep, splits, w.splitk, st);
  return gemm_simt<float, float, true, false>(dY, static_cast<const float*>(X), dW, nout, kin, rows, ldy, ldx, kin,
                                               ep, splits, w.splitk, st);
}


// bf16 tensor-core backward of the conv/fc trunk.  dgrad: B operand = the packed weights as stored
// (MN-major); wgrad: A = dY, B = patch matrix, both as stored (MN-major), split-K over grid.z with the
// fixed-order reduce un-packing into the state_dict layout.
static int tc_splits(int64_t M, int64_t N, int64_t K) {
  const int64_t bn = N <= 64 ? 64 : 128;
  const int64_t tiles = ((M + 127) / 128) * ((N + bn - 1) / bn);
  const int64_t kb = (K + 63) / 64;
  int64_t s = (2 * kNumSMs + tiles - 1) / tiles;
  if (s > kb / 4) s = kb / 4;
  const int64_t Np = (N + 31) & ~int64_t(31);  // partial rows are padded to 32 floats (gemm_tc.cu)
  if (s * M * Np > kSplitKScratchFloats) s = kSplitKScratchFloats / (M * Np);
  if (s > kNumSMs) s = kNumSMs;
  if (s < 1) s = 1;
  return int(s);
}

static int tc_wgrad(const HB& dYb, int64_t ldy, const HB& Xb, int64_t ldx, float* dW, int64_t rows, int64_t nout,
                    int64_t kin, int permP, int permQ, float scale, AtariWs& w, cudaStream_t st, const char* tag) {
  TcEpilogue te;
  te.C = dW; te.ldc = kin; te.permP = permP; te.permQ = permQ; te.scale = scale; te.tag = tag;
  te.a_lo = dYb.lo; te.b_lo = Xb.lo;
  return gemm_tc_bf16_ex(dYb, Xb, nout, kin, rows, ldy, ldx, true, true, te, tc_splits(nout, kin, rows), w.splitk, st);
}

static int atarinet_backward_trunk_bf16(const float* P, float* G_, const AtariParams& pp, AtariWs& w, int64_t N,
                                        cudaStream_t st) {
  using G = AtariGeom;
  const int64_t M1 = N * G::H1 * G::W1, M2 = N * G::H2 * G::W2, M3 = N * G::H3 * G::W3;
  // fc: ReLU mask (fp32, in place), bias grad, bf16 copy of dY
  TB_TRY(relu_mask_inplace(w.dcore_in, w.core_in, N, G::FC_OUT, pp.core, pp.core, st));
  TB_TRY(colsum(w.dcore_in, G_ + pp.fc_b, N, G::FC_OUT, pp.core, w.colsum_scratch, st));
  TB_TRY(f32_to_bf16(w.dcore_in, w.dfcb, N, G::FC_OUT, pp.core, G::FC_OUT, st, w.dfcb.lo));
  TB_TRY(tc_wgrad(w.dfcb, G::FC_OUT, w.act3b, G::FC_IN, G_ + pp.fc_w, N, G::FC_OUT, G::FC_IN, G::H3 * G::W3, G::C3, 1.0f, w,
                  st, "fc_wgrad"));
  TcEpilogue te;
  te = TcEpilogue(); te.C16 = w.dact3b.h(); te.ldc16 = G::FC_IN; te.c16_lo = w.dact3b.lo;
  te.mask16 = w.act3b.h(); te.ldmask = G::FC_IN; te.tag = "fc_dgrad"; te.a_lo = w.dfcb.lo; te.b_lo = w.wfcb.lo;
  TB_TRY(gemm_tc_bf16_ex(w.dfcb, w.wfcb, N, G::FC_IN, G::FC_OUT, G::FC_OUT, G::FC_IN, false, true, te, 1, nullptr, st));
  // conv3 (dact3b viewed as [M3, 64]); the weight gradients gather their patches from the activations
  TB_TRY(conv_tc_wgrad_implicit(w.dact3b, w.act2b, N, G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, G::C3, G_ + pp.conv3_w,
                                G::K3 * G::K3, G::C2, 1.0f, w.splitk, kSplitKScratchFloats, "conv3_wgrad", st, w.dact3b.lo,
                                w.act2b.lo));
  TB_TRY(colsum_bf16(w.dact3b, G_ + pp.conv3_b, M3, G::C3, G::C3, w.colsum_scratch, st, w.dact3b.lo));
  // gather-form transposed convolution on tensor cores: dY boxes through TMA (zero fill = padding), ReLU mask in the
  // epilogue
  TB_TRY(pack_dgrad_weights_bf16(P + pp.conv3_w, w.w3tb, G::C3, G::C2, G::K3, G::K3, G::S3, st, w.w3tb.lo));
  te = TcEpilogue(); te.C16 = w.dact2b.h(); te.ldc16 = G::C2; te.c16_lo = w.dact2b.lo;
  te.mask16 = w.act2b.h(); te.ldmask = G::C2; te.tag = "conv3_dgrad"; te.a_lo = w.dact3b.lo; te.b_lo = w.w3tb.lo;
  TB_TRY(conv_tc_dgrad_implicit(w.dact3b, w.w3tb, N, G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, G::C3, te, st));
  // conv2
  TB_TRY(conv_tc_wgrad_implicit(w.dact2b, w.act1b, N, G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, G::C2, G_ + pp.conv2_w,
                                G::K2 * G::K2, G::C1, 1.0f, w.splitk, kSplitKScratchFloats, "conv2_wgrad", st, w.dact2b.lo,
                                w.act1b.lo));
  TB_TRY(colsum_bf16(w.dact2b, G_ + pp.conv2_b, M2, G::C2, G::C2, w.colsum_scratch, st, w.dact2b.lo));
  TB_TRY(pack_dgrad_weights_bf16(P + pp.conv2_w, w.w2tb, G::C2, G::C1, G::K2, G::K2, G::S2, st, w.w2tb.lo));
  te = TcEpilogue(); te.C16 = w.dact1b.h(); te.ldc16 = G::C1; te.c16_lo = w.dact1b.lo;
  te.mask16 = w.act1b.h(); te.ldmask = G::C1; te.tag = "conv2_dgrad"; te.a_lo = w.dact2b.lo; te.b_lo = w.w2tb.lo;
  TB_TRY(conv_tc_dgrad_implicit(w.dact2b, w.w2tb, N, G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, G::C2, te, st));
  // conv1: frameb holds the bf16 frame image the forward left there (raw pixel values), so the weight gradient carries
  // the 1/255
  TB_TRY(conv_u8_wgrad_implicit(w.dact1b, w.frameb, N, G::H0, G::W0, G::S1, G_ + pp.conv1_w, 1.0f / 255.0f, w.splitk,
                                kSplitKScratchFloats, "conv1_wgrad", st, w.dact1b.lo));
  TB_TRY(colsum_bf16(w.dact1b, G_ + pp.conv1_b, M1, G::C1, G::C1, w.colsum_scratch, st, w.dact1b.lo));
  return 0;
}

// phases: bit 0 = heads + LSTM (after it the gradient slice [tb_atarinet_grad_split, total) is final unless the LSTM
// weight-gradient GEMMs were forked onto the side stream - then it is final after phase 2's join), bit 1 = conv/fc trunk
// (slice [0, split)).  3 = the whole backward.  The split lets a data-parallel learner start the all-reduce of the
// LSTM + heads slice (17 of 24 MB) while the trunk backward is still running (SURVEY 8(e) G1: bucket order = reverse of forward).
static int atarinet_backward(const float* grad_logits, const float* grad_baseline, const float* notdone,
                             const float* P, int64_t T1, int64_t B, int A, int use_lstm, int precision,
                             void* workspace, float* G_, cudaStream_t st, int phases = 3, int V = 1, int Dc = 0) {
  using G = AtariGeom;
  const int64_t N = T1 * B;
  const AtariParams pp = atari_params(A, use_lstm, V, Dc);
  AtariWs w = atari_ws(workspace, N, T1, B, A, use_lstm, precision, Dc);
  const int64_t M1 = N * G::H1 * G::W1, M2 = N * G::H2 * G::W2, M3 = N * G::H3 * G::W3;
  GemmEpilogue ep;
  if (phases & 1) {
  // heads: dcore_out = dlogits . Wp + dbaseline . Wb ; dWp, dbp, dWb, dbb.  The partials fit the split-K scratch at every
  // batch size: their slab count is capped, and the largest heads (A = 31, V = 64, F = 544) fit at the cap.
  static_assert(int64_t(kHeadsMaxSlabs) * (31 + kHeadsMaxValues) * (G::FC_OUT + 1 + 31 + 1) <= kSplitKScratchFloats,
                "heads scratch");
  TB_REQUIRE(heads_scratch_floats(N, pp.core, A, V) <= kSplitKScratchFloats, "atarinet_backward: heads scratch too small");
  TB_TRY(heads_backward(w.core_out, pp.core, P + pp.policy_w, P + pp.baseline_w, grad_logits, grad_baseline, N, pp.core, A,
                        w.dcore_out, pp.core, G_ + pp.policy_w, G_ + pp.policy_b, G_ + pp.baseline_w, G_ + pp.baseline_b, w.splitk,
                        st, V));
  }
  if (use_lstm && (phases & 1)) {
    LstmParams lp; LstmGrads lg;
    for (int l = 0; l < 2; ++l) {
      lp.w_ih[l] = P + pp.lstm[l][0]; lp.w_hh[l] = P + pp.lstm[l][1];
      lp.b_ih[l] = P + pp.lstm[l][2]; lp.b_hh[l] = P + pp.lstm[l][3];
      lg.w_ih[l] = G_ + pp.lstm[l][0]; lg.w_hh[l] = G_ + pp.lstm[l][1];
      lg.b_ih[l] = G_ + pp.lstm[l][2]; lg.b_hh[l] = G_ + pp.lstm[l][3];
    }
    TB_TRY(lstm_backward(w.dcore_out, w.core_in, notdone, lp, lg, T1, B, pp.core, pp.core, 2, w.lstm, w.dcore_in,
                         w.splitk, w.colsum_scratch, precision, st));
  }
  // phase 1 alone: the heads' gradients are final in stream order on `st`; the LSTM weight gradients in stream order on the
  // side stream their GEMMs were forked onto (the caller's aux stream, tb_set_aux_stream) - joined at the end of phase 2
  if (!(phases & 2)) return 0;
  if (precision) {
    TB_TRY(atarinet_backward_trunk_bf16(P, G_, pp, w, N, st));
    return lstm_backward_join(st);  // the LSTM weight-gradient GEMMs ran beside the trunk backward
  }
  // fc: ReLU mask on the first 512 columns, wgrad (un-packed into [o, c, (h,w)]), bias, dgrad (+ReLU mask of act3)
  TB_TRY(relu_mask_inplace(w.dcore_in, w.core_in, N, G::FC_OUT, pp.core, pp.core, st));
  TB_TRY(wgrad(w.dcore_in, pp.core, w.act3, false, G::FC_IN, G_ + pp.fc_w, N, G::FC_OUT, G::FC_IN, G::H3 * G::W3,
               G::C3, w, st, "fc_wgrad"));
  TB_TRY(colsum(w.dcore_in, G_ + pp.fc_b, N, G::FC_OUT, pp.core, w.colsum_scratch, st));
  ep = GemmEpilogue(); ep.mask = w.act3; ep.ldmask = G::FC_IN; ep.tag = "fc_dgrad";
  TB_TRY((gemm_simt<float, float, false, false>(w.dcore_in, w.wfcp, w.dact3, N, G::FC_IN, G::FC_OUT, pp.core,
                                                 G::FC_IN, G::FC_IN, ep, 1, nullptr, st)));
  // conv3: dact3 viewed as [M3, 64]
  TB_TRY(wgrad(w.dact3, G::C3, w.col3, false, G::KD3, G_ + pp.conv3_w, M3, G::C3, G::KD3, G::K3 * G::K3, G::C2, w, st, "conv3_wgrad"));
  TB_TRY(colsum(w.dact3, G_ + pp.conv3_b, M3, G::C3, G::C3, w.colsum_scratch, st));
  ep = GemmEpilogue(); ep.tag = "conv3_dgrad";
  TB_TRY((gemm_simt<float, float, false, false>(w.dact3, w.w3p, w.dcol3, M3, G::KD3, G::C3, G::C3, G::KD3, G::KD3, ep,
                                                 1, nullptr, st)));
  TB_TRY(col2im_f32_nhwc(w.dcol3, w.act2, w.dact2, N, G::H2, G::W2, G::C2, G::K3, G::K3, G::S3, st));
  // conv2
  TB_TRY(wgrad(w.dact2, G::C2, w.col2, false, G::KD2, G_ + pp.conv2_w, M2, G::C2, G::KD2, G::K2 * G::K2, G::C1, w, st, "conv2_wgrad"));
  TB_TRY(colsum(w.dact2, G_ + pp.conv2_b, M2, G::C2, G::C2, w.colsum_scratch, st));
  ep.tag = "conv2_dgrad";
  TB_TRY((gemm_simt<float, float, false, false>(w.dact2, w.w2p, w.dcol2, M2, G::KD2, G::C2, G::C2, G::KD2, G::KD2, ep,
                                                 1, nullptr, st)));
  TB_TRY(col2im_f32_nhwc(w.dcol2, w.act1, w.dact1, N, G::H1, G::W1, G::C1, G::K2, G::K2, G::S2, st));
  // conv1 (no input gradient needed)
  TB_TRY(wgrad(w.dact1, G::C1, w.col1, true, G::KD1, G_ + pp.conv1_w, M1, G::C1, G::KD1, 1, 1, w, st, "conv1_wgrad"));
  TB_TRY(colsum(w.dact1, G_ + pp.conv1_b, M1, G::C1, G::C1, w.colsum_scratch, st));
  return 0;
}

}  // namespace tb

// =======================================================================================
// C ABI
// =======================================================================================
using namespace tb;

extern "C" {

int64_t tb_atarinet_param_count(int num_actions, int num_values, int use_lstm) {
  return atari_params(num_actions, use_lstm, num_values).total;
}

int64_t tb_atarinet_grad_split(int num_actions, int use_lstm) {
  const AtariParams pp = atari_params(num_actions, use_lstm);
  return use_lstm ? pp.lstm[0][0] : pp.policy_w;  // first parameter after fc.bias
}

size_t tb_atarinet_workspace_bytes(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision) {
  return atari_ws(nullptr, T1 * B, T1, B, num_actions, use_lstm, precision).bytes;
}

// num_actions = 2D with 1 <= D <= TB_MAX_CONTINUOUS_DIM: the width of a continuous space's policy layer
static int continuous_width_ok(int num_actions, const char* who) {
  TB_REQUIRE(num_actions >= 2 && num_actions % 2 == 0 && num_actions / 2 <= TB_MAX_CONTINUOUS_DIM,
             "%s: num_actions = %d must be 2D with 1 <= D <= %d", who, num_actions, TB_MAX_CONTINUOUS_DIM);
  return 0;
}

// tb_atarinet_forward, with seg non-NULL tb_atarinet_forward_factored, and with clast_action non-NULL (last_action then
// NULL) tb_atarinet_forward_continuous
static int atarinet_forward_entry(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                                  const int64_t* last_action, const float* h0, const float* c0, const float* params,
                                  int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                                  void* workspace, void* stacked_scratch, float* policy_logits, float* baseline,
                                  float* hN, float* cN, void* stream, const ActionSegments* seg,
                                  const float* clast_action = nullptr) {
  TB_REQUIRE(num_values >= 1 && num_values <= kHeadsMaxValues, "atarinet_forward: num_values %d outside [1, %d]",
             num_values, kHeadsMaxValues);
  TB_REQUIRE(T1 >= 1 && B >= 1 && num_actions >= 1, "atarinet_forward: bad sizes T1=%lld B=%lld A=%d", (long long)T1,
             (long long)B, num_actions);
  TB_REQUIRE(frame && reward && (last_action || clast_action) && params && workspace && policy_logits && baseline,
             "atarinet_forward: null pointer");
  TB_REQUIRE(!use_lstm || (notdone && h0 && c0 && hN && cN), "atarinet_forward: LSTM needs notdone/h0/c0/hN/cN");
  TB_REQUIRE(precision >= 0 && precision <= 2,
             "atarinet_forward: precision must be 0 (fp32 SIMT), 1 (bf16 tensor cores) or 2 (split-bf16 tensor cores)");
  cudaStream_t st = (cudaStream_t)stream;
  // unstacked frames: the tensor-core backends' frame-image pass reads them directly; the fp32 one restacks them first
  if (done && !precision) {
    TB_REQUIRE(stacked_scratch, "atarinet_forward: the fp32 backend needs stacked_scratch "
                                "(tb_unstacked_scratch_bytes bytes)");
    uint8_t* stacked = static_cast<uint8_t*>(stacked_scratch);
    TB_TRY(restack_frames_u8(frame, done, T1, B, int64_t(AtariGeom::H0) * AtariGeom::W0, stacked, st));
    frame = stacked;
    done = nullptr;
  }
  return atarinet_forward(frame, done, reward, notdone, last_action, h0, c0, params, T1, B, num_actions, use_lstm, precision,
                          workspace, policy_logits, baseline, hN, cN, st, num_values, seg, clast_action);
}

int tb_atarinet_forward(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                        const int64_t* last_action, const float* h0, const float* c0, const float* params, int64_t T1,
                        int64_t B, int num_actions, int num_values, int use_lstm, int precision, void* workspace,
                        void* stacked_scratch, float* policy_logits, float* baseline, float* hN, float* cN,
                        void* stream) {
  return atarinet_forward_entry(frame, done, reward, notdone, last_action, h0, c0, params, T1, B, num_actions,
                                num_values, use_lstm, precision, workspace, stacked_scratch, policy_logits, baseline, hN,
                                cN, stream, nullptr);
}

int tb_atarinet_forward_factored(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                                 const int64_t* last_action, const float* h0, const float* c0, const float* params,
                                 int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                                 void* workspace, void* stacked_scratch, float* policy_logits, float* baseline,
                                 float* hN, float* cN, const tb_action_space* space, void* stream) {
  ActionSegments seg;
  TB_TRY(action_segments(space, num_actions, "atarinet_forward_factored", &seg));
  return atarinet_forward_entry(frame, done, reward, notdone, last_action, h0, c0, params, T1, B, num_actions,
                                num_values, use_lstm, precision, workspace, stacked_scratch, policy_logits, baseline, hN,
                                cN, stream, &seg);
}

// tb_atarinet_backward and, with Dc > 0, tb_atarinet_backward_continuous
static int atarinet_backward_entry(const float* grad_logits, const float* grad_baseline, const float* notdone,
                                   const float* params, int64_t T1, int64_t B, int num_actions, int num_values,
                                   int use_lstm, int precision, void* workspace, float* grads, int phase, void* stream,
                                   int Dc) {
  TB_REQUIRE(T1 >= 1 && B >= 1 && num_actions >= 1 && num_values >= 1 && num_values <= kHeadsMaxValues,
             "atarinet_backward: bad sizes");
  TB_REQUIRE(grad_logits && grad_baseline && params && workspace && grads, "atarinet_backward: null pointer");
  TB_REQUIRE(!use_lstm || notdone, "atarinet_backward: LSTM needs notdone");
  TB_REQUIRE(precision >= 0 && precision <= 2, "atarinet_backward: precision must be 0, 1 or 2");
  TB_REQUIRE(phase >= 1 && phase <= 3,
             "atarinet_backward: phase must be 1 (heads + LSTM), 2 (conv/fc trunk) or 3 (the whole backward)");
  return atarinet_backward(grad_logits, grad_baseline, notdone, params, T1, B, num_actions, use_lstm, precision, workspace,
                           grads, (cudaStream_t)stream, phase, num_values, Dc);
}

int tb_atarinet_backward(const float* grad_logits, const float* grad_baseline, const float* notdone,
                         const float* params, int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm,
                         int precision, void* workspace, float* grads, int phase, void* stream) {
  return atarinet_backward_entry(grad_logits, grad_baseline, notdone, params, T1, B, num_actions, num_values, use_lstm,
                                 precision, workspace, grads, phase, stream, 0);
}

int64_t tb_atarinet_param_count_continuous(int num_actions, int num_values, int use_lstm) {
  if (continuous_width_ok(num_actions, "atarinet_param_count_continuous")) return -1;
  return atari_params(num_actions, use_lstm, num_values, num_actions / 2).total;
}

size_t tb_atarinet_workspace_bytes_continuous(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision) {
  if (continuous_width_ok(num_actions, "atarinet_workspace_bytes_continuous")) return 0;
  return atari_ws(nullptr, T1 * B, T1, B, num_actions, use_lstm, precision, num_actions / 2).bytes;
}

int tb_atarinet_forward_continuous(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                                   const float* last_action, const float* h0, const float* c0, const float* params,
                                   int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                                   void* workspace, void* stacked_scratch, float* policy_logits, float* baseline,
                                   float* hN, float* cN, void* stream) {
  TB_TRY(continuous_width_ok(num_actions, "atarinet_forward_continuous"));
  TB_REQUIRE(last_action, "atarinet_forward_continuous: null last_action");
  return atarinet_forward_entry(frame, done, reward, notdone, nullptr, h0, c0, params, T1, B, num_actions, num_values,
                                use_lstm, precision, workspace, stacked_scratch, policy_logits, baseline, hN, cN, stream,
                                nullptr, last_action);
}

int tb_atarinet_backward_continuous(const float* grad_logits, const float* grad_baseline, const float* notdone,
                                    const float* params, int64_t T1, int64_t B, int num_actions, int num_values,
                                    int use_lstm, int precision, void* workspace, float* grads, int phase, void* stream) {
  TB_TRY(continuous_width_ok(num_actions, "atarinet_backward_continuous"));
  return atarinet_backward_entry(grad_logits, grad_baseline, notdone, params, T1, B, num_actions, num_values, use_lstm,
                                 precision, workspace, grads, phase, stream, num_actions / 2);
}

}  // extern "C"
