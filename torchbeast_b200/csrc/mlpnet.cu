// MLPNet forward / backward for vector observations (sm_90a), behind the C ABI.
//
// AtariNet with its conv trunk and fc replaced by dense layers (include/torchbeast_b200.h, "MLPNet"):
//   f32 obs [T1,B,O] -> [clamp((x - mean) * inv_std, -10, 10)] -> relu(x W_i^T + b_i) for each hidden width ->
//   cat[x, clip(reward), last-action encoding] -> [2-layer LSTM] -> policy / baseline.
//
// Structure: one staging kernel reads the observations once and writes the first GEMM's operand (fp32, or bf16 hi[/lo]
// planes with the row stride padded to a multiple of 8), normalised from the float64 running statistics; every dense
// layer is one GEMM with a fused bias + ReLU epilogue (gemm_simt at fp32, gemm_tc_bf16 otherwise), the last one writing
// the first H_last columns of the core input.  Core extras, LSTM and heads are AtariNet's.  The backward masks and
// sums the bias gradients (colsum / colsum_bf16), runs each weight gradient as a split-K GEMM over the rows and each
// input gradient with the ReLU mask of the layer below in its epilogue; the first layer needs no input gradient.
// The statistics kernels (tb_obs_norm_sums / tb_obs_norm_update) are at the end.
#include <cuda_bf16.h>

#include "gemm_simt.cuh"
#include "gemm_tc.cuh"
#include "heads.cuh"
#include "lstm.cuh"
#include "net_kernels.cuh"

namespace tb {

namespace {

constexpr int kMlpThreads = 256;

int64_t ld8(int64_t n) { return (n + 7) & ~int64_t(7); }

unsigned grid_of(int64_t total, int threads) {
  int64_t b = (total + threads - 1) / threads;
  if (b > int64_t(kNumSMs) * 16) b = int64_t(kNumSMs) * 16;
  return unsigned(b < 1 ? 1 : b);
}

// The action space of one call, from the entry point's (space, continuous_dim) arguments.
struct MlpSpace {
  const ActionSegments* seg = nullptr;  // a factored space
  ActionSegments segs;
  int Dc = 0;                           // a continuous space of Dc dimensions (A = 2 Dc)
  int core_actions = 0;                 // the core's last-action columns: A, or Dc
};

struct MlpParams {  // offsets (in floats) into the flat parameter / gradient buffers
  int64_t w[TB_MLP_MAX_LAYERS], b[TB_MLP_MAX_LAYERS];
  int64_t lstm[2][4];
  int64_t policy_w, policy_b, baseline_w, baseline_b, total;
  int core;  // H_last + 1 + core_actions
};

int check_config(const tb_mlp_config* c, const tb_action_space* space, int continuous_dim, MlpSpace* sp,
                 const char* who) {
  TB_REQUIRE(c, "%s: null config", who);
  TB_REQUIRE(c->obs_dim >= 1 && c->obs_dim <= TB_MLP_MAX_OBS, "%s: obs_dim %d outside [1, %d]", who, c->obs_dim,
             TB_MLP_MAX_OBS);
  TB_REQUIRE(c->num_layers >= 1 && c->num_layers <= TB_MLP_MAX_LAYERS, "%s: num_layers %d outside [1, %d]", who,
             c->num_layers, TB_MLP_MAX_LAYERS);
  for (int i = 0; i < c->num_layers; ++i)
    TB_REQUIRE(c->hidden[i] >= 8 && c->hidden[i] <= TB_MLP_MAX_WIDTH && c->hidden[i] % 8 == 0,
               "%s: hidden width %d (layer %d) must be a multiple of 8 in [8, %d]", who, c->hidden[i], i,
               TB_MLP_MAX_WIDTH);
  TB_REQUIRE(c->num_actions >= 1 && c->num_actions <= 31, "%s: num_actions %d outside [1, 31]", who, c->num_actions);
  TB_REQUIRE(c->num_values >= 1 && c->num_values <= kHeadsMaxValues, "%s: num_values %d outside [1, %d]", who,
             c->num_values, kHeadsMaxValues);
  TB_REQUIRE(!(space && continuous_dim), "%s: a factored space and a continuous dimension at once", who);
  *sp = MlpSpace();
  sp->core_actions = c->num_actions;
  if (space) {
    TB_TRY(action_segments(space, c->num_actions, who, &sp->segs));
    sp->seg = &sp->segs;
  } else if (continuous_dim) {
    TB_REQUIRE(continuous_dim >= 1 && c->num_actions == 2 * continuous_dim,
               "%s: continuous_dim %d needs num_actions = 2D, got %d", who, continuous_dim, c->num_actions);
    sp->Dc = continuous_dim;
    sp->core_actions = continuous_dim;
  }
  const int core = c->hidden[c->num_layers - 1] + 1 + sp->core_actions;
  TB_REQUIRE(!c->use_lstm || core <= TB_LSTM_MAX_HIDDEN, "%s: the LSTM needs H_last + 1 + %d <= %d, got %d", who,
             sp->core_actions, TB_LSTM_MAX_HIDDEN, core);
  return 0;
}

MlpParams mlp_params(const tb_mlp_config& c, const MlpSpace& sp) {
  MlpParams p;
  int64_t o = 0;
  auto take = [&](int64_t n) { int64_t r = o; o += n; return r; };
  int64_t in = c.obs_dim;
  for (int i = 0; i < TB_MLP_MAX_LAYERS; ++i) p.w[i] = p.b[i] = -1;
  for (int i = 0; i < c.num_layers; ++i) {
    p.w[i] = take(int64_t(c.hidden[i]) * in);
    p.b[i] = take(c.hidden[i]);
    in = c.hidden[i];
  }
  p.core = c.hidden[c.num_layers - 1] + 1 + sp.core_actions;
  for (int l = 0; l < 2; ++l)
    for (int k = 0; k < 4; ++k) p.lstm[l][k] = -1;
  if (c.use_lstm) {
    const int64_t H = p.core;
    for (int l = 0; l < 2; ++l) {
      p.lstm[l][0] = take(4 * H * H); p.lstm[l][1] = take(4 * H * H);
      p.lstm[l][2] = take(4 * H); p.lstm[l][3] = take(4 * H);
    }
  }
  p.policy_w = take(int64_t(c.num_actions) * p.core); p.policy_b = take(c.num_actions);
  p.baseline_w = take(int64_t(c.num_values) * p.core); p.baseline_b = take(c.num_values);
  p.total = o;
  return p;
}

// A layer input / output buffer: fp32 (precision 0) or bf16 with, at precision 2, the lo plane `lo` elements behind.
struct Buf {
  void* p = nullptr; int64_t lo = 0;
  float* f() const { return static_cast<float*>(p); }
  __nv_bfloat16* h() const { return static_cast<__nv_bfloat16*>(p); }
};

struct MlpWs {
  float *core_in, *core_out, *dcore_out, *dcore_in, *splitk, *colsum_scratch;
  Buf x[TB_MLP_MAX_LAYERS];    // x[i]: the input of layer i (x[0] the staged observations, row stride ldx[i])
  Buf dx[TB_MLP_MAX_LAYERS];   // dx[i]: the gradient at x[i], i >= 1 (masked by x[i] > 0)
  Buf wb[TB_MLP_MAX_LAYERS];   // tensor-core backends: bf16 weights [H_i, ldx[i]], pad columns zero
  Buf dlast;                   // tensor-core backends: bf16 copy of the last layer's masked output gradient [N, H_last]
  int64_t ldx[TB_MLP_MAX_LAYERS];
  LstmWs lstm;
  size_t bytes;
};

MlpWs mlp_ws(void* base, const tb_mlp_config& c, const MlpParams& pp, int64_t T1, int64_t B, int precision) {
  MlpWs w = MlpWs();
  size_t off = 0;
  auto take = [&](size_t nbytes) {
    void* p = base ? static_cast<char*>(base) + off : nullptr;
    off += (nbytes + 255) & ~size_t(255);
    return p;
  };
  const int64_t N = T1 * B;
  auto takef = [&](int64_t n) { return static_cast<float*>(take(size_t(n) * sizeof(float))); };
  auto takeb = [&](int64_t n) {  // a layer buffer of n elements in the precision's format
    Buf b;
    if (!precision) { b.p = takef(n); return b; }
    const size_t plane = (size_t(n) * 2 + 255) & ~size_t(255);
    b.p = take(precision == 2 ? 2 * plane : plane);
    b.lo = precision == 2 ? int64_t(plane / 2) : 0;
    return b;
  };
  w.core_in = takef(N * pp.core);
  w.core_out = c.use_lstm ? takef(N * pp.core) : w.core_in;
  w.dcore_out = takef(N * pp.core);
  w.dcore_in = c.use_lstm ? takef(N * pp.core) : w.dcore_out;
  const int L = c.num_layers;
  for (int i = 0; i < L; ++i) {
    const int64_t in = i ? c.hidden[i - 1] : c.obs_dim;
    w.ldx[i] = precision ? ld8(in) : in;
    w.x[i] = takeb(N * w.ldx[i]);
    if (i) w.dx[i] = takeb(N * w.ldx[i]);
    if (precision) w.wb[i] = takeb(int64_t(c.hidden[i]) * w.ldx[i]);
  }
  if (precision) w.dlast = takeb(N * c.hidden[L - 1]);
  w.splitk = takef(kSplitKScratchFloats);
  w.colsum_scratch = takef(colsum_scratch_floats(4 * int64_t(pp.core) > 512 ? 4 * int64_t(pp.core) : 512));
  if (c.use_lstm) {
    const size_t lbytes = lstm_ws_bytes(T1, B, pp.core, pp.core, 2, precision);
    w.lstm = lstm_ws(take(lbytes), T1, B, pp.core, pp.core, 2, precision);
  }
  w.bytes = off;
  return w;
}

// ---------------------------------------------------------------------------------------
// operand staging: x = obs, or clamp((obs - mean_f) * inv_std_f, -10, 10) with the per-feature fp32 statistics
// mean_f = float(mean), inv_std_f = float(1 / sqrt(var + 1e-8)) formed in float64 (a NaN passes the clamp as NaN)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMlpThreads) obs_stage_kernel(const float* __restrict__ obs, int64_t N, int O,
                                                                const double* __restrict__ mean,
                                                                const double* __restrict__ var, float* __restrict__ out32,
                                                                __nv_bfloat16* __restrict__ out16, int64_t lo, int64_t ld) {
  extern __shared__ float s_stat[];  // [O] mean_f, [O] inv_std_f
  const bool norm = mean != nullptr;
  if (norm) {
    for (int j = threadIdx.x; j < O; j += blockDim.x) {
      s_stat[j] = float(mean[j]);
      s_stat[O + j] = float(1.0 / sqrt(var[j] + TB_OBS_NORM_EPS));
    }
    __syncthreads();
  }
  const int64_t total = N * ld;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / ld;
    const int j = int(i - n * ld);
    float x = 0.0f;  // pad columns [O, ld) are zero
    if (j < O) {
      x = __ldg(obs + n * O + j);
      if (norm) {
        x = __fmul_rn(__fsub_rn(x, s_stat[j]), s_stat[O + j]);
        x = x < -TB_OBS_NORM_CLIP ? -TB_OBS_NORM_CLIP : (x > TB_OBS_NORM_CLIP ? TB_OBS_NORM_CLIP : x);
      }
    }
    if (out32) {
      out32[i] = x;
    } else {
      const __nv_bfloat16 h = __float2bfloat16_rn(x);
      out16[i] = h;
      if (lo) out16[lo + i] = __float2bfloat16_rn(x - __bfloat162float(h));
    }
  }
}

int obs_stage(const float* obs, int64_t N, int O, const double* mean, const double* var, int precision, void* out,
              int64_t lo, cudaStream_t st) {
  ProfScope prof("obs_stage", st);
  const int64_t ld = precision ? ld8(O) : O;
  if (N == 0) return 0;
  const size_t smem = mean ? size_t(2) * O * sizeof(float) : 0;
  obs_stage_kernel<<<grid_of(N * ld, kMlpThreads), kMlpThreads, smem, st>>>(
      obs, N, O, mean, var, precision ? nullptr : static_cast<float*>(out),
      precision ? static_cast<__nv_bfloat16*>(out) : nullptr, lo, ld);
  return check_launch("obs_stage_kernel");
}

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
int mlp_forward(const float* obs, const float* reward, const float* notdone, const void* last_action, const float* h0,
                const float* c0, const float* P, const double* mean, const double* var, const tb_mlp_config& c,
                const MlpSpace& sp, int64_t T1, int64_t B, int precision, void* workspace, float* logits,
                float* baseline, float* hN, float* cN, cudaStream_t st) {
  const int64_t N = T1 * B;
  const MlpParams pp = mlp_params(c, sp);
  MlpWs w = mlp_ws(workspace, c, pp, T1, B, precision);
  const int L = c.num_layers;
  TB_TRY(obs_stage(obs, N, c.obs_dim, c.normalize ? mean : nullptr, var, precision, w.x[0].p, w.x[0].lo, st));
  for (int i = 0; i < L; ++i) {
    const int64_t in = i ? c.hidden[i - 1] : c.obs_dim, out = c.hidden[i];
    const bool last = i == L - 1;
    if (precision) {
      TB_TRY(pack_weights_bf16(P + pp.w[i], w.wb[i].p, out, 1, int(in), w.ldx[i], st, w.wb[i].lo));
      TcEpilogue te;
      if (last) { te.C = w.core_in; te.ldc = pp.core; }
      else { te.C16 = w.x[i + 1].h(); te.ldc16 = w.ldx[i + 1]; te.c16_lo = w.x[i + 1].lo; }
      te.bias = P + pp.b[i]; te.relu = 1; te.tag = "mlp_fwd";
      te.a_lo = w.x[i].lo; te.b_lo = w.wb[i].lo;
      TB_TRY(gemm_tc_bf16(w.x[i].p, w.wb[i].p, N, out, in, w.ldx[i], w.ldx[i], te, st));
    } else {
      GemmEpilogue ep; ep.bias = P + pp.b[i]; ep.relu = 1; ep.tag = "mlp_fwd";
      TB_TRY((gemm_simt<float, float, false, true>(w.x[i].f(), P + pp.w[i], last ? w.core_in : w.x[i + 1].f(), N, out,
                                                    in, w.ldx[i], in, last ? pp.core : w.ldx[i + 1], ep, 1, nullptr,
                                                    st)));
    }
  }
  const int F = c.hidden[L - 1];
  if (sp.Dc)
    TB_TRY(core_extras_continuous(w.core_in, pp.core, N, F, reward, static_cast<const float*>(last_action), sp.Dc, st));
  else
    TB_TRY(core_extras(w.core_in, pp.core, N, F, reward, static_cast<const int64_t*>(last_action), c.num_actions, st,
                       sp.seg));
  if (c.use_lstm) {
    LstmParams lp;
    for (int l = 0; l < 2; ++l) {
      lp.w_ih[l] = P + pp.lstm[l][0]; lp.w_hh[l] = P + pp.lstm[l][1];
      lp.b_ih[l] = P + pp.lstm[l][2]; lp.b_hh[l] = P + pp.lstm[l][3];
    }
    TB_TRY(lstm_forward(w.core_in, notdone, h0, c0, lp, T1, B, pp.core, pp.core, 2, w.lstm, w.core_out, hN, cN, precision,
                        st));
  }
  return heads_forward(w.core_out, pp.core, P + pp.policy_w, P + pp.policy_b, P + pp.baseline_w, P + pp.baseline_b, N,
                       pp.core, c.num_actions, logits, baseline, st, c.num_values);
}

// ---------------------------------------------------------------------------------------
// backward: consumes the activations the forward left in the workspace
// ---------------------------------------------------------------------------------------
int tc_splits(int64_t M, int64_t N, int64_t K) {
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

int mlp_backward(const float* grad_logits, const float* grad_baseline, const float* notdone, const float* P,
                 const tb_mlp_config& c, const MlpSpace& sp, int64_t T1, int64_t B, int precision, void* workspace,
                 float* G, cudaStream_t st) {
  const int64_t N = T1 * B;
  const MlpParams pp = mlp_params(c, sp);
  MlpWs w = mlp_ws(workspace, c, pp, T1, B, precision);
  const int L = c.num_layers, A = c.num_actions, V = c.num_values;
  TB_REQUIRE(heads_scratch_floats(N, pp.core, A, V) <= kSplitKScratchFloats, "mlpnet_backward: heads scratch too small");
  TB_TRY(heads_backward(w.core_out, pp.core, P + pp.policy_w, P + pp.baseline_w, grad_logits, grad_baseline, N, pp.core,
                        A, w.dcore_out, pp.core, G + pp.policy_w, G + pp.policy_b, G + pp.baseline_w, G + pp.baseline_b,
                        w.splitk, st, V));
  if (c.use_lstm) {
    LstmParams lp; LstmGrads lg;
    for (int l = 0; l < 2; ++l) {
      lp.w_ih[l] = P + pp.lstm[l][0]; lp.w_hh[l] = P + pp.lstm[l][1];
      lp.b_ih[l] = P + pp.lstm[l][2]; lp.b_hh[l] = P + pp.lstm[l][3];
      lg.w_ih[l] = G + pp.lstm[l][0]; lg.w_hh[l] = G + pp.lstm[l][1];
      lg.b_ih[l] = G + pp.lstm[l][2]; lg.b_hh[l] = G + pp.lstm[l][3];
    }
    TB_TRY(lstm_backward(w.dcore_out, w.core_in, notdone, lp, lg, T1, B, pp.core, pp.core, 2, w.lstm, w.dcore_in,
                         w.splitk, w.colsum_scratch, precision, st));
  }
  // last layer: its output is the first H_last columns of the core input, its gradient those of dcore_in
  const int64_t HL = c.hidden[L - 1];
  TB_TRY(relu_mask_inplace(w.dcore_in, w.core_in, N, HL, pp.core, pp.core, st));
  TB_TRY(colsum(w.dcore_in, G + pp.b[L - 1], N, HL, pp.core, w.colsum_scratch, st));
  if (precision) TB_TRY(f32_to_bf16(w.dcore_in, w.dlast.p, N, HL, pp.core, HL, st, w.dlast.lo));
  for (int i = L - 1; i >= 0; --i) {
    const int64_t in = i ? c.hidden[i - 1] : c.obs_dim, out = c.hidden[i];
    if (i < L - 1) {  // a hidden layer's output gradient: dx[i + 1], masked by the input-gradient epilogue above
      if (precision)
        TB_TRY(colsum_bf16(w.dx[i + 1].p, G + pp.b[i], N, out, out, w.colsum_scratch, st, w.dx[i + 1].lo));
      else
        TB_TRY(colsum(w.dx[i + 1].f(), G + pp.b[i], N, out, out, w.colsum_scratch, st));
    }
    if (precision) {
      const Buf& dy = i == L - 1 ? w.dlast : w.dx[i + 1];
      // dW [out, in] = dY^T . X: both operands as stored (MN-major), split-K over the rows
      TcEpilogue te;
      te.C = G + pp.w[i]; te.ldc = in; te.tag = "mlp_wgrad"; te.a_lo = dy.lo; te.b_lo = w.x[i].lo;
      TB_TRY(gemm_tc_bf16_ex(dy.p, w.x[i].p, out, in, N, out, w.ldx[i], true, true, te, tc_splits(out, in, N), w.splitk,
                             st));
      if (i) {  // dX = dY . W, times the ReLU mask of X (the bf16 hi plane the forward wrote)
        te = TcEpilogue();
        te.C16 = w.dx[i].h(); te.ldc16 = w.ldx[i]; te.c16_lo = w.dx[i].lo; te.mask16 = w.x[i].h(); te.ldmask = w.ldx[i];
        te.tag = "mlp_dgrad"; te.a_lo = dy.lo; te.b_lo = w.wb[i].lo;
        TB_TRY(gemm_tc_bf16_ex(dy.p, w.wb[i].p, N, in, out, out, w.ldx[i], false, true, te, 1, nullptr, st));
      }
    } else {
      const float* dy = i == L - 1 ? w.dcore_in : w.dx[i + 1].f();
      const int64_t ldy = i == L - 1 ? pp.core : out;
      GemmEpilogue ep; ep.tag = "mlp_wgrad";
      const int splits = simt_splits(out, in, N, kSplitKScratchFloats, 128);
      TB_TRY((gemm_simt<float, float, true, false>(dy, w.x[i].f(), G + pp.w[i], out, in, N, ldy, w.ldx[i], in, ep, splits,
                                                    w.splitk, st)));
      if (i) {
        ep = GemmEpilogue(); ep.mask = w.x[i].f(); ep.ldmask = w.ldx[i]; ep.tag = "mlp_dgrad";
        TB_TRY((gemm_simt<float, float, false, false>(dy, P + pp.w[i], w.dx[i].f(), N, in, out, ldy, in, w.ldx[i], ep, 1,
                                                       nullptr, st)));
      }
    }
  }
  if (c.use_lstm && precision) return lstm_backward_join(st);  // the LSTM weight-gradient GEMMs ran beside the torso's
  return 0;
}

// ---------------------------------------------------------------------------------------
// running observation statistics
// ---------------------------------------------------------------------------------------
// CTA j owns feature j and walks the rows (t, b), t in [t_begin, T1), b < Bf, in a fixed pattern (thread k takes rows k,
// k + 256, ...; warps, then the CTA folded in index order): bit-identical from run to run without atomics.
__global__ void __launch_bounds__(kMlpThreads) obs_norm_sums_kernel(const float* __restrict__ obs, int64_t B, int O,
                                                                    int64_t t_begin, int64_t rows, int64_t Bf,
                                                                    double* __restrict__ sums) {
  __shared__ double sm[kMlpThreads / kWarp][3];
  const int j = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double n = 0.0, s = 0.0, s2 = 0.0;
  for (int64_t r = tid; r < rows; r += kMlpThreads) {
    const int64_t t = t_begin + r / Bf, b = r % Bf;
    const double x = double(__ldg(obs + (t * B + b) * O + j));
    if (isfinite(x)) { n += 1.0; s += x; s2 += x * x; }
  }
  n = warp_sum(n); s = warp_sum(s); s2 = warp_sum(s2);
  if (lane == 0) { sm[warp][0] = n; sm[warp][1] = s; sm[warp][2] = s2; }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0, d = 0.0;
    for (int k = 0; k < kMlpThreads / kWarp; ++k) { a += sm[k][0]; b += sm[k][1]; d += sm[k][2]; }
    sums[j] = a; sums[O + j] = b; sums[2 * O + j] = d;
  }
}

__global__ void obs_norm_update_kernel(const double* __restrict__ sums, double* count, double* mean, double* var, int O) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= O) return;
  const double nb = sums[j];
  if (!(nb > 0.0)) return;
  const double mb = sums[O + j] / nb;
  const double vb = fmax(sums[2 * O + j] / nb - mb * mb, 0.0);
  const double n = count[j], m = mean[j], v = var[j];
  const double tot = n + nb;
  const double delta = mb - m;
  mean[j] = m + delta * nb / tot;
  var[j] = (v * n + vb * nb + delta * delta * n * nb / tot) / tot;
  count[j] = tot;
}

}  // namespace

}  // namespace tb

// =======================================================================================
// C ABI
// =======================================================================================
using namespace tb;

extern "C" {

int64_t tb_mlpnet_param_count(const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim) {
  MlpSpace sp;
  if (check_config(cfg, space, continuous_dim, &sp, "mlpnet_param_count")) return -1;
  return mlp_params(*cfg, sp).total;
}

size_t tb_mlpnet_workspace_bytes(const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim, int64_t T1,
                                 int64_t B, int precision) {
  MlpSpace sp;
  if (check_config(cfg, space, continuous_dim, &sp, "mlpnet_workspace_bytes")) return 0;
  if (T1 < 1 || B < 1 || precision < 0 || precision > 2) {
    set_error("mlpnet_workspace_bytes: bad sizes T1=%lld B=%lld or precision %d", (long long)T1, (long long)B, precision);
    return 0;
  }
  return mlp_ws(nullptr, *cfg, mlp_params(*cfg, sp), T1, B, precision).bytes;
}

int tb_mlpnet_forward(const float* obs, const float* reward, const float* notdone, const void* last_action,
                      const float* h0, const float* c0, const float* params, const double* obs_mean,
                      const double* obs_var, const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim,
                      int64_t T1, int64_t B, int precision, void* workspace, float* policy_logits, float* baseline,
                      float* hN, float* cN, void* stream) {
  MlpSpace sp;
  TB_TRY(check_config(cfg, space, continuous_dim, &sp, "mlpnet_forward"));
  TB_REQUIRE(T1 >= 1 && B >= 1, "mlpnet_forward: bad sizes T1=%lld B=%lld", (long long)T1, (long long)B);
  TB_REQUIRE(obs && reward && last_action && params && workspace && policy_logits && baseline,
             "mlpnet_forward: null pointer");
  TB_REQUIRE(!cfg->normalize || (obs_mean && obs_var), "mlpnet_forward: normalisation needs obs_mean / obs_var");
  TB_REQUIRE(!cfg->use_lstm || (notdone && h0 && c0 && hN && cN), "mlpnet_forward: LSTM needs notdone/h0/c0/hN/cN");
  TB_REQUIRE(precision >= 0 && precision <= 2,
             "mlpnet_forward: precision must be 0 (fp32 SIMT), 1 (bf16 tensor cores) or 2 (split-bf16 tensor cores)");
  return mlp_forward(obs, reward, notdone, last_action, h0, c0, params, obs_mean, obs_var, *cfg, sp, T1, B, precision,
                     workspace, policy_logits, baseline, hN, cN, (cudaStream_t)stream);
}

int tb_mlpnet_backward(const float* grad_logits, const float* grad_baseline, const float* notdone, const float* params,
                       const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim, int64_t T1,
                       int64_t B, int precision, void* workspace, float* grads, void* stream) {
  MlpSpace sp;
  TB_TRY(check_config(cfg, space, continuous_dim, &sp, "mlpnet_backward"));
  TB_REQUIRE(T1 >= 1 && B >= 1, "mlpnet_backward: bad sizes T1=%lld B=%lld", (long long)T1, (long long)B);
  TB_REQUIRE(grad_logits && grad_baseline && params && workspace && grads, "mlpnet_backward: null pointer");
  TB_REQUIRE(!cfg->use_lstm || notdone, "mlpnet_backward: LSTM needs notdone");
  TB_REQUIRE(precision >= 0 && precision <= 2, "mlpnet_backward: precision must be 0, 1 or 2");
  return mlp_backward(grad_logits, grad_baseline, notdone, params, *cfg, sp, T1, B, precision, workspace, grads,
                      (cudaStream_t)stream);
}

int tb_obs_stage(const float* obs, int64_t N, int O, const double* obs_mean, const double* obs_var, int precision,
                 void* out, void* stream) {
  TB_REQUIRE(N >= 0 && O >= 1 && O <= TB_MLP_MAX_OBS, "obs_stage: bad sizes N=%lld O=%d", (long long)N, O);
  TB_REQUIRE(precision >= 0 && precision <= 2, "obs_stage: precision must be 0, 1 or 2");
  TB_REQUIRE((obs_mean == nullptr) == (obs_var == nullptr), "obs_stage: give both obs_mean and obs_var, or neither");
  TB_REQUIRE(N == 0 || (obs && out), "obs_stage: null pointer");
  return obs_stage(obs, N, O, obs_mean, obs_var, precision, out, precision == 2 ? N * ld8(O) : 0,
                   (cudaStream_t)stream);
}

int tb_obs_norm_sums(const float* obs, int64_t T1, int64_t B, int O, int64_t t_begin, int64_t Bf, double* sums,
                     void* stream) {
  TB_REQUIRE(O >= 1 && O <= TB_MLP_MAX_OBS && T1 >= 0 && B >= 0 && t_begin >= 0 && t_begin <= T1 && Bf >= 0 && Bf <= B,
             "obs_norm_sums: bad sizes T1=%lld B=%lld O=%d t_begin=%lld Bf=%lld", (long long)T1, (long long)B, O,
             (long long)t_begin, (long long)Bf);
  TB_REQUIRE(sums && (obs || (T1 - t_begin) * Bf == 0), "obs_norm_sums: null pointer");
  ProfScope prof("obs_norm_sums", (cudaStream_t)stream);
  obs_norm_sums_kernel<<<unsigned(O), kMlpThreads, 0, (cudaStream_t)stream>>>(obs, B, O, t_begin, (T1 - t_begin) * Bf,
                                                                                Bf > 0 ? Bf : 1, sums);
  return check_launch("obs_norm_sums_kernel");
}

int tb_obs_norm_update(const double* sums, double* count, double* mean, double* var, int O, void* stream) {
  TB_REQUIRE(O >= 1 && O <= TB_MLP_MAX_OBS, "obs_norm_update: O = %d outside [1, %d]", O, TB_MLP_MAX_OBS);
  TB_REQUIRE(sums && count && mean && var, "obs_norm_update: null pointer");
  ProfScope prof("obs_norm_update", (cudaStream_t)stream);
  obs_norm_update_kernel<<<unsigned((O + 255) / 256), 256, 0, (cudaStream_t)stream>>>(sums, count, mean, var, O);
  return check_launch("obs_norm_update_kernel");
}

}  // extern "C"
