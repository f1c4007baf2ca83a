// Stacked LSTM over the unroll with per-step done-reset (monobeast.py:603-611,
// polybeast_learner.py:241-249): declarations.  See lstm.cu.
#pragma once
#include "common.cuh"

namespace tb {

constexpr int kLstmMaxLayers = 2;
constexpr int64_t kSplitKScratchFloats = int64_t(8) << 20;  // 32 MB: the split-K GEMM scratch the callers provide

struct LstmParams {  // torch.nn.LSTM layout: weight_ih [4H, In], weight_hh [4H, H], gate order i,f,g,o
  const float* w_ih[kLstmMaxLayers]; const float* w_hh[kLstmMaxLayers];
  const float* b_ih[kLstmMaxLayers]; const float* b_hh[kLstmMaxLayers];
};
struct LstmGrads {
  float* w_ih[kLstmMaxLayers]; float* w_hh[kLstmMaxLayers];
  float* b_ih[kLstmMaxLayers]; float* b_hh[kLstmMaxLayers];
};

struct LstmLayerWs {
  float* gates;   // [T1*B, 4H]  pre-activations, overwritten by activated i,f,g,o
  float* hs;      // [T1*B, H]   h_t
  float* cs;      // [T1*B, H]   c_t
  float* hm;      // [T1*B, Hp]  h_{t-1} * notdone_t (recurrent input used at step t), rows zero-padded to Hp
  float* cm;      // [T1*B, H]   c_{t-1} * notdone_t
  void* xb;       // bf16 [T1*B, ld16(In)]   this layer's input (tensor-core backend)
  void* wihb;     // bf16 [4H, ld16(In)]     W_ih
  void* dgb;      // bf16 [T1*B, ld16(4H)]   gate gradients
  void* hmb;      // bf16 [T1*B, ld16(H)]    masked recurrent inputs
  int64_t xb_lo = 0, wihb_lo = 0, dgb_lo = 0, hmb_lo = 0;  // precision 2 (split-bf16): element offsets of the lo planes
  int64_t hq_lo = 0, hmq_lo = 0, dgq_lo = 0;               // same for the recurrence kernels' exchange / masked-h planes
  float* gact = nullptr;  // (precision 2) activated gates, CTA-blocked [T1][ceil(H/4)][32][16] - see lstm2_fwd_wave_split_kernel
  float* csb = nullptr;   // (precision 2) cell state, CTA-blocked [T1+1][ceil(H/4)][32][4]: slot 0 = c0, slot t+1 = c_t
  void* hmq;      // bf16 [T1*B, Hq]         masked recurrent inputs written by the tensor-core recurrence (Hq = mma_hq(H))
  void* hq;       // bf16 [(T1+1)*B, Hq]     raw h (slot 0 = initial state) written by the two-layer wavefront kernels
  void* hx = nullptr;  // (precision 2, two layers) the same h as hi / lo planes, slice-blocked for the split wavefront's
                       // exchange: [T1+1][kXSlotE] - see lstm2_fwd_wave_split_kernel
  void* dgq;      // bf16 [2][4, B, Hq]      this step's gate gradients for the tensor-core backward recurrence
  void* dgx = nullptr;  // (precision 2, two layers) the split backward wavefront's gate-gradient exchange ring, hi / lo
                        // planes blocked by k-group: [2 slots][k-group][kBwdGroupE] - see lstm2_bwd_wave_split_kernel
  float* wp;      // [4H+4, Hp]  W_hh with rows zero-padded to Hp floats (16-byte multiples for bulk copies)
  float* dgates;  // [T1*B, 4H]  backward: d pre-activations
  float* bsum;    // [4H]        b_ih + b_hh
  float* w_hh_t;  // [H+4, 4*Hp] W_hh^T, gate segments zero-padded to Hp: wt[k][g*Hp+j] = W_hh[g*H+j][k]
};

struct LstmWs {
  LstmLayerWs layer[kLstmMaxLayers];
  float* dh;      // [B, H] carry
  float* dc;      // [B, H] carry
  float* dx_mid;  // [T1*B, H] gradient w.r.t. the output of layer 0 (input of layer 1)
  unsigned* sync; // [64] grid-barrier counters of the persistent recurrence kernels (zeroed per launch)
  float* bwd_rec = nullptr;  // (precision 2, two layers) the split backward's dh partials: [role][2 slots][k-groups][column blocks][32][8]
  float* bwd_dxr = nullptr;  // (precision 2, two layers) its dL/dh_lower partials, upper -> lower role: [2][k-groups][column blocks][32][8]
  unsigned* flags; // [1024] per-CTA step flags of the split-precision recurrence kernels (forward [0,512), backward [512,1024))
  float* wg_scratch;  // split-K scratch private to the weight-gradient GEMMs (two layers, bf16 backend): lets them run on a
                      // side stream beside the caller's trunk backward, which uses the caller's scratch
  float* dgp;     // [2][4, B, Hp] (double-buffered for the persistent backward)
  //               this step's gate gradients, gate-major and zero padded (recurrent product operand)
  int Hp = 0;     // padded row length of hm / wp
  size_t bytes = 0;
};

size_t lstm_ws_bytes(int64_t T1, int64_t B, int In, int H, int layers, int precision);
LstmWs lstm_ws(void* base, int64_t T1, int64_t B, int In, int H, int layers, int precision);

// precision: 0 = fp32 SIMT GEMMs and the fp32 recurrence kernels; 1 = bf16 wgmma GEMMs for the hoisted projections and
// bf16 mma.sync operands in the recurrence where it fits; 2 = split-bf16 (hi/lo planes, 3 MMAs) wgmma GEMMs, and a
// split-bf16 recurrence where one fits (the two-layer wavefront, or the 16-CTA cluster kernels for H = 256), the fp32
// recurrence kernels elsewhere.  lstm_plan (lstm.cu) picks the recurrence of each shape.  State, gate activations and
// accumulation are fp32 in every mode.
// x [T1*B, In] -> y [T1*B, H]; h0/c0/hN/cN [layers, B, H]; notdone [T1*B] (float, multiplies the state
// before each step).
int lstm_forward(const float* x, const float* notdone, const float* h0, const float* c0, const LstmParams& p,
                 int64_t T1, int64_t B, int In, int H, int layers, LstmWs& ws, float* y, float* hN, float* cN,
                 int precision, cudaStream_t stream);

// Gradients at the two ends of the recurrence, each [layers, B, H] and each optional (null: not given / not wanted).
// dhN / dcN arrive at the final state and enter every layer's backward recurrence at t = T1-1; dh0 / dc0 are the gradients
// with respect to the h0 / c0 the forward was given, so they include the notdone_0 mask (a column that starts an episode at
// t = 0 gets zeros).  All null: lstm_backward runs exactly the kernels, and computes exactly the values, it runs without them.
struct LstmStateGrads {
  const float* dhN = nullptr; const float* dcN = nullptr;
  float* dh0 = nullptr; float* dc0 = nullptr;
};

// dy [T1*B, H] -> dx [T1*B, In]; parameter gradients written (overwritten) into g.  splitk: GEMM scratch
// (kSplitKScratchFloats).
// Joins the side stream lstm_backward may have forked (weight-gradient GEMMs overlapping the caller's own backward):
// call on the same stream after the work that may overlap, before anything consumes the LSTM parameter gradients.
int lstm_backward_join(cudaStream_t stream);

int lstm_backward(const float* dy, const float* x, const float* notdone, const LstmParams& p, const LstmGrads& g,
                  int64_t T1, int64_t B, int In, int H, int layers, LstmWs& ws, float* dx, float* splitk,
                  float* colsum_scratch, int precision, cudaStream_t stream, const LstmStateGrads& sg = LstmStateGrads());

}  // namespace tb
