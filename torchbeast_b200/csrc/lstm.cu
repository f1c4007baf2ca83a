// Stacked LSTM over the unroll with per-step done-reset, forward + BPTT (sm_90a).
//
// Replaces the reference's 81 seq_len-1 nn.LSTM calls and their autograd graph
// (/root/reference/torchbeast/monobeast.py:603-611, polybeast_learner.py:241-249):
//     for t: state *= notdone_t;  out_t, state = LSTM(x_t, state)         (all layers per t)
// Re-ordered layer-major: layer l only depends on layer l-1's outputs, so for each layer the
// input projection of ALL T+1 steps is hoisted into one [N,In]x[In,4H] GEMM, the recurrence runs
// as T+1 fused step kernels (recurrent product + gate non-linearities + state update + next
// step's masked state, W_hh slice and h tile staged in shared memory), and BPTT accumulates
// the weight gradients with two [4H,N]x[N,*] GEMMs after the time loop instead of per step.
// torch.nn.LSTM conventions: gate order i,f,g,o; weight_ih [4H,In], weight_hh [4H,H]; two biases.
#include "lstm.cuh"

#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <stdlib.h>

#include "gemm_simt.cuh"
#include "gemm_tc.cuh"
#include "net_kernels.cuh"
#include "tc_common.cuh"

namespace tb {

static inline int padded_h(int H) {
  int hp = (H + 3) & ~3;
  if (((hp / 4) & 1) == 0) hp += 4;  // odd number of 16-byte groups per row: conflict-free LDS.128
  return hp;
}

static inline int64_t ld16(int64_t n) { return (n + 7) & ~int64_t(7); }
// row length (bf16 elements) of the tensor-core recurrence's operand tiles: K padded to 16, +8 so that a
// row is an odd number of 16-byte chunks (conflict-free ldmatrix)
static inline int mma_hq(int H) { return ((H + 15) & ~15) + 8; }

size_t lstm_ws_bytes(int64_t T1, int64_t B, int In, int H, int layers, int precision) {
  return lstm_ws(nullptr, T1, B, In, H, layers, precision).bytes;
}

LstmWs lstm_ws(void* base, int64_t T1, int64_t B, int In, int H, int layers, int precision) {
  LstmWs w;
  size_t off = 0;
  auto takef = [&](int64_t n) {
    float* p = base ? reinterpret_cast<float*>(static_cast<char*>(base) + off) : nullptr;
    off += (size_t(n) * sizeof(float) + 255) & ~size_t(255);
    return p;
  };
  const int64_t N = T1 * B;
  for (int l = 0; l < kLstmMaxLayers; ++l) {
    LstmLayerWs& L = w.layer[l];
    if (l < layers) {
      const int Hp = padded_h(H);
      L.gates = takef(N * 4 * H); L.hs = takef(N * H); L.cs = takef(N * H); L.hm = takef(N * Hp);
      L.cm = takef(N * H); L.dgates = takef(N * 4 * H); L.bsum = takef(4 * H); L.w_hh_t = takef(int64_t(H + 4) * 4 * Hp);
      L.wp = takef(int64_t(4 * H + 4) * Hp);
      L.xb = L.wihb = L.dgb = L.hmb = L.hmq = L.dgq = L.hq = nullptr;
      L.xb_lo = L.wihb_lo = L.dgb_lo = L.hmb_lo = L.hq_lo = L.hmq_lo = L.dgq_lo = 0;
      L.gact = L.csb = nullptr;
      if (precision) {  // bf16 operand copies (2 bytes per element: take half the float count, rounded up)
        const int64_t in_l = (l == 0) ? In : H;
        // precision 2 (split-bf16): every GEMM operand also has a lo plane right behind its hi plane
        auto takeh = [&](int64_t n, int64_t* lo) {
          const int64_t plane = ((n * 2 + 255) & ~int64_t(255)) / 2;  // elements, 256-byte multiple
          void* ptr = takef(((precision == 2 ? 2 * plane : plane) + 1) / 2);
          *lo = precision == 2 ? plane : 0;
          return ptr;
        };
        L.xb = takeh(N * ld16(in_l), &L.xb_lo); L.wihb = takeh(int64_t(4) * H * ld16(in_l), &L.wihb_lo);
        L.dgb = takeh(N * ld16(4 * H), &L.dgb_lo); L.hmb = takeh(N * ld16(H), &L.hmb_lo);
        L.hmq = takeh(N * mma_hq(H), &L.hmq_lo); L.hq = takeh((N + B) * mma_hq(H), &L.hq_lo);
        L.dgq = takeh(int64_t(2) * 4 * B * mma_hq(H), &L.dgq_lo);
        if (precision == 2) {
          const int64_t nC4 = (H + 3) / 4;
          L.gact = takef(T1 * nC4 * 512); L.csb = takef((T1 + 1) * nC4 * 128);
        }
      }
    } else {
      L = LstmLayerWs();
    }
  }
  w.dh = takef(B * H); w.dc = takef(B * H);
  w.dx_mid = takef(N * (H > In ? H : In));
  w.wg_scratch = (precision && layers == 2) ? takef(int64_t(4) * 4 * H * (((H > In ? H : In) + 31) & ~31)) : nullptr;
  w.dgp = takef(int64_t(2) * 4 * B * padded_h(H));
  w.sync = reinterpret_cast<unsigned*>(takef(64));
  w.dxb = (precision == 2 && layers == 2) ? takef(T1 * int64_t((H + 7) / 8) * 256) : nullptr;
  w.flags = reinterpret_cast<unsigned*>(takef(2 * 512 * 32));  // 2 x 512 flags, 128 bytes apart (kFlagStride)
  w.Hp = padded_h(H);
  w.bytes = off;
  return w;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__global__ void add2_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o, int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] + b[i];
}

// ---------------------------------------------------------------------------------------
// forward step: one CTA = 4 hidden units (x 4 gates = 16 rows of W_hh) x a 32-row batch tile.
// 512 threads: lane = batch row, warp = (gate q, k-quarter ks); each thread accumulates gate q of the
// 4 units over a quarter of the reduction, partial sums are combined through shared memory (16 warps
// per SM hide the LDS/FMA latency that a 4-warp CTA exposed: ncu 'No Eligible' 86%).
// Operands are staged by the bulk-copy engine (cp.async.bulk -> UBLKCP, mbarrier complete_tx):
// four 8 KB W_hh gate slices - issued BEFORE griddepcontrol.wait, so with programmatic
// dependent launch they stream in while the previous time step is still finishing - and the
// 67 KB masked-h tile the previous step produced.
// ---------------------------------------------------------------------------------------
constexpr int kStepUnits = 4;
constexpr int kStepThreads = 512;
constexpr int kStepKSplit = 4;

struct StepArgs {
  const float* hm;      // [B,Hp] masked recurrent input of this step (h_{t-1} * nd_t), zero padded
  const float* cm;      // [B,H]  masked previous cell state
  const float* nd_next; // [B] notdone_{t+1} or nullptr at the last step
  const float* wp;      // [4H+4,Hp] padded W_hh
  float* gates;         // [B,4H] in: x-projection + biases; out: activated gates
  float* hs; float* cs; // [B,H] this step's outputs
  float* hm_next; float* cm_next;  // [B,Hp] / [B,H] masked state for step t+1 (nullptr at the last step)
  int B, H, Hp;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE_%=;\n"
      "bra LAB_WAIT_%=;\n"
      "LAB_DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__global__ void __launch_bounds__(kStepThreads) lstm_step_fwd_kernel(StepArgs a) {
  extern __shared__ __align__(128) float smem[];
  float* Ws = smem;                                  // [16][Hp]
  float* Xs = smem + 16 * a.Hp;                      // [32][Hp]  masked h_prev tile
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 48 * a.Hp);  // [0]: W slices, [1]: h tile
  __shared__ float act_s[4][kStepUnits][33];
  __shared__ float part_s[kStepKSplit][4][kStepUnits][33];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5, q = wrp & 3, ks = wrp >> 2;
  const int H = a.H, Hp = a.Hp;
  const int j0 = blockIdx.x * kStepUnits;
  const int b0 = blockIdx.y * 32;
  const int rows = (a.B - b0 < 32) ? (a.B - b0) : 32;
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint32_t wbytes = uint32_t(kStepUnits) * Hp * sizeof(float);
    mbar_expect_tx(&bar[0], 4 * wbytes);
#pragma unroll
    for (int g = 0; g < 4; ++g)  // rows g*H + j0 .. +3 are contiguous in the padded matrix
      bulk_g2s(Ws + g * kStepUnits * Hp, a.wp + (int64_t(g) * H + j0) * Hp, wbytes, &bar[0]);
    // everything above is independent of the previous step; the h tile is not
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const uint32_t xbytes = uint32_t(rows) * Hp * sizeof(float);
    mbar_expect_tx(&bar[1], xbytes);
    bulk_g2s(Xs, a.hm + int64_t(b0) * Hp, xbytes, &bar[1]);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // Issue the epilogue's global loads now so their latency hides behind the operand staging and the
  // dot products (ncu: they were the top long-scoreboard stalls when loaded at the point of use).
  const int b = b0 + lane;
  float pre_in[kStepUnits] = {0.f, 0.f, 0.f, 0.f};
  float cm_in = 0.f, ndn_in = 0.f;
  if (ks == 0 && lane < rows) {
#pragma unroll
    for (int u = 0; u < kStepUnits; ++u)
      if (j0 + u < H) pre_in[u] = a.gates[int64_t(b) * 4 * H + int64_t(q) * H + j0 + u];
    if (j0 + q < H) {
      cm_in = a.cm[int64_t(b) * H + j0 + q];
      if (a.nd_next) ndn_in = a.nd_next[b];
    }
  }
  __syncthreads();  // barrier inits visible to the waiting threads
  mbar_wait(&bar[0], 0);
  mbar_wait(&bar[1], 0);
  float acc[kStepUnits] = {0.f, 0.f, 0.f, 0.f};
  const float4* x4 = reinterpret_cast<const float4*>(Xs + lane * Hp);
  const float4* w4 = reinterpret_cast<const float4*>(Ws + (q * 4) * Hp);
  const int k4n = Hp / 4;
  const int kper = (k4n + kStepKSplit - 1) / kStepKSplit;
  const int k4a = ks * kper, k4b = (k4a + kper < k4n) ? k4a + kper : k4n;
  if (lane < rows) {
#pragma unroll 4
    for (int k4 = k4a; k4 < k4b; ++k4) {
      const float4 x = x4[k4];
#pragma unroll
      for (int u = 0; u < kStepUnits; ++u) {
        const float4 w = w4[u * k4n + k4];
        acc[u] = fmaf(x.x, w.x, acc[u]); acc[u] = fmaf(x.y, w.y, acc[u]);
        acc[u] = fmaf(x.z, w.z, acc[u]); acc[u] = fmaf(x.w, w.w, acc[u]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < kStepUnits; ++u) part_s[ks][q][u][lane] = acc[u];
  __syncthreads();
  if (ks == 0) {
#pragma unroll
    for (int u = 0; u < kStepUnits; ++u) {
      float v = 0.0f;
      if (lane < rows && j0 + u < H) {
        const float dot = (part_s[0][q][u][lane] + part_s[1][q][u][lane]) + (part_s[2][q][u][lane] + part_s[3][q][u][lane]);
        const float pre = pre_in[u] + dot;
        v = (q == 2) ? tanhf(pre) : sigmoidf_(pre);
        a.gates[int64_t(b) * 4 * H + int64_t(q) * H + j0 + u] = v;
      }
      act_s[q][u][lane] = v;
    }
  }
  __syncthreads();
  // state update: thread = (batch row lane, unit u) on the first four warps
  const int u = q;
  if (ks == 0 && lane < rows && j0 + u < H) {
    const int64_t o = int64_t(b) * H + j0 + u;
    const float cmv = cm_in;
    const float ig = act_s[0][u][lane], fg = act_s[1][u][lane], gg = act_s[2][u][lane], og = act_s[3][u][lane];
    const float c = fg * cmv + ig * gg;
    const float h = og * tanhf(c);
    a.cs[o] = c;
    a.hs[o] = h;
    if (a.hm_next) {
      const float ndn = ndn_in;
      a.hm_next[int64_t(b) * Hp + j0 + u] = h * ndn;
      a.cm_next[o] = c * ndn;
    }
  }
}

// padded copies: wp[r, :H] = w_hh[r, :], zero elsewhere (incl. 4 extra rows)
__global__ void lstm_pack_whh_kernel(const float* __restrict__ w, float* __restrict__ wp, int H, int Hp) {
  const int64_t total = int64_t(4 * H + 4) * Hp;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t r = i / Hp;
    const int k = int(i % Hp);
    wp[i] = (r < 4 * H && k < H) ? w[r * H + k] : 0.0f;
  }
}

// hm[0] = h0 * nd_0 (zero padded), cm[0] = c0 * nd_0
__global__ void lstm_init_state_kernel(const float* __restrict__ h0, const float* __restrict__ c0,
                                       const float* __restrict__ nd, float* __restrict__ hm, float* __restrict__ cm,
                                       int B, int H, int Hp) {
  const int64_t total = int64_t(B) * Hp;
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = int(i / Hp), k = int(i % Hp);
  if (k < H) {
    hm[i] = h0[int64_t(b) * H + k] * nd[b];
    cm[int64_t(b) * H + k] = c0[int64_t(b) * H + k] * nd[b];
  } else {
    hm[i] = 0.0f;
  }
}

// ---------------------------------------------------------------------------------------
// backward step, pointwise part: dgates_t (pre-activation) and the cell-state carry.
//   dh = dy_t + dh_raw * nd_next   (dh_raw = dgates_{t+1} . W_hh, masked by notdone_{t+1})
// ---------------------------------------------------------------------------------------
struct BwdPointArgs {
  const float* dy; const float* dh_raw; const float* nd_next;  // dh_raw/nd_next null at the last step
  const float* nd;                                             // notdone_t
  const float* gates; const float* cs; const float* cm;        // forward saves at t
  float* dc;                                                   // [B,H] carry in/out (dL/dc_t in, dL/dc_{t-1} out)
  float* dgates;                                               // [B,4H]
  float* dgp; int Hp;                                          // [4,B,Hp] gate-major padded copy
  int B, H; int first;                                         // first != 0: carries are zero (t = T1-1)
};

__global__ void lstm_step_bwd_point_kernel(BwdPointArgs a) {
  const int64_t total = int64_t(a.B) * a.H;
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = int(i / a.H), j = int(i % a.H);
  const int64_t g0 = int64_t(b) * 4 * a.H + j;
  const float ig = a.gates[g0], fg = a.gates[g0 + a.H], gg = a.gates[g0 + 2 * a.H], og = a.gates[g0 + 3 * a.H];
  float dh = a.dy[i];
  float dc = 0.0f;
  if (!a.first) {
    dh += a.dh_raw[i] * a.nd_next[b];
    dc = a.dc[i];
  }
  const float tc = tanhf(a.cs[i]);
  const float d_o = dh * tc;
  dc += dh * og * (1.0f - tc * tc);
  const float d_i = dc * gg, d_f = dc * a.cm[i], d_g = dc * ig;
  const float p_i = d_i * ig * (1.0f - ig), p_f = d_f * fg * (1.0f - fg);
  const float p_g = d_g * (1.0f - gg * gg), p_o = d_o * og * (1.0f - og);
  a.dgates[g0] = p_i; a.dgates[g0 + a.H] = p_f; a.dgates[g0 + 2 * a.H] = p_g; a.dgates[g0 + 3 * a.H] = p_o;
  const int64_t gs = int64_t(a.B) * a.Hp, gp = int64_t(b) * a.Hp + j;
  a.dgp[gp] = p_i; a.dgp[gs + gp] = p_f; a.dgp[2 * gs + gp] = p_g; a.dgp[3 * gs + gp] = p_o;
  a.dc[i] = dc * fg * a.nd[b];
}


// ---------------------------------------------------------------------------------------
// backward step, recurrent product: dh_raw[b,k] = sum_g sum_j dgates_g[b,j] * W_hh[g*H+j][k].
// One CTA = 4 output columns k x a 32-row batch tile; lane = batch row, warp = column.  The
// 4 x 4*Hp slice of W_hh^T arrives by one bulk copy before griddepcontrol.wait; the four
// [32,Hp] gate-gradient tiles stream through a 2-deep shared-memory ring (bulk copies).
// ---------------------------------------------------------------------------------------
struct DhArgs {
  const float* dgp;   // [4,B,Hp]
  const float* wtp;   // [H+4, 4*Hp]
  float* dh_raw;      // [B,H]
  int B, H, Hp;
};

__global__ void __launch_bounds__(kStepThreads) lstm_step_bwd_dh_kernel(DhArgs a) {
  extern __shared__ __align__(128) float smem[];
  const int Hp = a.Hp, H = a.H;
  float* Ws = smem;                       // [4][4*Hp]
  float* Xs = smem + 16 * Hp;             // [2][32][Hp]
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 80 * Hp);  // [0]: W, [1],[2]: ring slots
  __shared__ float part_s[kStepKSplit][4][33];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5, q = wrp & 3, ks = wrp >> 2;
  const int k0 = blockIdx.x * 4;
  const int b0 = blockIdx.y * 32;
  const int rows = (a.B - b0 < 32) ? (a.B - b0) : 32;
  const uint32_t xbytes = uint32_t(rows) * Hp * sizeof(float);
  if (tid == 0) {
    mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); mbar_init(&bar[2], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint32_t wbytes = uint32_t(16) * Hp * sizeof(float);
    mbar_expect_tx(&bar[0], wbytes);
    bulk_g2s(Ws, a.wtp + int64_t(k0) * 4 * Hp, wbytes, &bar[0]);
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int g = 0; g < 2; ++g) {
      mbar_expect_tx(&bar[1 + g], xbytes);
      bulk_g2s(Xs + g * 32 * Hp, a.dgp + (int64_t(g) * a.B + b0) * Hp, xbytes, &bar[1 + g]);
    }
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  __syncthreads();
  mbar_wait(&bar[0], 0);
  float acc = 0.0f;
  const int k4n = Hp / 4;
  const int kper = (k4n + kStepKSplit - 1) / kStepKSplit;
  const int k4a = ks * kper, k4b = (k4a + kper < k4n) ? k4a + kper : k4n;
  for (int g = 0; g < 4; ++g) {
    const int slot = g & 1;
    mbar_wait(&bar[1 + slot], (g >> 1) & 1);
    if (lane < rows) {
      const float4* x4 = reinterpret_cast<const float4*>(Xs + (slot * 32 + lane) * Hp);
      const float4* w4 = reinterpret_cast<const float4*>(Ws + (q * 4 + g) * Hp);
#pragma unroll 4
      for (int k4 = k4a; k4 < k4b; ++k4) {
        const float4 x = x4[k4];
        const float4 w = w4[k4];
        acc = fmaf(x.x, w.x, acc); acc = fmaf(x.y, w.y, acc); acc = fmaf(x.z, w.z, acc); acc = fmaf(x.w, w.w, acc);
      }
    }
    __syncthreads();  // everyone is done with this ring slot
    if (tid == 0 && g + 2 < 4) {
      mbar_expect_tx(&bar[1 + slot], xbytes);
      bulk_g2s(Xs + slot * 32 * Hp, a.dgp + (int64_t(g + 2) * a.B + b0) * Hp, xbytes, &bar[1 + slot]);
    }
  }
  part_s[ks][q][lane] = acc;
  __syncthreads();
  if (ks == 0 && lane < rows && k0 + q < H)
    a.dh_raw[int64_t(b0 + lane) * H + k0 + q] = (part_s[0][q][lane] + part_s[1][q][lane]) + (part_s[2][q][lane] + part_s[3][q][lane]);
}

// wtp[k][g*Hp + j] = W_hh[g*H + j][k], zero padded (j >= H, k >= H)
__global__ void lstm_pack_whh_t_kernel(const float* __restrict__ w, float* __restrict__ wtp, int H, int Hp) {
  const int64_t total = int64_t(H + 4) * 4 * Hp;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t k = i / (4 * Hp);
    const int r = int(i % (4 * Hp));
    const int g = r / Hp, j = r % Hp;
    wtp[i] = (k < H && j < H) ? w[(int64_t(g) * H + j) * H + k] : 0.0f;
  }
}

static int launch_step_bwd_dh(const DhArgs& a, cudaStream_t st) {
  static bool attr_set = false;
  const size_t smem = size_t(80) * a.Hp * sizeof(float) + 32;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(lstm_step_bwd_dh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    TB_REQUIRE(e == cudaSuccess, "lstm: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  TB_REQUIRE(smem <= 220 * 1024, "lstm: hidden size %d too large for the backward step kernel", a.H);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((a.H + 3) / 4, (a.B + 31) / 32);
  cfg.blockDim = dim3(kStepThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, lstm_step_bwd_dh_kernel, a);
  TB_REQUIRE(e == cudaSuccess, "lstm_step_bwd_dh_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm_step_bwd_dh_kernel");
}

static int launch_step_fwd(const StepArgs& a, cudaStream_t st) {
  static bool attr_set = false;
  const size_t smem = size_t(48) * a.Hp * sizeof(float) + 16;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(lstm_step_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    TB_REQUIRE(e == cudaSuccess, "lstm: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  TB_REQUIRE(smem <= 200 * 1024, "lstm: hidden size %d too large for the step kernel", a.H);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((a.H + kStepUnits - 1) / kStepUnits, (a.B + 31) / 32);
  cfg.blockDim = dim3(kStepThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // PDL: overlap W staging with the previous step
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, lstm_step_fwd_kernel, a);
  TB_REQUIRE(e == cudaSuccess, "lstm_step_fwd_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm_step_fwd_kernel");
}


// =========================================================================================
// Persistent recurrence kernels: ONE cooperative launch runs all T+1 steps of a layer.
// The CTA's W_hh slice is staged once and stays in shared memory; the steps are separated by a
// grid-wide barrier (release add / acquire spin on a global counter) instead of kernel
// boundaries, and the only data that crosses CTAs per step (the masked h tile forward, the gate
// gradients backward) is pulled by bulk copies right after the barrier.
// =========================================================================================
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void grid_wait(const unsigned* ctr, unsigned target) {
  // Spin on cheap relaxed loads, then ONE acquire load: it reads a value written by the last red.release of the
  // arrivals (or a later one in the same release sequence), which is what synchronizes this thread with every
  // arriving CTA.  History: acquire loads in the spin cost an L1 invalidation per poll (30 % of the step at the
  // barrier); relaxed spin + fence.acq_rel.gpu fixed that but the fence is a full MEMBAR.ALL.GPU - ncu showed the
  // waiting thread spending as long in it as in the release fence of the arrive.
  while (ld_relaxed_u32(ctr) < target) {}
  (void)ld_acquire_u32(ctr);
  asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy writes of other CTAs -> our bulk copies
}

struct PersistFwdArgs {
  const float* wp; float* gates; float* hs; float* cs; float* hm; float* cm; const float* nd;
  unsigned* counter;
  int T1, B, H, Hp; unsigned nctas;
};

__global__ void __launch_bounds__(kStepThreads) lstm_fwd_persistent_kernel(PersistFwdArgs a) {
  // 16 warps; warp = k-slice (1/16 of the reduction), lane = batch row, every thread accumulates all
  // 16 outputs (4 gates x 4 units) of its row over its k-slice: one 4-wavefront LDS.128 of the h tile
  // feeds 64 FMAs (W comes by broadcast LDS.128), which roughly halves shared-memory traffic per FMA
  // against the per-step kernel (ncu: FFMA issue was short-scoreboard/LDS bound).
  extern __shared__ __align__(128) float smem[];
  float* Ws = smem;
  float* Xs = smem + 16 * a.Hp;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 48 * a.Hp);
  __shared__ float act_s[4][kStepUnits][33];
  __shared__ float part_s[16][16][33];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hp = a.Hp, B = a.B;
  const int j0 = blockIdx.x * kStepUnits;
  const int b0 = blockIdx.y * 32;
  const int rows = (B - b0 < 32) ? (B - b0) : 32;
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint32_t wbytes = uint32_t(kStepUnits) * Hp * sizeof(float);
    mbar_expect_tx(&bar[0], 4 * wbytes);
#pragma unroll
    for (int g = 0; g < 4; ++g)
      bulk_g2s(Ws + g * kStepUnits * Hp, a.wp + (int64_t(g) * H + j0) * Hp, wbytes, &bar[0]);
  }
  __syncthreads();
  mbar_wait(&bar[0], 0);
  const int b = b0 + lane;
  const int k4n = Hp / 4;
  const int kper = (k4n + 15) / 16;
  const int k4a = wrp * kper, k4b = (k4a + kper < k4n) ? k4a + kper : k4n;
  const float4* x4 = reinterpret_cast<const float4*>(Xs + lane * Hp);
  const float4* w4 = reinterpret_cast<const float4*>(Ws);
  float4* Xs4 = reinterpret_cast<float4*>(Xs);
  const int oq = wrp >> 2, ou = wrp & 3;  // the output (gate oq, unit ou) this thread finalises
  for (int t = 0; t < a.T1; ++t) {
    const int64_t row0 = int64_t(t) * B;
    const bool last = (t == a.T1 - 1);
    if (tid == 0 && t > 0) grid_wait(a.counter, unsigned(t) * a.nctas);  // every CTA finished step t-1
    __syncthreads();
    // cooperative L2 -> smem copy of the masked h tile (written by all CTAs in the previous step)
    const float4* src = reinterpret_cast<const float4*>(a.hm + (row0 + b0) * Hp);
    for (int i = tid; i < rows * k4n; i += kStepThreads) Xs4[i] = __ldcg(src + i);
    float pre_in = 0.f, cm_in = 0.f, ndn_in = 0.f;
    if (lane < rows && j0 + ou < H) {
      pre_in = a.gates[(row0 + b) * 4 * H + int64_t(oq) * H + j0 + ou];
      if (wrp < 4 && j0 + wrp < H) {
        cm_in = a.cm[(row0 + b) * H + j0 + wrp];
        if (!last) ndn_in = __ldg(a.nd + row0 + B + b);
      }
    }
    __syncthreads();
    float acc[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[o] = 0.f;
    if (lane < rows) {
      for (int k4 = k4a; k4 < k4b; ++k4) {
        const float4 x = x4[k4];
#pragma unroll
        for (int o = 0; o < 16; ++o) {
          const float4 w = w4[o * k4n + k4];
          acc[o] = fmaf(x.x, w.x, acc[o]); acc[o] = fmaf(x.y, w.y, acc[o]);
          acc[o] = fmaf(x.z, w.z, acc[o]); acc[o] = fmaf(x.w, w.w, acc[o]);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < 16; ++o) part_s[wrp][o][lane] = acc[o];
    __syncthreads();
    float gate_v = 0.0f;
    {
      if (lane < rows && j0 + ou < H) {
        float dot = 0.f;
#pragma unroll
        for (int sidx = 0; sidx < 16; ++sidx) dot += part_s[sidx][wrp][lane];
        const float pre = pre_in + dot;
        gate_v = (oq == 2) ? tanhf(pre) : sigmoidf_(pre);
      }
      act_s[oq][ou][lane] = gate_v;
    }
    __syncthreads();
    float c_new = 0.f, h_new = 0.f;
    const bool upd = (wrp < 4 && lane < rows && j0 + wrp < H);
    if (upd) {
      const int u = wrp;
      const float ig = act_s[0][u][lane], fg = act_s[1][u][lane], gg = act_s[2][u][lane], og = act_s[3][u][lane];
      c_new = fg * cm_in + ig * gg;
      h_new = og * tanhf(c_new);
      // the only value other CTAs wait for: next step's masked recurrent input
      if (!last) a.hm[(row0 + B + b) * Hp + j0 + u] = h_new * ndn_in;
    }
    __syncthreads();
    if (tid == 0 && !last) red_release_add(a.counter, 1u);
    // everything below is consumed by this CTA (cm) or after the kernel (gates, cs, hs): off the critical path
    if (lane < rows && j0 + ou < H) a.gates[(row0 + b) * 4 * H + int64_t(oq) * H + j0 + ou] = gate_v;
    if (upd) {
      const int64_t o = (row0 + b) * H + j0 + wrp;
      a.cs[o] = c_new;
      a.hs[o] = h_new;
      if (!last) a.cm[o + int64_t(B) * H] = c_new * ndn_in;
    }
  }
}

struct PersistBwdArgs {
  const float* wtp; const float* dy; const float* nd;
  const float* gates; const float* cs; const float* cm;
  float* dgates; float* dgp;
  unsigned* counter;
  int T1, B, H, Hp; unsigned nctas;
};

__global__ void __launch_bounds__(kStepThreads) lstm_bwd_persistent_kernel(PersistBwdArgs a) {
  extern __shared__ __align__(128) float smem[];
  const int Hp = a.Hp, H = a.H, B = a.B;
  float* Ws = smem;               // [4][4*Hp]
  float* Xs = smem + 16 * Hp;     // [2][32][Hp]
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 80 * Hp);
  __shared__ float part16_s[16][4][33];
  __shared__ float dh_s[4][33];   // dL/dh_{t} contribution from step t+1 for this CTA's 4 units (unmasked)
  __shared__ float dc_s[4][33];   // dL/dc_t carry
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5, q = wrp & 3, ks = wrp >> 2;
  const int k0 = blockIdx.x * 4;
  const int rows = B < 32 ? B : 32;  // single batch tile (host guarantees B <= 32)
  const uint32_t xbytes = uint32_t(rows) * Hp * sizeof(float);
  if (tid == 0) {
    mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); mbar_init(&bar[2], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint32_t wbytes = uint32_t(16) * Hp * sizeof(float);
    mbar_expect_tx(&bar[0], wbytes);
    bulk_g2s(Ws, a.wtp + int64_t(k0) * 4 * Hp, wbytes, &bar[0]);
  }
  if (tid < 128) { dh_s[q][lane] = 0.0f; dc_s[q][lane] = 0.0f; }
  __syncthreads();
  mbar_wait(&bar[0], 0);
  const int k4n = Hp / 4;
  const int64_t gs = int64_t(B) * Hp;
  int it = 0;
  for (int t = a.T1 - 1; t >= 0; --t, ++it) {
    const int64_t row0 = int64_t(t) * B;
    float* dgp_t = a.dgp + int64_t(it & 1) * 4 * gs;
    // ---- phase A: gate gradients of this CTA's 4 units (thread = batch row x unit) ----
    const bool actA = (ks == 0 && lane < rows && k0 + q < H);
    float p_i = 0.f, p_f = 0.f, p_g = 0.f, p_o = 0.f;
    int64_t g0 = 0;
    if (actA) {
      const int j = k0 + q;
      const int64_t i = (row0 + lane) * H + j;
      g0 = (row0 + lane) * 4 * H + j;
      const float ig = a.gates[g0], fg = a.gates[g0 + H], gg = a.gates[g0 + 2 * H], og = a.gates[g0 + 3 * H];
      float dh = a.dy[i];
      float dc = 0.0f;
      if (it > 0) {
        dh += dh_s[q][lane] * a.nd[row0 + B + lane];
        dc = dc_s[q][lane];
      }
      const float tc = tanhf(a.cs[i]);
      const float d_o = dh * tc;
      dc += dh * og * (1.0f - tc * tc);
      const float d_i = dc * gg, d_f = dc * a.cm[i], d_g = dc * ig;
      p_i = d_i * ig * (1.0f - ig); p_f = d_f * fg * (1.0f - fg);
      p_g = d_g * (1.0f - gg * gg); p_o = d_o * og * (1.0f - og);
      // what the other CTAs wait for: the gate-major padded copy feeding everybody's recurrent product
      const int64_t gp = int64_t(lane) * Hp + j;
      dgp_t[gp] = p_i; dgp_t[gs + gp] = p_f; dgp_t[2 * gs + gp] = p_g; dgp_t[3 * gs + gp] = p_o;
      dc_s[q][lane] = dc * fg * a.nd[row0 + lane];
    }
    if (t == 0) {  // uniform: no earlier step needs dh
      if (actA) { a.dgates[g0] = p_i; a.dgates[g0 + H] = p_f; a.dgates[g0 + 2 * H] = p_g; a.dgates[g0 + 3 * H] = p_o; }
      break;
    }
    __syncthreads();
    // ---- grid barrier: every CTA's gate gradients of step t are visible ----
    if (tid == 0) {
      red_release_add(a.counter, 1u);
      grid_wait(a.counter, unsigned(it + 1) * a.nctas);
      for (int g = 0; g < 2; ++g) {
        mbar_expect_tx(&bar[1 + g], xbytes);
        bulk_g2s(Xs + g * 32 * Hp, dgp_t + int64_t(g) * gs, xbytes, &bar[1 + g]);
      }
    }
    // row-major copy for the weight-gradient GEMMs after the loop: off the critical path
    if (actA) { a.dgates[g0] = p_i; a.dgates[g0 + H] = p_f; a.dgates[g0 + 2 * H] = p_g; a.dgates[g0 + 3 * H] = p_o; }
    // ---- phase B: dh_raw[b, k0+c] = sum_g dgates_g[b,:] . W_hh[g*H + :, k0+c], c = 0..3 ----
    // warp = k-slice (1/16), every thread accumulates all 4 columns of its batch row
    float acc4[4] = {0.f, 0.f, 0.f, 0.f};
    const int kper16 = (k4n + 15) / 16;
    const int ka = wrp * kper16, kb = (ka + kper16 < k4n) ? ka + kper16 : k4n;
    for (int g = 0; g < 4; ++g) {
      const int slot = g & 1;
      mbar_wait(&bar[1 + slot], (g >> 1) & 1);
      if (lane < rows) {
        const float4* x4 = reinterpret_cast<const float4*>(Xs + (slot * 32 + lane) * Hp);
        const float4* w4 = reinterpret_cast<const float4*>(Ws + g * Hp);
        for (int k4 = ka; k4 < kb; ++k4) {
          const float4 x = x4[k4];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 w = w4[c * 4 * k4n + k4];
            acc4[c] = fmaf(x.x, w.x, acc4[c]); acc4[c] = fmaf(x.y, w.y, acc4[c]);
            acc4[c] = fmaf(x.z, w.z, acc4[c]); acc4[c] = fmaf(x.w, w.w, acc4[c]);
          }
        }
      }
      __syncthreads();
      if (tid == 0 && g + 2 < 4) {
        mbar_expect_tx(&bar[1 + slot], xbytes);
        bulk_g2s(Xs + slot * 32 * Hp, dgp_t + int64_t(g + 2) * gs, xbytes, &bar[1 + slot]);
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) part16_s[wrp][c][lane] = acc4[c];
    __syncthreads();
    if (wrp < 4) {
      float d = 0.f;
#pragma unroll
      for (int sidx = 0; sidx < 16; ++sidx) d += part16_s[sidx][wrp][lane];
      dh_s[wrp][lane] = d;
    }
    __syncthreads();
  }
}

// 1 if the whole grid of `kernel` (blocks of `threads`, `smem` bytes of dynamic shared memory) is co-resident on the
// current device, as a cooperative launch needs; 0 otherwise
static int persistent_ok(const void* kernel, dim3 grid, int threads, size_t smem) {
  int dev = 0, sms = 0, coop = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  if (!coop) return 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return int64_t(per_sm) * sms >= int64_t(grid.x) * grid.y;
}

// cudaFuncSetAttribute is per device: the attribute caches are indexed by the current device
static inline size_t* per_device(size_t (&cache)[64]) {
  int dev = 0;
  cudaGetDevice(&dev);
  return &cache[dev & 63];
}

// raises the kernel's dynamic shared-memory limit to `smem` (once per device; *attr_smem caches the limit already set),
// then checks co-residency.  0: the kernel cannot run as one cooperative grid here
template <typename Kernel>
static int coop_fit(Kernel kernel, dim3 grid, size_t smem, int threads, size_t* attr_smem) {
  if (*attr_smem < smem) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) {
      cudaGetLastError();
      return 0;
    }
    *attr_smem = smem;
  }
  return persistent_ok((const void*)kernel, grid, threads, smem);
}

static size_t g_fwd_persist_attr_dev[64] = {0}, g_bwd_persist_attr_dev[64] = {0};

static int lstm_fwd_persistent(const LstmLayerWs& L, float* hs, const float* notdone, int64_t T1, int64_t B, int H,
                               unsigned* counter, cudaStream_t st) {
  if (B > 64) return -1;
  const int Hp = padded_h(H);
  const size_t smem = size_t(48) * Hp * sizeof(float) + 16;
  if (smem > 200 * 1024) return -1;
  dim3 grid((H + kStepUnits - 1) / kStepUnits, (unsigned)((B + 31) / 32));
  if (!coop_fit(lstm_fwd_persistent_kernel, grid, smem, kStepThreads, per_device(g_fwd_persist_attr_dev))) return -1;
  cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned), st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  PersistFwdArgs a;
  a.wp = L.wp; a.gates = L.gates; a.hs = hs; a.cs = L.cs; a.hm = L.hm; a.cm = L.cm; a.nd = notdone; a.counter = counter;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hp = Hp; a.nctas = grid.x * grid.y;
  void* args[] = {&a};
  e = cudaLaunchCooperativeKernel((const void*)lstm_fwd_persistent_kernel, grid, dim3(kStepThreads), args, smem, st);
  TB_REQUIRE(e == cudaSuccess, "lstm_fwd_persistent_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm_fwd_persistent_kernel");
}

static int lstm_bwd_persistent(const LstmLayerWs& L, const LstmWs& ws, const float* dy, const float* notdone, int64_t T1,
                               int64_t B, int H, unsigned* counter, cudaStream_t st) {
  if (B > 32) return -1;
  const int Hp = padded_h(H);
  const size_t smem = size_t(80) * Hp * sizeof(float) + 32;
  if (smem > 220 * 1024) return -1;
  dim3 grid((H + 3) / 4, 1);
  if (!coop_fit(lstm_bwd_persistent_kernel, grid, smem, kStepThreads, per_device(g_bwd_persist_attr_dev))) return -1;
  cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(ws.dgp, 0, sizeof(float) * 2 * 4 * B * Hp, st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  PersistBwdArgs a;
  a.wtp = L.w_hh_t; a.dy = dy; a.nd = notdone; a.gates = L.gates; a.cs = L.cs; a.cm = L.cm; a.dgates = L.dgates;
  a.dgp = ws.dgp; a.counter = counter; a.T1 = int(T1); a.B = int(B); a.H = H; a.Hp = Hp; a.nctas = grid.x;
  void* args[] = {&a};
  e = cudaLaunchCooperativeKernel((const void*)lstm_bwd_persistent_kernel, grid, dim3(kStepThreads), args, smem, st);
  TB_REQUIRE(e == cudaSuccess, "lstm_bwd_persistent_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm_bwd_persistent_kernel");
}


// =========================================================================================
// Tensor-core variants of the persistent recurrence (bf16 backend): the per-step recurrent products run
// on mma.sync.m16n8k16 (bf16 x bf16 -> fp32).  wgmma needs M >= 64 and smem-resident B, so for this
// M = 32, N = 16/4, weights-in-registers product the warp-level MMA is the right tool: the CTA's W_hh
// slice lives in REGISTERS as B fragments for all T+1 steps (nothing but the 34 KB bf16 h tile moves
// per step), A fragments come from shared memory via ldmatrix.
// =========================================================================================
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_ptr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(smem_ptr)));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

struct PersistFwdMmaArgs {
  const float* w_hh;            // [4H, H] fp32 (converted to bf16 fragments once)
  float* gates; float* hs; float* cs; float* cm; const float* nd;
  __nv_bfloat16* hmq;           // [T1*B, Hq] masked recurrent inputs (hmq[0] pre-initialised)
  unsigned* counter;
  int T1, B, H, Hq; unsigned nctas;
};

constexpr int kMmaWarps = 8;     // warps that own k-slices of the product
constexpr int kMaxKSteps = 6;    // ceil(ceil(H/16) / kMmaWarps) upper bound (H <= 768)

__global__ void __launch_bounds__(kStepThreads) lstm_fwd_persistent_mma_kernel(PersistFwdMmaArgs a) {
  extern __shared__ __align__(128) unsigned char smem_b[];
  __nv_bfloat16* Xs = reinterpret_cast<__nv_bfloat16*>(smem_b);  // [32][Hq]
  __shared__ float act_s[4][kStepUnits][33];
  __shared__ float part_s[kMmaWarps][16][33];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hq = a.Hq, B = a.B;
  const int j0 = blockIdx.x * kStepUnits;
  const int b0 = blockIdx.y * 32;
  const int rows = (B - b0 < 32) ? (B - b0) : 32;
  const int ksteps = (H + 15) / 16;
  const int kper = (ksteps + kMmaWarps - 1) / kMmaWarps;
  const int ks0 = wrp * kper, ks1 = (ks0 + kper < ksteps) ? ks0 + kper : ksteps;
  // B fragments of this CTA's 16 gate rows (o = gate*4 + unit), k-slice of this warp: registers for all steps
  uint32_t bf[kMaxKSteps][2][2];
  if (wrp < kMmaWarps) {
#pragma unroll
    for (int s = 0; s < kMaxKSteps; ++s) {
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        const int o = nt * 8 + (lane >> 2);
        const int g = o >> 2, u = o & 3;
        const bool okrow = (j0 + u < H);
        const float* wr = a.w_hh + (int64_t(g) * H + j0 + u) * H;
        const int k = (ks0 + s) * 16 + (lane & 3) * 2;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (okrow && ks0 + s < ks1) {
          if (k < H) v[0] = wr[k];
          if (k + 1 < H) v[1] = wr[k + 1];
          if (k + 8 < H) v[2] = wr[k + 8];
          if (k + 9 < H) v[3] = wr[k + 9];
        }
        bf[s][nt][0] = pack_bf16(v[0], v[1]);
        bf[s][nt][1] = pack_bf16(v[2], v[3]);
      }
    }
  }
  const int b = b0 + lane;
  const int oq = wrp >> 2, ou = wrp & 3;
  const int chunks_per_row = Hq / 8;               // 16-byte chunks
  uint4* Xs4 = reinterpret_cast<uint4*>(Xs);
  for (int t = 0; t < a.T1; ++t) {
    const int64_t row0 = int64_t(t) * B;
    const bool last = (t == a.T1 - 1);
    if (tid == 0 && t > 0) grid_wait(a.counter, unsigned(t) * a.nctas);
    __syncthreads();
    const uint4* src = reinterpret_cast<const uint4*>(a.hmq + (row0 + b0) * Hq);
    {
      const int nchunk = rows * chunks_per_row;  // <= 5 chunks per thread: all loads in flight, then the stores
      uint4 v[5];
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        const int i = tid + u * kStepThreads;
        if (i < nchunk) v[u] = __ldcg(src + i);
      }
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        const int i = tid + u * kStepThreads;
        if (i < nchunk) Xs4[i] = v[u];
      }
    }
    float pre_in = 0.f, cm_in = 0.f, ndn_in = 0.f;
    if (lane < rows && j0 + ou < H) {
      pre_in = a.gates[(row0 + b) * 4 * H + int64_t(oq) * H + j0 + ou];
      if (wrp < 4 && j0 + wrp < H) {
        cm_in = a.cm[(row0 + b) * H + j0 + wrp];
        if (!last) ndn_in = __ldg(a.nd + row0 + B + b);
      }
    }
    __syncthreads();
    if (wrp < kMmaWarps) {
      float acc[2][2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
#pragma unroll
      for (int s = 0; s < kMaxKSteps; ++s) {
        if (ks0 + s < ks1) {
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            uint32_t af[4];
            ldmatrix_x4(af, Xs + (mt * 16 + (lane & 15)) * Hq + (ks0 + s) * 16 + (lane >> 4) * 8);
            mma_bf16_16816(acc[mt][0], af, bf[s][0][0], bf[s][0][1]);
            mma_bf16_16816(acc[mt][1], af, bf[s][1][0], bf[s][1][1]);
          }
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int r = mt * 16 + (lane >> 2), c = nt * 8 + (lane & 3) * 2;
          part_s[wrp][c][r] = acc[mt][nt][0]; part_s[wrp][c + 1][r] = acc[mt][nt][1];
          part_s[wrp][c][r + 8] = acc[mt][nt][2]; part_s[wrp][c + 1][r + 8] = acc[mt][nt][3];
        }
    }
    __syncthreads();
    float gate_v = 0.0f;
    if (lane < rows && j0 + ou < H) {
      float dot = 0.f;
#pragma unroll
      for (int sidx = 0; sidx < kMmaWarps; ++sidx) dot += part_s[sidx][wrp][lane];
      const float pre = pre_in + dot;
      gate_v = (oq == 2) ? tanhf(pre) : sigmoidf_(pre);
    }
    act_s[oq][ou][lane] = gate_v;
    __syncthreads();
    float c_new = 0.f, h_new = 0.f;
    const bool upd = (wrp < 4 && lane < rows && j0 + wrp < H);
    if (upd) {
      const int u = wrp;
      const float ig = act_s[0][u][lane], fg = act_s[1][u][lane], gg = act_s[2][u][lane], og = act_s[3][u][lane];
      c_new = fg * cm_in + ig * gg;
      h_new = og * tanhf(c_new);
      if (!last) a.hmq[(row0 + B + b) * Hq + j0 + u] = __float2bfloat16_rn(h_new * ndn_in);
    }
    __syncthreads();
    if (tid == 0 && !last) red_release_add(a.counter, 1u);
    if (lane < rows && j0 + ou < H) a.gates[(row0 + b) * 4 * H + int64_t(oq) * H + j0 + ou] = gate_v;
    if (upd) {
      const int64_t o = (row0 + b) * H + j0 + wrp;
      a.cs[o] = c_new;
      a.hs[o] = h_new;
      if (!last) a.cm[o + int64_t(B) * H] = c_new * ndn_in;
    }
  }
}

// ---- two stacked layers as ONE wavefront ------------------------------------------------------
// Layer 1 at time t needs only layer 0's h at time t, so wave step s runs layer 0 at t = s and layer 1
// at t = s-1 side by side: T1+1 grid barriers instead of 2*T1, the input projection of layer 1 rides
// on the same tensor-core pass (its operand tile h0_{s-1} is the one layer 0's recurrence loads anyway),
// and the hoisted layer-1 projection GEMM disappears.  Each CTA owns kStepUnits hidden units of BOTH
// layers.  The done-mask is applied to the recurrent PRODUCT (a 0/1 row scale commutes with the GEMM),
// so only the raw bf16 h tiles are exchanged; the masked copies (hmq) are still written for the
// weight-gradient GEMMs.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}

struct WaveFwdArgs {
  const float* w_hh0; const float* w_ih1; const float* w_hh1; const float* bias1;
  float* gates[2]; float* hs[2]; float* cs[2]; float* cm[2];
  __nv_bfloat16* hq[2];    // raw h: [(T1+1)*B, Hq]; slot 0 = initial state, slot t+1 = h_t
  __nv_bfloat16* hmq[2];   // masked recurrent inputs [T1*B, Hq] (slot 0 pre-initialised)
  const float* nd; unsigned* counter;
  int T1, B, H, Hq; unsigned nctas;
};

constexpr int kWaveK = 3;  // k-steps per warp, all 16 warps own a k-slice: ceil(ceil(H/16)/16) (H <= 768)

__global__ void __launch_bounds__(kStepThreads) lstm2_fwd_wave_mma_kernel(WaveFwdArgs a) {
  extern __shared__ __align__(128) unsigned char smem_b[];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hq = a.Hq, B = a.B;
  __nv_bfloat16* X0 = reinterpret_cast<__nv_bfloat16*>(smem_b);  // [32][Hq]  h0_{s-1}
  __nv_bfloat16* X1 = X0 + 32 * Hq;                              // [32][Hq]  h1_{s-2}
  typedef float PartT[2][16][33];
  PartT* part = reinterpret_cast<PartT*>(smem_b + size_t(2) * 32 * Hq * 2);  // [16 warps][set][col][row]
  __shared__ float act_s[2][4][kStepUnits][33];
  __shared__ float nd_s[2][32];
  const int j0 = blockIdx.x * kStepUnits;
  const int rows = (B < 32) ? B : 32;
  const int ksteps = (H + 15) / 16;
  const int kper = (ksteps + 15) / 16;
  const int ks0 = wrp * kper, ks1 = (ks0 + kper < ksteps) ? ks0 + kper : ksteps;
  // B fragments of this CTA's 16 gate rows (o = gate*4 + unit) of the three weight matrices
  uint32_t bf[3][kWaveK][2][2];
  {
    const float* wm[3] = {a.w_hh0, a.w_ih1, a.w_hh1};
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int s = 0; s < kWaveK; ++s)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int o = nt * 8 + (lane >> 2);
          const int g = o >> 2, u = o & 3;
          const float* wr = wm[m] + (int64_t(g) * H + j0 + u) * H;
          const int k = (ks0 + s) * 16 + (lane & 3) * 2;
          float v[4] = {0.f, 0.f, 0.f, 0.f};
          if (j0 + u < H && ks0 + s < ks1) {
            if (k < H) v[0] = wr[k];
            if (k + 1 < H) v[1] = wr[k + 1];
            if (k + 8 < H) v[2] = wr[k + 8];
            if (k + 9 < H) v[3] = wr[k + 9];
          }
          bf[m][s][nt][0] = pack_bf16(v[0], v[1]);
          bf[m][s][nt][1] = pack_bf16(v[2], v[3]);
        }
  }
  const int b = lane;
  const int oq = wrp >> 2, ou = wrp & 3;           // activation role: gate column o = wrp of both layers
  const bool colok = (lane < rows && j0 + ou < H);
  const float bias1 = colok ? a.bias1[int64_t(oq) * H + j0 + ou] : 0.f;
  const int ul = (wrp >> 2) & 1, uu = wrp & 3;     // update role: warps 0..3 layer 0, warps 4..7 layer 1
  const bool updrole = (wrp < 8 && lane < rows && j0 + uu < H);
  // per-role pointers picked once (dynamic indexing of the parameter arrays would go through local memory)
  float* const cm_u = ul ? a.cm[1] : a.cm[0];
  float* const cs_u = ul ? a.cs[1] : a.cs[0];
  float* const hs_u = ul ? a.hs[1] : a.hs[0];
  __nv_bfloat16* const hq_u = ul ? a.hq[1] : a.hq[0];
  __nv_bfloat16* const hmq_u = ul ? a.hmq[1] : a.hmq[0];
  const int chunks_per_row = Hq / 8;               // 16-byte chunks
  const int nchunk = rows * chunks_per_row;
  uint4* X04 = reinterpret_cast<uint4*>(X0);
  uint4* X14 = reinterpret_cast<uint4*>(X1);
  for (int s = 0; s <= a.T1; ++s) {
    const bool act0 = (s < a.T1), act1 = (s >= 1);
    if (tid == 0 && s > 0) grid_wait(a.counter, unsigned(s) * a.nctas);
    __syncthreads();
    {
      const uint4* src0 = reinterpret_cast<const uint4*>(a.hq[0] + int64_t(s) * B * Hq);
      const uint4* src1 = reinterpret_cast<const uint4*>(a.hq[1] + int64_t(s > 0 ? s - 1 : 0) * B * Hq);
      // per-thread async copies (LDGSTS, L1 bypass): ten 16-byte chunks in flight without staging registers
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        const int i = tid + u * kStepThreads;
        if (i < nchunk) {
          cp_async16(X04 + i, src0 + i);
          if (act1) cp_async16(X14 + i, src1 + i);
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (tid < 64) {
      const int l = tid >> 5, r = tid & 31, t = s - l;
      nd_s[l][r] = (r < rows && t >= 0 && t < a.T1) ? __ldg(a.nd + int64_t(t) * B + r) : 0.f;
    }
    float pre0 = 0.f, cm_in = 0.f, ndn_in = 0.f;
    if (colok && act0) pre0 = a.gates[0][(int64_t(s) * B + b) * 4 * H + int64_t(oq) * H + j0 + ou];
    const int tu = s - ul;                          // time step of this thread's update role
    const bool upd = updrole && (ul ? act1 : act0);
    if (upd) {
      cm_in = cm_u[(int64_t(tu) * B + b) * H + j0 + uu];
      if (tu < a.T1 - 1) ndn_in = __ldg(a.nd + int64_t(tu + 1) * B + b);
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    {
      float acc0[2][2][4], accI[2][2][4], acc1[2][2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) { acc0[mt][nt][e] = 0.f; accI[mt][nt][e] = 0.f; acc1[mt][nt][e] = 0.f; }
#pragma unroll
      for (int sk = 0; sk < kWaveK; ++sk) {
        if (ks0 + sk < ks1) {
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            uint32_t af[4];
            const int off = (mt * 16 + (lane & 15)) * Hq + (ks0 + sk) * 16 + (lane >> 4) * 8;
            ldmatrix_x4(af, X0 + off);
            if (act0) {
              mma_bf16_16816(acc0[mt][0], af, bf[0][sk][0][0], bf[0][sk][0][1]);
              mma_bf16_16816(acc0[mt][1], af, bf[0][sk][1][0], bf[0][sk][1][1]);
            }
            if (act1) {
              mma_bf16_16816(accI[mt][0], af, bf[1][sk][0][0], bf[1][sk][0][1]);
              mma_bf16_16816(accI[mt][1], af, bf[1][sk][1][0], bf[1][sk][1][1]);
              ldmatrix_x4(af, X1 + off);
              mma_bf16_16816(acc1[mt][0], af, bf[2][sk][0][0], bf[2][sk][0][1]);
              mma_bf16_16816(acc1[mt][1], af, bf[2][sk][1][0], bf[2][sk][1][1]);
            }
          }
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r = mt * 16 + (lane >> 2);
        const float m0a = nd_s[0][r], m0b = nd_s[0][r + 8], m1a = nd_s[1][r], m1b = nd_s[1][r + 8];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int c = nt * 8 + (lane & 3) * 2;
          part[wrp][0][c][r] = acc0[mt][nt][0] * m0a; part[wrp][0][c + 1][r] = acc0[mt][nt][1] * m0a;
          part[wrp][0][c][r + 8] = acc0[mt][nt][2] * m0b; part[wrp][0][c + 1][r + 8] = acc0[mt][nt][3] * m0b;
          part[wrp][1][c][r] = accI[mt][nt][0] + acc1[mt][nt][0] * m1a;
          part[wrp][1][c + 1][r] = accI[mt][nt][1] + acc1[mt][nt][1] * m1a;
          part[wrp][1][c][r + 8] = accI[mt][nt][2] + acc1[mt][nt][2] * m1b;
          part[wrp][1][c + 1][r + 8] = accI[mt][nt][3] + acc1[mt][nt][3] * m1b;
        }
      }
    }
    __syncthreads();
    float gate0 = 0.f, gate1 = 0.f;
    if (colok) {
      float d0 = 0.f, d1 = 0.f;
#pragma unroll
      for (int w = 0; w < 16; ++w) { d0 += part[w][0][wrp][lane]; d1 += part[w][1][wrp][lane]; }
      if (act0) { const float pre = pre0 + d0; gate0 = (oq == 2) ? tanhf(pre) : sigmoidf_(pre); }
      if (act1) { const float pre = bias1 + d1; gate1 = (oq == 2) ? tanhf(pre) : sigmoidf_(pre); }
    }
    act_s[0][oq][ou][lane] = gate0;
    act_s[1][oq][ou][lane] = gate1;
    __syncthreads();
    float c_new = 0.f, h_new = 0.f;
    if (upd) {
      const float ig = act_s[ul][0][uu][lane], fg = act_s[ul][1][uu][lane], gg = act_s[ul][2][uu][lane],
                  og = act_s[ul][3][uu][lane];
      c_new = fg * cm_in + ig * gg;
      h_new = og * tanhf(c_new);
      hq_u[(int64_t(tu + 1) * B + b) * Hq + j0 + uu] = __float2bfloat16_rn(h_new);
    }
    __syncthreads();
    if (tid == 0 && s < a.T1) red_release_add(a.counter, 1u);
    if (colok) {
      if (act0) a.gates[0][(int64_t(s) * B + b) * 4 * H + int64_t(oq) * H + j0 + ou] = gate0;
      if (act1) a.gates[1][(int64_t(s - 1) * B + b) * 4 * H + int64_t(oq) * H + j0 + ou] = gate1;
    }
    if (upd) {
      const int64_t o = (int64_t(tu) * B + b) * H + j0 + uu;
      cs_u[o] = c_new;
      hs_u[o] = h_new;
      if (tu < a.T1 - 1) {
        cm_u[o + int64_t(B) * H] = c_new * ndn_in;
        hmq_u[(int64_t(tu + 1) * B + b) * Hq + j0 + uu] = __float2bfloat16_rn(h_new * ndn_in);
      }
    }
  }
}

struct PersistBwdMmaArgs {
  const float* w_hh; const float* dy; const float* nd;
  const float* gates; const float* cs; const float* cm;
  __nv_bfloat16* dgb; int lg;          // gate gradients of all steps, bf16 [T1*B, lg] (operand of the hoisted GEMMs)
  float* db;                           // [4H] bias gradient = sum over steps and rows of the gate gradients
  __nv_bfloat16* dgq;                  // dgq: [2][4, B, Hq]
  unsigned* counter;
  int T1, B, H, Hq; unsigned nctas;
};

constexpr int kMaxKStepsBwd = 12;  // ceil(4*ceil(H/16) / 16) upper bound (H <= 768)
constexpr int kBwdCols = 8;        // output columns (hidden units) per CTA: one full n8 MMA tile
constexpr int kBwdNT = kBwdCols / 8;

// Every CTA needs ALL gate gradients of the step (4 x [32, H] bf16 = 137 KB, pulled L2 -> smem with all loads
// of a thread in flight at once); 8 columns per CTA (65 CTAs) fill the n8 MMA tile and halve the per-step L2
// traffic against 4 columns (16 columns leave too few SMs pulling).
__global__ void __launch_bounds__(kStepThreads) lstm_bwd_persistent_mma_kernel(PersistBwdMmaArgs a) {
  extern __shared__ __align__(128) unsigned char smem_b[];
  __nv_bfloat16* Xs = reinterpret_cast<__nv_bfloat16*>(smem_b);  // [4 gates][32][Hq]
  __shared__ float part16_s[16][kBwdCols][33];
  __shared__ float dh_s[kBwdCols][33];
  __shared__ float dc_s[kBwdCols][33];
  __shared__ __align__(16) __nv_bfloat16 stg_s[4][32][kBwdCols];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hq = a.Hq, B = a.B;
  const int k0 = blockIdx.x * kBwdCols;
  const int rows = B < 32 ? B : 32;
  const int kpg = (H + 15) / 16;           // k16 steps per gate
  const int ksteps = 4 * kpg;
  const int kper = (ksteps + 15) / 16;
  const int ks0 = wrp * kper, ks1 = (ks0 + kper < ksteps) ? ks0 + kper : ksteps;
  // B fragments: B[kk][n] = W_hh[g*H + j][k0 + n], kk = g*kpg*16 + j
  uint32_t bf[kMaxKStepsBwd][kBwdNT][2];
#pragma unroll
  for (int s = 0; s < kMaxKStepsBwd; ++s) {
    const int st = ks0 + s;
    const int g = st / kpg, j = (st % kpg) * 16 + (lane & 3) * 2;
#pragma unroll
    for (int nt = 0; nt < kBwdNT; ++nt) {
      const int n = nt * 8 + (lane >> 2);
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (st < ks1 && k0 + n < H) {
        const float* wc = a.w_hh + int64_t(g) * H * H + (k0 + n);
        if (j < H) v[0] = wc[int64_t(j) * H];
        if (j + 1 < H) v[1] = wc[int64_t(j + 1) * H];
        if (j + 8 < H) v[2] = wc[int64_t(j + 8) * H];
        if (j + 9 < H) v[3] = wc[int64_t(j + 9) * H];
      }
      bf[s][nt][0] = pack_bf16(v[0], v[1]);
      bf[s][nt][1] = pack_bf16(v[2], v[3]);
    }
  }
  if (wrp < kBwdCols) { dh_s[wrp][lane] = 0.0f; dc_s[wrp][lane] = 0.0f; }
  __syncthreads();
  const int64_t gs = int64_t(B) * Hq;
  const int chunks_per_row = Hq / 8;
  uint4* Xs4 = reinterpret_cast<uint4*>(Xs);
  int it = 0;
  const int q = wrp;  // phase A: thread = (batch row lane, unit k0 + wrp)
  const bool actA = (wrp < kBwdCols && lane < rows && k0 + q < H);
  float n_ig = 0.f, n_fg = 0.f, n_gg = 0.f, n_og = 0.f, n_dy = 0.f, n_cs = 0.f, n_cm = 0.f, n_nd = 0.f, n_ndn = 0.f;
  auto prefetch = [&](int t) {
    if (!actA || t < 0) return;
    const int64_t r0 = int64_t(t) * B;
    const int64_t i = (r0 + lane) * H + k0 + q, g = (r0 + lane) * 4 * H + k0 + q;
    n_ig = a.gates[g]; n_fg = a.gates[g + H]; n_gg = a.gates[g + 2 * H]; n_og = a.gates[g + 3 * H];
    n_dy = a.dy[i]; n_cs = a.cs[i]; n_cm = a.cm[i]; n_nd = a.nd[r0 + lane];
    n_ndn = (t + 1 < a.T1) ? a.nd[r0 + B + lane] : 0.f;
  };
  prefetch(a.T1 - 1);
  float bs_i = 0.f, bs_f = 0.f, bs_g = 0.f, bs_o = 0.f;  // bias gradients: this thread's (row, unit) summed over time
  auto store_dg = [&](int64_t row, float p_i, float p_f, float p_g, float p_o) {
    __nv_bfloat16* d = a.dgb + row * a.lg + k0 + q;
    d[0] = __float2bfloat16_rn(p_i); d[H] = __float2bfloat16_rn(p_f);
    d[2 * H] = __float2bfloat16_rn(p_g); d[3 * H] = __float2bfloat16_rn(p_o);
  };
  for (int t = a.T1 - 1; t >= 0; --t, ++it) {
    const int64_t row0 = int64_t(t) * B;
    __nv_bfloat16* dgq_t = a.dgq + int64_t(it & 1) * 4 * gs;
    float p_i = 0.f, p_f = 0.f, p_g = 0.f, p_o = 0.f;
    if (actA) {
      const float ig = n_ig, fg = n_fg, gg = n_gg, og = n_og;
      float dh = n_dy;
      float dc = 0.0f;
      if (it > 0) {
        dh += dh_s[q][lane] * n_ndn;
        dc = dc_s[q][lane];
      }
      const float tc = tanhf(n_cs);
      const float d_o = dh * tc;
      dc += dh * og * (1.0f - tc * tc);
      const float d_i = dc * gg, d_f = dc * n_cm, d_g = dc * ig;
      p_i = d_i * ig * (1.0f - ig); p_f = d_f * fg * (1.0f - fg);
      p_g = d_g * (1.0f - gg * gg); p_o = d_o * og * (1.0f - og);
      dc_s[q][lane] = dc * fg * n_nd;
      bs_i += p_i; bs_f += p_f; bs_g += p_g; bs_o += p_o;
    }
    if (t == 0) {
      if (actA) store_dg(row0 + lane, p_i, p_f, p_g, p_o);
      break;
    }
    // publish this CTA's 8 columns of the four gate-gradient tiles with 16-byte stores (staged through smem:
    // 128 full-sector stores instead of 1024 scattered 2-byte ones ahead of the grid release)
    if (wrp < kBwdCols) {
      stg_s[0][lane][q] = __float2bfloat16_rn(p_i); stg_s[1][lane][q] = __float2bfloat16_rn(p_f);
      stg_s[2][lane][q] = __float2bfloat16_rn(p_g); stg_s[3][lane][q] = __float2bfloat16_rn(p_o);
    }
    __syncthreads();
    if (tid < 128 && (tid & 31) < rows) {
      const int g = tid >> 5, bb = tid & 31;
      *reinterpret_cast<uint4*>(dgq_t + int64_t(g) * gs + int64_t(bb) * Hq + k0) = *reinterpret_cast<const uint4*>(&stg_s[g][bb][0]);
    }
    __syncthreads();
    if (tid == 0) {
      red_release_add(a.counter, 1u);
      grid_wait(a.counter, unsigned(it + 1) * a.nctas);
    }
    if (actA) store_dg(row0 + lane, p_i, p_f, p_g, p_o);
    prefetch(t - 1);
    __syncthreads();
    // all four gate-gradient tiles of this step: [4][rows][Hq] bf16, L2 -> smem as per-thread async 16-byte copies
    // (up to 20 in flight per thread, no staging registers)
    {
      const int nchunk = rows * chunks_per_row;
#pragma unroll
      for (int gg = 0; gg < 4; ++gg) {
        const uint4* src = reinterpret_cast<const uint4*>(dgq_t + int64_t(gg) * gs);
        uint4* dst = Xs4 + int64_t(gg) * 32 * chunks_per_row;
#pragma unroll
        for (int u = 0; u < 5; ++u) {
          const int i = tid + u * kStepThreads;
          if (i < nchunk) cp_async16(dst + i, src + i);
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    float acc[2][kBwdNT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < kBwdNT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
#pragma unroll
    for (int s = 0; s < kMaxKStepsBwd; ++s) {
      const int st = ks0 + s;
      if (st < ks1) {
        const int g = st / kpg, kk = (st % kpg) * 16;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          uint32_t af[4];
          ldmatrix_x4(af, Xs + (int64_t(g) * 32 + mt * 16 + (lane & 15)) * Hq + kk + (lane >> 4) * 8);
#pragma unroll
          for (int nt = 0; nt < kBwdNT; ++nt) mma_bf16_16816(acc[mt][nt], af, bf[s][nt][0], bf[s][nt][1]);
        }
      }
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < kBwdNT; ++nt) {
        const int r = mt * 16 + (lane >> 2), c = nt * 8 + (lane & 3) * 2;
        part16_s[wrp][c][r] = acc[mt][nt][0]; part16_s[wrp][c + 1][r] = acc[mt][nt][1];
        part16_s[wrp][c][r + 8] = acc[mt][nt][2]; part16_s[wrp][c + 1][r + 8] = acc[mt][nt][3];
      }
    __syncthreads();
    if (wrp < kBwdCols) {
      float d = 0.f;
#pragma unroll
      for (int sidx = 0; sidx < 16; ++sidx) d += part16_s[sidx][wrp][lane];
      dh_s[wrp][lane] = d;
    }
    __syncthreads();
  }
  // bias gradients: fold the 32 batch rows of each unit (fixed order: time inside the thread, rows by shuffles)
  if (wrp < kBwdCols) {
    bs_i = warp_sum(bs_i); bs_f = warp_sum(bs_f); bs_g = warp_sum(bs_g); bs_o = warp_sum(bs_o);
    if (lane == 0 && k0 + q < H) {
      a.db[k0 + q] = bs_i; a.db[H + k0 + q] = bs_f; a.db[2 * H + k0 + q] = bs_g; a.db[3 * H + k0 + q] = bs_o;
    }
  }
}

// ---- two stacked layers, backward, as ONE wavefront -------------------------------------------
// The lower layer at time t needs dL/d(its output)[t] = dgates_upper[t] . W_ih_upper, and the upper layer's CTAs
// already hold the tile dgates_upper[t] in shared memory for their own recurrent product.  So the grid is
// role-split: CTAs [0, nc) run the UPPER layer's recurrence (as lstm_bwd_persistent_mma_kernel) and, from the same
// tile, ALSO produce their 8 columns of dL/dh_lower[t] (W_ih_upper^T fragments staged in shared memory);
// CTAs [nc, 2nc) run the LOWER layer's recurrence two wave steps behind (the product for time t is written after
// barrier s and must be visible before it is prefetched).  T+2 grid barriers instead of 2T, no hoisted
// input-gradient GEMM for the upper layer, and 130 instead of 65 SMs busy.
struct WaveBwdArgs {
  const float* w_hh_up; const float* w_hh_lo; const float* w_ih_up;
  const float* dy;                  // dL/d(upper output) [T1*B, H]
  const float* nd;
  const float* gates_up; const float* cs_up; const float* cm_up;
  const float* gates_lo; const float* cs_lo; const float* cm_lo;
  __nv_bfloat16* dgb_up; __nv_bfloat16* dgb_lo; int lg;
  float* db_up; float* db_lo;
  __nv_bfloat16* dgq_up; __nv_bfloat16* dgq_lo;   // each [2][4, B, Hq]
  float* dxm;                       // [T1*B, H] dL/d(lower output): written by the upper role, read by the lower
  unsigned* counter;
  int T1, B, H, Hq; unsigned nc;    // nc = CTAs per role
};

__global__ void __launch_bounds__(kStepThreads) lstm2_bwd_wave_mma_kernel(WaveBwdArgs a) {
  extern __shared__ __align__(128) unsigned char smem_b[];
  __nv_bfloat16* Xs = reinterpret_cast<__nv_bfloat16*>(smem_b);  // [4 gates][32][Hq]
  __shared__ float part16_s[16][kBwdCols][33];
  __shared__ float part16b_s[16][kBwdCols][33];
  __shared__ float dh_s[kBwdCols][33];
  __shared__ float dc_s[kBwdCols][33];
  __shared__ __align__(16) __nv_bfloat16 stg_s[4][32][kBwdCols];
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hq = a.Hq, B = a.B;
  const bool upper = blockIdx.x < a.nc;
  const int k0 = int(upper ? blockIdx.x : blockIdx.x - a.nc) * kBwdCols;
  const int rows = B < 32 ? B : 32;
  const int kpg = (H + 15) / 16;           // k16 steps per gate
  const int ksteps = 4 * kpg;
  const int kper = (ksteps + 15) / 16;
  const int ks0 = wrp * kper, ks1 = (ks0 + kper < ksteps) ? ks0 + kper : ksteps;
  uint2* Wih_s = reinterpret_cast<uint2*>(smem_b + size_t(4) * 32 * Hq * 2);  // [16 warps][kper][32 lanes] fragments
  const float* const w_hh = upper ? a.w_hh_up : a.w_hh_lo;
  const float* const gates = upper ? a.gates_up : a.gates_lo;
  const float* const cs = upper ? a.cs_up : a.cs_lo;
  const float* const cm = upper ? a.cm_up : a.cm_lo;
  __nv_bfloat16* const dgb = upper ? a.dgb_up : a.dgb_lo;
  __nv_bfloat16* const dgq = upper ? a.dgq_up : a.dgq_lo;
  // B fragments: B[kk][n] = W[g*H + j][k0 + n], kk = g*kpg*16 + j  (W = this role's W_hh; the upper role also
  // stages the same fragments of W_ih_upper in shared memory)
  auto load_frag = [&](const float* w, int st, uint32_t& f0, uint32_t& f1) {
    const int g = st / kpg, j = (st % kpg) * 16 + (lane & 3) * 2;
    const int n = lane >> 2;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (st < ks1 && k0 + n < H) {
      const float* wc = w + int64_t(g) * H * H + (k0 + n);
      if (j < H) v[0] = wc[int64_t(j) * H];
      if (j + 1 < H) v[1] = wc[int64_t(j + 1) * H];
      if (j + 8 < H) v[2] = wc[int64_t(j + 8) * H];
      if (j + 9 < H) v[3] = wc[int64_t(j + 9) * H];
    }
    f0 = pack_bf16(v[0], v[1]);
    f1 = pack_bf16(v[2], v[3]);
  };
  uint32_t bf[kMaxKStepsBwd][2];
#pragma unroll
  for (int s = 0; s < kMaxKStepsBwd; ++s) load_frag(w_hh, ks0 + s, bf[s][0], bf[s][1]);
  if (upper) {
    for (int s = 0; s < kper; ++s) {
      uint32_t f0, f1;
      load_frag(a.w_ih_up, ks0 + s, f0, f1);
      Wih_s[(wrp * kper + s) * 32 + lane] = make_uint2(f0, f1);
    }
  }
  if (wrp < kBwdCols) { dh_s[wrp][lane] = 0.0f; dc_s[wrp][lane] = 0.0f; }
  __syncthreads();
  const int64_t gs = int64_t(B) * Hq;
  const int chunks_per_row = Hq / 8;
  uint4* Xs4 = reinterpret_cast<uint4*>(Xs);
  const int q = wrp;  // pointwise role: thread = (batch row lane, unit k0 + wrp)
  const bool actA = (wrp < kBwdCols && lane < rows && k0 + q < H);
  // role time line: the upper layer handles t = T1-1-s at wave step s, the lower layer t = T1+1-s
  auto time_of = [&](int s) { return upper ? a.T1 - 1 - s : a.T1 + 1 - s; };
  float n_ig = 0.f, n_fg = 0.f, n_gg = 0.f, n_og = 0.f, n_dy = 0.f, n_cs = 0.f, n_cm = 0.f, n_nd = 0.f, n_ndn = 0.f;
  auto prefetch = [&](int t) {
    if (!actA || t < 0 || t >= a.T1) return;
    const int64_t r0 = int64_t(t) * B;
    const int64_t i = (r0 + lane) * H + k0 + q, g = (r0 + lane) * 4 * H + k0 + q;
    n_ig = gates[g]; n_fg = gates[g + H]; n_gg = gates[g + 2 * H]; n_og = gates[g + 3 * H];
    if (upper) n_dy = a.dy[i];  // the lower role's dy comes from the upper role: fetched AFTER the barrier (fetch_dxm)
    n_cs = cs[i]; n_cm = cm[i]; n_nd = a.nd[r0 + lane];
    n_ndn = (t + 1 < a.T1) ? a.nd[r0 + B + lane] : 0.f;
  };
  auto fetch_dxm = [&](int t) {
    if (upper || !actA || t < 0 || t >= a.T1) return;
    n_dy = __ldcg(a.dxm + (int64_t(t) * B + lane) * H + k0 + q);
  };
  if (upper) prefetch(a.T1 - 1);
  float bs_i = 0.f, bs_f = 0.f, bs_g = 0.f, bs_o = 0.f;
  auto store_dg = [&](int64_t row, float p_i, float p_f, float p_g, float p_o) {
    __nv_bfloat16* d = dgb + row * a.lg + k0 + q;
    d[0] = __float2bfloat16_rn(p_i); d[H] = __float2bfloat16_rn(p_f);
    d[2 * H] = __float2bfloat16_rn(p_g); d[3 * H] = __float2bfloat16_rn(p_o);
  };
  const int last_s = a.T1 + 1;
  int it = 0;  // this role's active-step counter
  for (int s = 0; s <= last_s; ++s) {
    const int t = time_of(s);
    const bool active = (t >= 0 && t < a.T1);
    const int64_t row0 = int64_t(active ? t : 0) * B;
    __nv_bfloat16* dgq_t = dgq + int64_t(it & 1) * 4 * gs;
    float p_i = 0.f, p_f = 0.f, p_g = 0.f, p_o = 0.f;
    if (active) {
      if (actA) {
        const float ig = n_ig, fg = n_fg, gg = n_gg, og = n_og;
        float dh = n_dy;
        float dc = 0.0f;
        if (it > 0) {
          dh += dh_s[q][lane] * n_ndn;
          dc = dc_s[q][lane];
        }
        const float tc = tanhf(n_cs);
        const float d_o = dh * tc;
        dc += dh * og * (1.0f - tc * tc);
        const float d_i = dc * gg, d_f = dc * n_cm, d_g = dc * ig;
        p_i = d_i * ig * (1.0f - ig); p_f = d_f * fg * (1.0f - fg);
        p_g = d_g * (1.0f - gg * gg); p_o = d_o * og * (1.0f - og);
        dc_s[q][lane] = dc * fg * n_nd;
        bs_i += p_i; bs_f += p_f; bs_g += p_g; bs_o += p_o;
      }
      // publish this CTA's 8 columns of the four gate-gradient tiles (16-byte stores staged through smem)
      if (wrp < kBwdCols) {
        stg_s[0][lane][q] = __float2bfloat16_rn(p_i); stg_s[1][lane][q] = __float2bfloat16_rn(p_f);
        stg_s[2][lane][q] = __float2bfloat16_rn(p_g); stg_s[3][lane][q] = __float2bfloat16_rn(p_o);
      }
      __syncthreads();
      if (tid < 128 && (tid & 31) < rows) {
        const int g = tid >> 5, bb = tid & 31;
        *reinterpret_cast<uint4*>(dgq_t + int64_t(g) * gs + int64_t(bb) * Hq + k0) = *reinterpret_cast<const uint4*>(&stg_s[g][bb][0]);
      }
    }
    if (s == last_s) {
      if (active && actA) store_dg(row0 + lane, p_i, p_f, p_g, p_o);
      break;
    }
    __syncthreads();
    if (tid == 0) {
      red_release_add(a.counter, 1u);
      grid_wait(a.counter, unsigned(s + 1) * 2u * a.nc);
    }
    if (active && actA) store_dg(row0 + lane, p_i, p_f, p_g, p_o);
    prefetch(time_of(s + 1));  // forward-pass operands only: overlaps the barrier wait
    __syncthreads();
    fetch_dxm(time_of(s + 1));  // written by the upper role before it arrived at this barrier
    // post-barrier products from the tile this role published at this wave step: the recurrent carry for time t-1,
    // and (upper role) dL/dh_lower[t]
    const bool need_rec = active && t > 0;
    const bool need_dx = active && upper;
    if (need_rec || need_dx) {
      const int nchunk = rows * chunks_per_row;
#pragma unroll
      for (int gg = 0; gg < 4; ++gg) {
        const uint4* src = reinterpret_cast<const uint4*>(dgq_t + int64_t(gg) * gs);
        uint4* dst = Xs4 + int64_t(gg) * 32 * chunks_per_row;
#pragma unroll
        for (int u = 0; u < 5; ++u) {
          const int i = tid + u * kStepThreads;
          if (i < nchunk) cp_async16(dst + i, src + i);
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();
      // one sweep over the tile feeds both products (the A fragments are loaded once): acc0 with this role's W_hh^T
      // fragments (registers) -> recurrent carry, acc1 with W_ih_upper^T fragments (shared memory) -> dL/dh_lower
      float acc0[2][4], acc1[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) { acc0[mt][e] = 0.f; acc1[mt][e] = 0.f; }
#pragma unroll
      for (int sk = 0; sk < kMaxKStepsBwd; ++sk) {
        const int st = ks0 + sk;
        if (st < ks1) {
          const int g = st / kpg, kk = (st % kpg) * 16;
          uint2 w = make_uint2(0u, 0u);
          if (need_dx) w = Wih_s[(wrp * kper + sk) * 32 + lane];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            uint32_t af[4];
            ldmatrix_x4(af, Xs + (int64_t(g) * 32 + mt * 16 + (lane & 15)) * Hq + kk + (lane >> 4) * 8);
            if (need_rec) mma_bf16_16816(acc0[mt], af, bf[sk][0], bf[sk][1]);
            if (need_dx) mma_bf16_16816(acc1[mt], af, w.x, w.y);
          }
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r = mt * 16 + (lane >> 2), c = (lane & 3) * 2;
        part16_s[wrp][c][r] = acc0[mt][0]; part16_s[wrp][c + 1][r] = acc0[mt][1];
        part16_s[wrp][c][r + 8] = acc0[mt][2]; part16_s[wrp][c + 1][r + 8] = acc0[mt][3];
        part16b_s[wrp][c][r] = acc1[mt][0]; part16b_s[wrp][c + 1][r] = acc1[mt][1];
        part16b_s[wrp][c][r + 8] = acc1[mt][2]; part16b_s[wrp][c + 1][r + 8] = acc1[mt][3];
      }
      __syncthreads();
      if (wrp < kBwdCols) {            // warps 0..7: recurrent carry
        if (need_rec) {
          float d = 0.f;
#pragma unroll
          for (int sidx = 0; sidx < 16; ++sidx) d += part16_s[sidx][wrp][lane];
          dh_s[wrp][lane] = d;
        }
      } else if (need_dx) {            // warps 8..15: dL/dh_lower[t], this CTA's 8 columns
        const int cw = wrp - kBwdCols;
        float d = 0.f;
#pragma unroll
        for (int sidx = 0; sidx < 16; ++sidx) d += part16b_s[sidx][cw][lane];
        if (lane < rows && k0 + cw < H) a.dxm[(row0 + lane) * H + k0 + cw] = d;
      }
      __syncthreads();
    }
    if (active) ++it;
  }
  if (wrp < kBwdCols) {
    bs_i = warp_sum(bs_i); bs_f = warp_sum(bs_f); bs_g = warp_sum(bs_g); bs_o = warp_sum(bs_o);
    float* db = upper ? a.db_up : a.db_lo;
    if (lane == 0 && k0 + q < H) {
      db[k0 + q] = bs_i; db[H + k0 + q] = bs_f; db[2 * H + k0 + q] = bs_g; db[3 * H + k0 + q] = bs_o;
    }
  }
}

// hmq[0][b][:] = bf16(h0 * nd_0), zero padded; cm[0] = c0 * nd_0
__global__ void lstm_init_state_q_kernel(const float* __restrict__ h0, const float* __restrict__ c0,
                                         const float* __restrict__ nd, __nv_bfloat16* __restrict__ hmq,
                                         float* __restrict__ cm, int B, int H, int Hq,
                                         __nv_bfloat16* __restrict__ hq_raw = nullptr) {
  const int64_t total = int64_t(B) * Hq;
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = int(i / Hq), k = int(i % Hq);
  if (k < H) {
    hmq[i] = __float2bfloat16_rn(h0[int64_t(b) * H + k] * nd[b]);
    if (hq_raw) hq_raw[i] = __float2bfloat16_rn(h0[int64_t(b) * H + k]);
    cm[int64_t(b) * H + k] = c0[int64_t(b) * H + k] * nd[b];
  } else {
    hmq[i] = __float2bfloat16_rn(0.0f);
    if (hq_raw) hq_raw[i] = __float2bfloat16_rn(0.0f);
  }
}


// =========================================================================================
// Split-precision ("bf16x3") recurrence, forward, two stacked layers as one wavefront (precision 2).
//
// Same wavefront as lstm2_fwd_wave_mma_kernel (layer 0 at t = s, layer 1 at t = s-1 per wave step, the
// layer-1 input projection riding on the pass), but every MMA operand is a hi/lo bf16 PAIR (x = hi + lo,
// hi.hi + hi.lo + lo.hi in fp32: ~2^-17 relative per product, fp32-grade) so that the recurrence holds the
// 1e-4 parity contract the bf16 kernel cannot.  What changed with the 3x MMA count (tools/ubench/ubench_lstm.cu
// measures the mma.sync, gather and hand-off rates this layout is built around):
//   * 11 MMA warps x 3 k16-steps cover K = 528 exactly (33 k-steps): no padded k-steps, weights of all three
//     matrices as hi AND lo B fragments in registers (72 per thread) for all steps;
//   * h is exchanged as two bf16 planes (hq: raw h, slot t+1 = h_t) written with 8-byte stores (4 units x
//     bf16 of one row and plane) and pulled per warp as TMA boxes of its 48 (+8) columns; the CTAs run as 2-CTA
//     clusters and each CTA of a pair loads one 16-row half and multicasts it, so the pair reads each tile once;
//   * the cell state lives in a register of the thread that owns (layer, unit, row) for all steps;
//   * the grid barrier is per-CTA FLAGS instead of one contended counter: producer = stores, bar.sync,
//     fence.acq_rel.gpu, st flag[cta] = step; consumers = one thread per producer
//     spinning on its flag with relaxed loads, one acquire load, bar.sync.
// CTA = kStepUnits hidden units x 4 gates of BOTH layers, B <= 32 rows, ceil(H/16) <= 33.
// =========================================================================================
constexpr int kFlagStride = 32;   // one flag per 128-byte line: 130 CTAs polling 130 flags packed into 5 lines make those
                                  // lines' L2 slices the bottleneck
constexpr int kSplitWarps = 11;
constexpr int kSplitThreads = kSplitWarps * 32;
constexpr int kSplitK = 3;  // k16 steps per warp

struct WaveFwdSplitArgs {
  const float* w_hh0; const float* w_ih1; const float* w_hh1; const float* bias1;
  const float* c0;          // [2, B, H] initial cell state
  const float* xproj;       // layer 0: hoisted input projection + biases [T1*B, 4H]
  // What only the LSTM kernels themselves consume is kept in CTA-BLOCKED layouts so that every access is a coalesced
  // run (a [T1*B, 4H] / [T1*B, H] layout makes each warp store touch 32 cache lines - the LSU time of those scattered
  // 4-byte stores sat in front of the next step's tile fetch: ncu / clock64 trace r2):
  float* gact[2];           // activated gates [T1][nctas][32 rows][16 = gate*4 + unit]
  float* csb[2];            // cell state [T1+1][nctas][32 rows][4 units]: slot 0 = c0, slot t+1 = c_t
  float* y;                 // layer-1 output [T1*B, H] (the heads' input)
  float* hN; float* cN;     // [2, B, H] final state
  __nv_bfloat16* hq[2];     // raw h planes [(T1+1)*B, Hq] (+ hq_lo): slot 0 = initial state, slot t+1 = h_t
  __nv_bfloat16* hmq[2];    // masked recurrent inputs [T1*B, Hq] (+ hmq_lo): operand of the weight-gradient GEMMs
  int64_t hq_lo, hmq_lo;
  const float* nd; unsigned* flags;
  int T1, B, H, Hq; unsigned nctas;
};

__device__ __forceinline__ void split_pack(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void st_relaxed_u32(unsigned* p, unsigned v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// ---- 2-CTA cluster tile exchange of the split kernels: each CTA of a pair loads one 16-row half of every tile box and
// multicasts it into both CTAs' shared memory (halves the L2 -> SM traffic of the all-gather: tools/ubench/ubench_lstm.cu)
constexpr int kTileRowE = kSplitK * 16 + 8;     // elements per tile row: a warp's 48 columns + 8 (112 B: conflict-free ldmatrix)
constexpr int kHalfE = 2 * 16 * kTileRowE;      // one box: [hi, lo][16 rows][kTileRowE]
constexpr uint32_t kSlotBytes = 2 * kHalfE * 2; // both row halves of one tile slot
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the peer CTA's copy of a local shared-memory mbarrier
__device__ __forceinline__ uint32_t peer_addr(const void* p, uint32_t peer) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(peer));
  return r;
}
__device__ __forceinline__ void mbar_arrive_local(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}
// wait on an mbarrier phase that the peer CTA's warp also arrives on (acquire at cluster scope)
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LAB_DONE_%=;\n"
      "bra LAB_WAIT_%=;\n"
      "LAB_DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// generic-proxy global writes (h / gate-gradient stores) vs the TMA reads of the same bytes
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// one box of a rank-4 / rank-5 map into the same shared-memory offset of both CTAs of the pair; completes tx on the
// mbarrier at `bar`'s offset in each of them
__device__ __forceinline__ void tma_multicast_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(
          smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"((uint16_t)3)
      : "memory");
}
__device__ __forceinline__ void tma_multicast_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5, %6, %7}], [%2], %8;" ::"r"(
          smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "h"((uint16_t)3)
      : "memory");
}
// 128-byte aligned start of the dynamic shared memory (TMA destinations); the kernels request 128 bytes of slack
__device__ __forceinline__ unsigned char* smem_align128(unsigned char* p) {
  return p + ((128u - (smem_u32(p) & 127u)) & 127u);
}

// hi.hi + hi.lo + lo.hi (small terms first) of one m16n8k16 tile product
__device__ __forceinline__ void mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint32_t bh0, uint32_t bh1,
                                     uint32_t bl0, uint32_t bl1) {
  mma_bf16_16816(c, al, bh0, bh1);
  mma_bf16_16816(c, ah, bl0, bl1);
  mma_bf16_16816(c, ah, bh0, bh1);
}

// hq_map[l]: the hq planes of layer l as a rank-4 map {Hq, B, T1 + 1, plane}, box {kTileRowE, 16, 1, 2}: rows >= B and
// columns >= Hq are zero-filled.  Launched as 2-CTA clusters; a padding CTA (index >= a.nctas, all units past H) only
// takes part in the loads.
__global__ void __launch_bounds__(kSplitThreads, 1) lstm2_fwd_wave_split_kernel(const __grid_constant__ CUtensorMap hq_map0,
                                                                               const __grid_constant__ CUtensorMap hq_map1,
                                                                               WaveFwdSplitArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* const smem_b = smem_align128(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hq = a.Hq, B = a.B;
  const bool idle = blockIdx.x >= a.nctas;
  // warp-private tiles [group: h0, h1][row half = CTA rank that loads it][hi, lo][16 rows][kTileRowE] of this warp's 48 columns
  __nv_bfloat16* const X = reinterpret_cast<__nv_bfloat16*>(smem_b) + int64_t(wrp) * 4 * kHalfE;
  typedef float PartT[2][16][33];
  PartT* part = reinterpret_cast<PartT*>(smem_b + size_t(kSplitWarps) * 2 * kSlotBytes);  // [11 warps][set][col][row]
  __shared__ float act_s[2][4][kStepUnits][33];
  // per warp: full[group] (this CTA's expect_tx, both CTAs' bytes), empty (this warp + the peer CTA's warp done reading)
  __shared__ __align__(8) uint64_t full_s[kSplitWarps][2], empty_s[kSplitWarps];
  const uint32_t rank = cluster_rank();
  if (lane == 0) {
    mbar_init(&full_s[wrp][0], 1); mbar_init(&full_s[wrp][1], 1); mbar_init(&empty_s[wrp], 2);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const uint32_t peer_empty = peer_addr(&empty_s[wrp], rank ^ 1u);
  const int j0 = blockIdx.x * kStepUnits;
  const int rows = (B < 32) ? B : 32;
  const int ksteps = (H + 15) / 16;
  const int ks0 = wrp * kSplitK;
  // B fragments (hi, lo) of this CTA's 16 gate rows (o = gate*4 + unit) of the three weight matrices, this warp's k-steps
  uint32_t bh[3][kSplitK][2][2], bl[3][kSplitK][2][2];
  {
    const float* wm[3] = {a.w_hh0, a.w_ih1, a.w_hh1};
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int sk = 0; sk < kSplitK; ++sk)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int o = nt * 8 + (lane >> 2);
          const int g = o >> 2, u = o & 3;
          const float* wr = wm[m] + (int64_t(g) * H + j0 + u) * H;
          const int k = (ks0 + sk) * 16 + (lane & 3) * 2;
          float v[4] = {0.f, 0.f, 0.f, 0.f};
          if (j0 + u < H && ks0 + sk < ksteps) {
            if (k < H) v[0] = wr[k];
            if (k + 1 < H) v[1] = wr[k + 1];
            if (k + 8 < H) v[2] = wr[k + 8];
            if (k + 9 < H) v[3] = wr[k + 9];
          }
          split_pack(v[0], v[1], bh[m][sk][nt][0], bl[m][sk][nt][0]);
          split_pack(v[2], v[3], bh[m][sk][nt][1], bl[m][sk][nt][1]);
        }
  }
  // activation role (warps 0..7): gate columns c0 = wrp and c1 = wrp + 8 of both layers, row = lane
  const bool actrole = wrp < 8;
  const int cA = wrp, cB = wrp + 8;                     // col = gate*4 + unit
  const bool okA = actrole && lane < rows && j0 + (cA & 3) < H, okB = actrole && lane < rows && j0 + (cB & 3) < H;
  const int64_t gA = int64_t(cA >> 2) * H + j0 + (cA & 3), gB = int64_t(cB >> 2) * H + j0 + (cB & 3);
  const float bias1A = okA ? a.bias1[gA] : 0.f, bias1B = okB ? a.bias1[gB] : 0.f;
  // update role (threads 0..255): layer ul, row ur, unit uu - the 4 units of a row sit in 4 adjacent lanes
  const bool updthread = tid < 256;
  const int ul = tid >> 7, ur = (tid & 127) >> 2, uu = tid & 3;
  const bool updrole = updthread && ur < rows && j0 + uu < H;
  float* const csb_u = ul ? a.csb[1] : a.csb[0];
  __nv_bfloat16* const hq_u = ul ? a.hq[1] : a.hq[0];
  __nv_bfloat16* const hmq_u = ul ? a.hmq[1] : a.hmq[0];
  float c_state = updrole ? a.c0[(int64_t(ul) * B + ur) * H + j0 + uu] : 0.f;  // c_{t-1} of this (layer, row, unit)
  if (updthread && !idle) csb_u[int64_t(blockIdx.x) * 128 + (tid & 127)] = c_state;    // slot 0
  cluster_sync_all();   // the peer's mbarriers are initialised before any multicast or remote arrive
  for (int s = 0; s <= a.T1; ++s) {
    const bool act0 = (s < a.T1), act1 = (s >= 1);
    // inputs that do not depend on other CTAs: issued before the wait
    float preA = 0.f, preB = 0.f;
    if (act0) {
      if (okA) preA = __ldg(a.xproj + (int64_t(s) * B + lane) * 4 * H + gA);
      if (okB) preB = __ldg(a.xproj + (int64_t(s) * B + lane) * 4 * H + gB);
    }
    const int tu = s - ul;                                 // time step of this thread's update role
    const bool upd = updrole && (ul ? act1 : act0);
    float nd_t = 0.f, nd_n = 0.f;
    if (upd) {
      nd_t = __ldg(a.nd + int64_t(tu) * B + ur);
      if (tu < a.T1 - 1) nd_n = __ldg(a.nd + int64_t(tu + 1) * B + ur);
    }
    // Every tile element is consumed by exactly ONE warp (K is split across the warps), so each warp waits only for the
    // CTAs that produce ITS k-range (units [16*ks0, 16*ks0 + 48) -> 12 producer CTAs) and fetches its own columns of the
    // four planes - no block-wide barrier between the hand-off and the products.  The same warp of the peer CTA needs the
    // same columns: each loads one 16-row half and multicasts it to both.  (History: 130 threads per CTA polling 130
    // flag words - 17 k pollers chip-wide on 5 cache lines - made the L2 slices of those lines the bottleneck: ncu
    // showed over a third of all samples in the spin.)
    if (s > 0) {
      const int p0 = (ks0 * 16) / kStepUnits + lane;                   // producer CTA of this lane
      const int pend = (min((ks0 + kSplitK) * 16, H) + kStepUnits - 1) / kStepUnits;
      if (lane < 12 && p0 < pend && p0 < int(a.nctas)) {
        while (ld_relaxed_u32(a.flags + p0 * kFlagStride) < unsigned(s)) {}
        (void)ld_acquire_u32(a.flags + p0 * kFlagStride);
        fence_proxy_async_global();
      }
      __syncwarp();
    }
    if (lane == 0) {
      // Two groups: the h0 planes first, so the layer-0 / input-projection MMAs start while the h1 planes land.  At s = 0
      // the h1 group (slot 0) is loaded but not used, which keeps one phase per step on every barrier.
      if (s > 0) mbar_wait_cluster(&empty_s[wrp], (s - 1) & 1);   // both CTAs' warps have read step s-1's tiles
      fence_proxy_async_global();
      mbar_expect_tx(&full_s[wrp][0], kSlotBytes);
      tma_multicast_4d(X + rank * kHalfE, &hq_map0, &full_s[wrp][0], ks0 * 16, 16 * int(rank), s, 0);
      mbar_expect_tx(&full_s[wrp][1], kSlotBytes);
      tma_multicast_4d(X + (2 + rank) * kHalfE, &hq_map1, &full_s[wrp][1], ks0 * 16, 16 * int(rank), s > 0 ? s - 1 : 0, 0);
    }
    float m0[2][2], m1[2][2];   // done masks of this thread's accumulator rows (layer 0 at t = s, layer 1 at t = s-1)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = mt * 16 + (lane >> 2) + hh * 8;
        m0[mt][hh] = (r < rows && act0) ? __ldg(a.nd + int64_t(s) * B + r) : 0.f;
        m1[mt][hh] = (r < rows && act1) ? __ldg(a.nd + int64_t(s - 1) * B + r) : 0.f;
      }
    {
      float acc0[2][2][4], accI[2][2][4], acc1[2][2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) { acc0[mt][nt][e] = 0.f; accI[mt][nt][e] = 0.f; acc1[mt][nt][e] = 0.f; }
      mbar_wait(&full_s[wrp][0], s & 1);   // the h0 planes
#pragma unroll
      for (int sk = 0; sk < kSplitK; ++sk) {
        if (ks0 + sk < ksteps) {
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {   // m16 tile mt = the row half CTA rank mt loaded
            uint32_t ah[4], al[4];
            const int off = mt * kHalfE + (lane & 15) * kTileRowE + sk * 16 + (lane >> 4) * 8;
            ldmatrix_x4(ah, X + off);
            ldmatrix_x4(al, X + 16 * kTileRowE + off);
            if (act0) {
              mma3(acc0[mt][0], ah, al, bh[0][sk][0][0], bh[0][sk][0][1], bl[0][sk][0][0], bl[0][sk][0][1]);
              mma3(acc0[mt][1], ah, al, bh[0][sk][1][0], bh[0][sk][1][1], bl[0][sk][1][0], bl[0][sk][1][1]);
            }
            if (act1) {
              mma3(accI[mt][0], ah, al, bh[1][sk][0][0], bh[1][sk][0][1], bl[1][sk][0][0], bl[1][sk][0][1]);
              mma3(accI[mt][1], ah, al, bh[1][sk][1][0], bh[1][sk][1][1], bl[1][sk][1][0], bl[1][sk][1][1]);
            }
          }
        }
      }
      mbar_wait(&full_s[wrp][1], s & 1);   // the h1 planes
      if (act1) {
#pragma unroll
        for (int sk = 0; sk < kSplitK; ++sk) {
          if (ks0 + sk < ksteps) {
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
              uint32_t ah[4], al[4];
              const int off = (2 + mt) * kHalfE + (lane & 15) * kTileRowE + sk * 16 + (lane >> 4) * 8;
              ldmatrix_x4(ah, X + off);
              ldmatrix_x4(al, X + 16 * kTileRowE + off);
              mma3(acc1[mt][0], ah, al, bh[2][sk][0][0], bh[2][sk][0][1], bl[2][sk][0][0], bl[2][sk][0][1]);
              mma3(acc1[mt][1], ah, al, bh[2][sk][1][0], bh[2][sk][1][1], bl[2][sk][1][0], bl[2][sk][1][1]);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) {   // this warp's tiles are read: free them for both loaders of step s+1
        mbar_arrive_local(&empty_s[wrp]);
        mbar_arrive_remote(peer_empty);
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r = mt * 16 + (lane >> 2);
        const float m0a = m0[mt][0], m0b = m0[mt][1], m1a = m1[mt][0], m1b = m1[mt][1];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const int c = nt * 8 + (lane & 3) * 2;
          part[wrp][0][c][r] = acc0[mt][nt][0] * m0a; part[wrp][0][c + 1][r] = acc0[mt][nt][1] * m0a;
          part[wrp][0][c][r + 8] = acc0[mt][nt][2] * m0b; part[wrp][0][c + 1][r + 8] = acc0[mt][nt][3] * m0b;
          part[wrp][1][c][r] = accI[mt][nt][0] + acc1[mt][nt][0] * m1a;
          part[wrp][1][c + 1][r] = accI[mt][nt][1] + acc1[mt][nt][1] * m1a;
          part[wrp][1][c][r + 8] = accI[mt][nt][2] + acc1[mt][nt][2] * m1b;
          part[wrp][1][c + 1][r + 8] = accI[mt][nt][3] + acc1[mt][nt][3] * m1b;
        }
      }
    }
    __syncthreads();
    float g0A = 0.f, g0B = 0.f, g1A = 0.f, g1B = 0.f;
    if (actrole) {
      float d0A = 0.f, d0B = 0.f, d1A = 0.f, d1B = 0.f;
#pragma unroll
      for (int w = 0; w < kSplitWarps; ++w) {  // fixed order: deterministic
        d0A += part[w][0][cA][lane]; d0B += part[w][0][cB][lane];
        d1A += part[w][1][cA][lane]; d1B += part[w][1][cB][lane];
      }
      const bool tanhA = (cA >> 2) == 2, tanhB = (cB >> 2) == 2;
      if (act0) {
        if (okA) { const float p = preA + d0A; g0A = tanhA ? tanhf(p) : sigmoidf_(p); }
        if (okB) { const float p = preB + d0B; g0B = tanhB ? tanhf(p) : sigmoidf_(p); }
      }
      if (act1) {
        if (okA) { const float p = bias1A + d1A; g1A = tanhA ? tanhf(p) : sigmoidf_(p); }
        if (okB) { const float p = bias1B + d1B; g1B = tanhB ? tanhf(p) : sigmoidf_(p); }
      }
      act_s[0][cA >> 2][cA & 3][lane] = g0A; act_s[0][cB >> 2][cB & 3][lane] = g0B;
      act_s[1][cA >> 2][cA & 3][lane] = g1A; act_s[1][cB >> 2][cB & 3][lane] = g1B;
    }
    __syncthreads();
    float c_new = 0.f, h_new = 0.f, cm_in = 0.f;
    if (updthread) {
      if (upd) {
        const float ig = act_s[ul][0][uu][ur], fg = act_s[ul][1][uu][ur], gg = act_s[ul][2][uu][ur], og = act_s[ul][3][uu][ur];
        cm_in = c_state * nd_t;      // state *= notdone_t before the step (monobeast.py:603-606)
        c_new = fg * cm_in + ig * gg;
        h_new = og * tanhf(c_new);
        c_state = c_new;
      }
      // publish raw h_t: the 4 units of a row sit in 4 adjacent lanes -> one 8-byte store per (row, plane)
      const bool live = (ul ? act1 : act0);
      const __nv_bfloat16 hh = __float2bfloat16_rn(h_new);
      const __nv_bfloat16 hl = __float2bfloat16_rn(h_new - __bfloat162float(hh));
      const uint32_t vh = uint32_t(__bfloat16_as_ushort(hh)), vl = uint32_t(__bfloat16_as_ushort(hl));
      const uint32_t ph = vh | (__shfl_down_sync(0xffffffffu, vh, 1) << 16), pl = vl | (__shfl_down_sync(0xffffffffu, vl, 1) << 16);
      const uint32_t ph2 = __shfl_down_sync(0xffffffffu, ph, 2), pl2 = __shfl_down_sync(0xffffffffu, pl, 2);
      if (live && !idle && uu == 0 && ur < rows) {
        __nv_bfloat16* d = hq_u + (int64_t(tu + 1) * B + ur) * Hq + j0;
        *reinterpret_cast<uint2*>(d) = make_uint2(ph, ph2);
        *reinterpret_cast<uint2*>(d + a.hq_lo) = make_uint2(pl, pl2);
        fence_proxy_async_global();   // consumers read h through TMA
      }
    }
    __syncthreads();
    if (tid == 0 && s < a.T1 && !idle) {
      asm volatile("fence.acq_rel.gpu;" ::: "memory");
      st_relaxed_u32(a.flags + blockIdx.x * kFlagStride, unsigned(s + 1));
    }
    // ---- everything below is consumed by this CTA or after the kernel: off the critical path ----
    // activated gates -> CTA-blocked [row][16] tiles, straight from act_s (rewritten only after the next step's barrier)
    for (int idx = tid; idx < 1024 && !idle; idx += kSplitThreads) {
      const int l = idx >> 9, e = idx & 511, row = e >> 4, c = e & 15;
      const int tl = s - l;
      if ((l ? act1 : act0) && row < rows)
        a.gact[l][(int64_t(tl) * a.nctas + blockIdx.x) * 512 + e] = act_s[l][c >> 2][c & 3][row];
    }
    if (updthread && !idle) {
      // masked recurrent input of the NEXT step (h_t * notdone_{t+1}) for the weight-gradient GEMMs, as hi / lo planes
      const float hm = h_new * nd_n;
      const __nv_bfloat16 mh = __float2bfloat16_rn(hm);
      const __nv_bfloat16 ml = __float2bfloat16_rn(hm - __bfloat162float(mh));
      const uint32_t vh = uint32_t(__bfloat16_as_ushort(mh)), vl = uint32_t(__bfloat16_as_ushort(ml));
      const uint32_t ph = vh | (__shfl_down_sync(0xffffffffu, vh, 1) << 16), pl = vl | (__shfl_down_sync(0xffffffffu, vl, 1) << 16);
      const uint32_t ph2 = __shfl_down_sync(0xffffffffu, ph, 2), pl2 = __shfl_down_sync(0xffffffffu, pl, 2);
      const bool live = (ul ? act1 : act0) && tu < a.T1 - 1;
      if (live && uu == 0 && ur < rows) {
        __nv_bfloat16* d = hmq_u + (int64_t(tu + 1) * B + ur) * Hq + j0;
        *reinterpret_cast<uint2*>(d) = make_uint2(ph, ph2);
        *reinterpret_cast<uint2*>(d + a.hmq_lo) = make_uint2(pl, pl2);
      }
      if ((ul ? act1 : act0) && ur < rows)   // c_t, blocked (units past H hold 0)
        csb_u[(int64_t(tu + 1) * a.nctas + blockIdx.x) * 128 + (tid & 127)] = c_new;
      if (upd) {
        const int64_t o = (int64_t(tu) * B + ur) * H + j0 + uu;
        if (ul) a.y[o] = h_new;
        if (tu == a.T1 - 1) {
          a.hN[(int64_t(ul) * B + ur) * H + j0 + uu] = h_new;
          a.cN[(int64_t(ul) * B + ur) * H + j0 + uu] = c_new;
        }
      }
    }
  }
  cluster_sync_all();   // no CTA exits with multicast writes or remote arrives into it still in flight
}

// ---- split-precision backward wavefront (precision 2) ----------------------------------------------
// lstm2_bwd_wave_mma_kernel's role split (CTAs [0, nc): upper layer recurrence + dL/dh_lower from the same tile;
// CTAs [nc, 2nc): lower layer two wave steps behind; 8 hidden units per CTA) with hi/lo operand planes:
//   * the four gate-gradient tiles of a step are 4 x (hi + lo) x 34 KB = 274 KB - more than shared memory - so they
//     stream through a 2-deep ring by gate (the multicast TMA boxes of gate g+2 under the MMAs of gate g+1);
//   * 11 MMA warps x 3 k16-steps cover one gate's K = 528 exactly; W_hh^T (and, upper role, W_ih_upper^T) as hi AND lo
//     B fragments in registers (96 per thread);
//   * per-CTA flags instead of the counter barrier (see lstm2_fwd_wave_split_kernel): a CTA waits for the CTAs of its
//     own role (they produce the tile it pulls) and, lower role, for the upper CTA that owns the same 8 columns
//     (it produces this CTA's dL/dh_lower).
struct WaveBwdSplitArgs {
  const float* w_hh_up; const float* w_hh_lo; const float* w_ih_up;
  const float* dy; const float* nd;
  const float* gact_up; const float* csb_up;   // CTA-blocked forward saves (see WaveFwdSplitArgs); nfwd = forward CTAs
  const float* gact_lo; const float* csb_lo;
  int nfwd;
  __nv_bfloat16* dgb_up; __nv_bfloat16* dgb_lo; int lg; int64_t dgb_lo_off;   // gate gradients of all steps, hi plane (+ lo offset)
  float* db_up; float* db_lo;
  __nv_bfloat16* dgq_up; __nv_bfloat16* dgq_lo; int64_t dgq_lo_off;          // exchange planes: [2][4, B, Hq] (+ lo offset)
  float* dxb;                       // dL/dh_lower, blocked [T1][ncol][32 rows][8 cols]: upper role -> lower role
  unsigned* flags;                  // [2 * nc]
  int T1, B, H, Hq;
  unsigned nc;                      // CTAs per role, padded to whole clusters
  unsigned ncol;                    // CTAs per role that own columns < H (= ceil(H / 8))
};

// dgq_map[role]: that role's exchange planes as a rank-5 map {Hq, B, gate, ping-pong buffer, plane}, box
// {kTileRowE, 16, 1, 1, 2}: rows >= B and columns >= Hq are zero-filled.  Launched as 2-CTA clusters, every pair within
// one role; a role's padding CTA (index >= ncol, all columns past H) takes part in the loads and the flag protocol only.
__global__ void __launch_bounds__(kSplitThreads, 1) lstm2_bwd_wave_split_kernel(const __grid_constant__ CUtensorMap dgq_map_up,
                                                                               const __grid_constant__ CUtensorMap dgq_map_lo,
                                                                               WaveBwdSplitArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* const smem_b = smem_align128(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int H = a.H, Hq = a.Hq, B = a.B;
  // Every tile element is consumed by exactly one warp (K = (gate, unit) is split across the warps: this warp owns units
  // [16*ks0, 16*ks0 + 48) of every gate), so the tiles stream through WARP-PRIVATE 2-slot rings - slot = one gate,
  // [row half = CTA rank that loads it][hi, lo][16 rows][kTileRowE] - with no block barrier anywhere in the fetch / MMA
  // phase.  The same warp of the peer CTA streams the same columns: each CTA loads one row half and multicasts it.
  __nv_bfloat16* const X = reinterpret_cast<__nv_bfloat16*>(smem_b) + int64_t(wrp) * 4 * kHalfE;
  typedef float PartT[2][kBwdCols][33];
  PartT* part = reinterpret_cast<PartT*>(smem_b + size_t(kSplitWarps) * 2 * kSlotBytes);  // [11 warps][product][col][row]
  __shared__ float dh_s[kBwdCols][33];
  __shared__ float dc_s[kBwdCols][33];
  __shared__ __align__(16) __nv_bfloat16 stg_s[2][4][32][kBwdCols];       // [plane][gate][row][col]
  // per warp and ring slot: full (this CTA's expect_tx, both CTAs' bytes), empty (this warp + the peer CTA's warp done)
  __shared__ __align__(8) uint64_t full_s[kSplitWarps][2], empty_s[kSplitWarps][2];
  const uint32_t rank = cluster_rank();
  if (lane == 0) {
    mbar_init(&full_s[wrp][0], 1); mbar_init(&full_s[wrp][1], 1);
    mbar_init(&empty_s[wrp][0], 2); mbar_init(&empty_s[wrp][1], 2);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const uint32_t peer_empty0 = peer_addr(&empty_s[wrp][0], rank ^ 1u), peer_empty1 = peer_addr(&empty_s[wrp][1], rank ^ 1u);
  const bool upper = blockIdx.x < a.nc;
  const CUtensorMap* const dgq_map = upper ? &dgq_map_up : &dgq_map_lo;
  const int cidx = int(upper ? blockIdx.x : blockIdx.x - a.nc);
  const int k0 = cidx * kBwdCols;
  const int rows = B < 32 ? B : 32;
  const int kpg = (H + 15) / 16;           // k16 steps per gate (<= 33)
  const int ks0 = wrp * kSplitK;           // this warp's k-steps inside every gate
  const float* const w_hh = upper ? a.w_hh_up : a.w_hh_lo;
  const float* const gact = upper ? a.gact_up : a.gact_lo;
  const float* const csb = upper ? a.csb_up : a.csb_lo;
  __nv_bfloat16* const dgb = upper ? a.dgb_up : a.dgb_lo;
  __nv_bfloat16* const dgq = upper ? a.dgq_up : a.dgq_lo;
  const bool idle = cidx >= int(a.ncol);
  // B fragments: B[kk][n] = W[g*H + j][k0 + n] for kk = (gate g, j)
  uint32_t bh[4][kSplitK][2], bl[4][kSplitK][2], ih[4][kSplitK][2], il[4][kSplitK][2];
  // The pointwise operands of the NEXT step (forward saves: 4 gates, c, masked c_prev, dy, 2 done masks) are prefetched
  // into SHARED memory with 4-byte cp.async while this step's hand-off and products run: held in registers they spilled
  // to local memory (168-register cap with the 96 fragment registers) and their load latency landed on the critical path.
  // layout: [0,1024) activated gates of the two forward CTAs whose units this CTA owns ([2][32 rows][16]); [1024,1280) c_t
  // ([2][32][4]); [1280,1536) c_{t-1}; [1536,1792) dy ([32 rows][8 cols], upper role); [1792,1856) notdone_t, notdone_{t+1}
  float* const pre_s = reinterpret_cast<float*>(smem_b + size_t(kSplitWarps) * 2 * kSlotBytes + sizeof(float) * kSplitWarps * 2 * kBwdCols * 33);
  {
    const int n = lane >> 2;
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
      for (int sk = 0; sk < kSplitK; ++sk) {
        const int j = (ks0 + sk) * 16 + (lane & 3) * 2;
        float v[4] = {0.f, 0.f, 0.f, 0.f}, u[4] = {0.f, 0.f, 0.f, 0.f};
        if (ks0 + sk < kpg && k0 + n < H) {
          const float* wc = w_hh + int64_t(g) * H * H + (k0 + n);
          const float* ic = a.w_ih_up + int64_t(g) * H * H + (k0 + n);
          if (j < H) { v[0] = wc[int64_t(j) * H]; if (upper) u[0] = ic[int64_t(j) * H]; }
          if (j + 1 < H) { v[1] = wc[int64_t(j + 1) * H]; if (upper) u[1] = ic[int64_t(j + 1) * H]; }
          if (j + 8 < H) { v[2] = wc[int64_t(j + 8) * H]; if (upper) u[2] = ic[int64_t(j + 8) * H]; }
          if (j + 9 < H) { v[3] = wc[int64_t(j + 9) * H]; if (upper) u[3] = ic[int64_t(j + 9) * H]; }
        }
        split_pack(v[0], v[1], bh[g][sk][0], bl[g][sk][0]);
        split_pack(v[2], v[3], bh[g][sk][1], bl[g][sk][1]);
        split_pack(u[0], u[1], ih[g][sk][0], il[g][sk][0]);
        split_pack(u[2], u[3], ih[g][sk][1], il[g][sk][1]);
      }
  }
  if (wrp < kBwdCols) { dh_s[wrp][lane] = 0.0f; dc_s[wrp][lane] = 0.0f; }
  cluster_sync_all();   // also: the peer's mbarriers are initialised before any multicast or remote arrive
  const int64_t gs = int64_t(B) * Hq;      // one gate of one exchange buffer
  const int q = wrp;  // pointwise role: thread = (batch row lane, unit k0 + wrp), warps 0..7
  const bool actA = (wrp < kBwdCols && lane < rows && k0 + q < H);
  auto time_of = [&](int s) { return upper ? a.T1 - 1 - s : a.T1 + 1 - s; };
  float n_dy = 0.f;
  auto prefetch = [&](int t) {   // every thread commits one group; all copies are coalesced runs
    if (t >= 0 && t < a.T1) {
      for (int idx = tid; idx < 384; idx += kSplitThreads) {
        const float* src; float* dst;
        if (idx < 256) {          // activated gates: 2 forward-CTA blocks x 128 chunks
          const int blk = idx >> 7, fc = 2 * cidx + blk;
          src = gact + (int64_t(t) * a.nfwd + fc) * 512 + (idx & 127) * 4; dst = pre_s + idx * 4;
          if (fc >= a.nfwd) src = nullptr;
        } else {                  // c_t (slot t+1) and c_{t-1} (slot t): 2 blocks x 32 chunks each
          const int j = idx - 256, prev = j >> 6, blk = (j >> 5) & 1, fc = 2 * cidx + blk;
          src = csb + (int64_t(t + 1 - prev) * a.nfwd + fc) * 128 + (j & 31) * 4; dst = pre_s + 1024 + j * 4;
          if (fc >= a.nfwd) src = nullptr;
        }
        if (src) cp_async16(dst, src);
      }
      if (upper && tid < 256) {   // dy rows of this CTA's 8 columns
        const int r = tid >> 3, c = tid & 7;
        if (r < rows && k0 + c < H)
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(pre_s + 1536 + tid)),
                       "l"(a.dy + (int64_t(t) * B + r) * H + k0 + c) : "memory");
      }
      if (tid < 64) {
        const int r = tid & 31, tt = t + (tid >> 5);
        if (r < rows && tt < a.T1)
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(pre_s + 1792 + tid)), "l"(a.nd + int64_t(tt) * B + r) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto fetch_dxm = [&](int t) {
    if (upper || !actA || t < 0 || t >= a.T1) return;
    n_dy = __ldcg(a.dxb + (int64_t(t) * a.ncol + cidx) * 256 + lane * 8 + q);
  };
  // gate-gradient rows of all steps for the hoisted weight-gradient GEMMs ([N, lg] hi / lo planes): written from the staging
  // tile with 8 lanes per 16-byte run (4 cache lines per warp store; one 2-byte store per lane-row touched 32)
  auto store_dg = [&](int64_t row0s) {
    for (int idx = tid; idx < 2048; idx += kSplitThreads) {
      const int pl = idx >> 10, g = (idx >> 8) & 3, r = (idx >> 3) & 31, e = idx & 7;
      if (r < rows && k0 + e < H)
        dgb[(pl ? a.dgb_lo_off : 0) + (row0s + r) * a.lg + int64_t(g) * H + k0 + e] = stg_s[pl][g][r][e];
    }
  };
  if (upper) prefetch(a.T1 - 1); else asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  float bs_i = 0.f, bs_f = 0.f, bs_g = 0.f, bs_o = 0.f;
  const int last_s = a.T1 + 1;
  unsigned* const my_flag = a.flags + blockIdx.x * kFlagStride;
  const unsigned* const role_flags = a.flags + (upper ? 0 : a.nc) * kFlagStride;
  int it = 0;  // this role's active-step counter
  bool fetched = false;   // a tile fetch has run (the ring's empty barriers have completed phases)
  for (int s = 0; s <= last_s; ++s) {
    const int t = time_of(s);
    const bool active = (t >= 0 && t < a.T1);
    const int64_t row0 = int64_t(active ? t : 0) * B;
    __nv_bfloat16* dgq_t = dgq + int64_t(it & 1) * 4 * gs;
    float p_i = 0.f, p_f = 0.f, p_g = 0.f, p_o = 0.f;
    if (active) {
      if (actA) {   // (the prefetched operands were waited for, and made visible by the barrier, at the end of the previous step)
        const int gb = (q >> 2) * 512 + lane * 16 + (q & 3), cb = (q >> 2) * 128 + lane * 4 + (q & 3);
        const float ig = pre_s[gb], fg = pre_s[gb + 4], gg = pre_s[gb + 8], og = pre_s[gb + 12];
        const float n_nd = pre_s[1792 + lane];
        const float n_cs = pre_s[1024 + cb], n_cm = pre_s[1280 + cb] * n_nd;   // c_{t-1} * notdone_t
        const float n_ndn = (t + 1 < a.T1) ? pre_s[1824 + lane] : 0.f;
        float dh = upper ? pre_s[1536 + lane * 8 + q] : n_dy;
        float dc = 0.0f;
        if (it > 0) {
          dh += dh_s[q][lane] * n_ndn;
          dc = dc_s[q][lane];
        }
        const float tc = tanhf(n_cs);
        const float d_o = dh * tc;
        dc += dh * og * (1.0f - tc * tc);
        const float d_i = dc * gg, d_f = dc * n_cm, d_g = dc * ig;
        p_i = d_i * ig * (1.0f - ig); p_f = d_f * fg * (1.0f - fg);
        p_g = d_g * (1.0f - gg * gg); p_o = d_o * og * (1.0f - og);
        dc_s[q][lane] = dc * fg * n_nd;
        bs_i += p_i; bs_f += p_f; bs_g += p_g; bs_o += p_o;
      }
      // publish this CTA's 8 columns of the four gate-gradient tiles, hi and lo planes (16-byte stores staged through smem)
      if (wrp < kBwdCols) {
        const float p[4] = {p_i, p_f, p_g, p_o};
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const __nv_bfloat16 h = __float2bfloat16_rn(p[g]);
          stg_s[0][g][lane][q] = h;
          stg_s[1][g][lane][q] = __float2bfloat16_rn(p[g] - __bfloat162float(h));
        }
      }
      __syncthreads();
      if (tid < 256 && (tid & 31) < rows && !idle) {
        const int pl = tid >> 7, g = (tid >> 5) & 3, bb = tid & 31;
        *reinterpret_cast<uint4*>(dgq_t + (pl ? a.dgq_lo_off : 0) + int64_t(g) * gs + int64_t(bb) * Hq + k0) =
            *reinterpret_cast<const uint4*>(&stg_s[pl][g][bb][0]);
        fence_proxy_async_global();   // consumers read the tiles through TMA
      }
    }
    if (s == last_s) {
      if (active) { __syncthreads(); store_dg(row0); }
      break;
    }
    __syncthreads();
    if (tid == 0) {  // this CTA's tile columns of wave step s (and, upper role, its dxm of step s-1) are out
      asm volatile("fence.acq_rel.gpu;" ::: "memory");
      st_relaxed_u32(my_flag, unsigned(s + 1));
    }
    if (active) store_dg(row0);
    prefetch(time_of(s + 1));  // forward-pass operands only: overlaps the wait
    // hand-off: this warp needs the tile columns of units [16*ks0, 16*ks0 + 48) -> the 6 CTAs of its own role that own
    // them; the pointwise threads of the lower role additionally need the upper CTA with the same 8 columns (its dxm)
    {
      const int p0 = (ks0 * 16) / kBwdCols + lane;
      const int pend = (min((ks0 + kSplitK) * 16, H) + kBwdCols - 1) / kBwdCols;
      if (lane < 6 && p0 < pend && p0 < int(a.ncol)) {
        while (ld_relaxed_u32(role_flags + p0 * kFlagStride) < unsigned(s + 1)) {}
        (void)ld_acquire_u32(role_flags + p0 * kFlagStride);
        fence_proxy_async_global();
      } else if (!upper && lane == 8 && wrp < kBwdCols) {
        while (ld_relaxed_u32(a.flags + cidx * kFlagStride) < unsigned(s + 1)) {}
        (void)ld_acquire_u32(a.flags + cidx * kFlagStride);
      }
      __syncwarp();
    }
    fetch_dxm(time_of(s + 1));  // written by the upper role before it published wave step s
    const bool need_rec = active && t > 0;
    const bool need_dx = active && upper;
    if (need_rec || need_dx) {
      // Ring slot g & 1 holds gate g: its full and empty barriers complete twice per fetching step (gates g & 1 and
      // (g & 1) + 2), so the phase parity of gate g is g >> 1 on the full barrier; before gate g is loaded, the empty
      // barrier's previous phase (gate g - 2, or gate g + 2 of the previous fetching step) must have completed.
      auto issue = [&](int g) {   // lane 0: this CTA's row half of this warp's columns of gate g, both planes
        if (g >= 2 || fetched) mbar_wait_cluster(&empty_s[wrp][g & 1], g >= 2 ? 0u : 1u);
        fence_proxy_async_global();
        mbar_expect_tx(&full_s[wrp][g & 1], kSlotBytes);
        tma_multicast_5d(X + ((g & 1) * 2 + rank) * kHalfE, dgq_map, &full_s[wrp][g & 1], ks0 * 16, 16 * int(rank), g, it & 1, 0);
      };
      float acc0[2][4], acc1[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) { acc0[mt][e] = 0.f; acc1[mt][e] = 0.f; }
      if (lane == 0) { issue(0); issue(1); }
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        mbar_wait(&full_s[wrp][g & 1], uint32_t(g >> 1));
        const __nv_bfloat16* Xg = X + (g & 1) * 2 * kHalfE;
#pragma unroll
        for (int sk = 0; sk < kSplitK; ++sk) {
          if (ks0 + sk < kpg) {
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {   // m16 tile mt = the row half CTA rank mt loaded
              uint32_t ah[4], al[4];
              const int off = mt * kHalfE + (lane & 15) * kTileRowE + sk * 16 + (lane >> 4) * 8;
              ldmatrix_x4(ah, Xg + off);
              ldmatrix_x4(al, Xg + 16 * kTileRowE + off);
              if (need_rec) mma3(acc0[mt], ah, al, bh[g][sk][0], bh[g][sk][1], bl[g][sk][0], bl[g][sk][1]);
              if (need_dx) mma3(acc1[mt], ah, al, ih[g][sk][0], ih[g][sk][1], il[g][sk][0], il[g][sk][1]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) {   // slot read: free it for both loaders
          mbar_arrive_local(&empty_s[wrp][g & 1]);
          mbar_arrive_remote((g & 1) ? peer_empty1 : peer_empty0);
          if (g + 2 < 4) issue(g + 2);
        }
      }
      fetched = true;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r = mt * 16 + (lane >> 2), c = (lane & 3) * 2;
        part[wrp][0][c][r] = acc0[mt][0]; part[wrp][0][c + 1][r] = acc0[mt][1];
        part[wrp][0][c][r + 8] = acc0[mt][2]; part[wrp][0][c + 1][r + 8] = acc0[mt][3];
        part[wrp][1][c][r] = acc1[mt][0]; part[wrp][1][c + 1][r] = acc1[mt][1];
        part[wrp][1][c][r + 8] = acc1[mt][2]; part[wrp][1][c + 1][r + 8] = acc1[mt][3];
      }
      __syncthreads();
      if (wrp < kBwdCols) {            // warps 0..7: recurrent carry for time t-1 (fixed summation order)
        if (need_rec) {
          float d = 0.f;
#pragma unroll
          for (int w = 0; w < kSplitWarps; ++w) d += part[w][0][wrp][lane];
          dh_s[wrp][lane] = d;
        }
        if (need_dx) {                 // dL/dh_lower[t], this CTA's 8 columns
          float d = 0.f;
#pragma unroll
          for (int w = 0; w < kSplitWarps; ++w) d += part[w][1][wrp][lane];
          if (lane < rows && !idle) a.dxb[(int64_t(t) * a.ncol + cidx) * 256 + lane * 8 + wrp] = d;
        }
      }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");   // next step's prefetched pointwise operands (all threads' copies)
    __syncthreads();
    if (active) ++it;
  }
  if (wrp < kBwdCols) {
    bs_i = warp_sum(bs_i); bs_f = warp_sum(bs_f); bs_g = warp_sum(bs_g); bs_o = warp_sum(bs_o);
    float* db = upper ? a.db_up : a.db_lo;
    if (lane == 0 && k0 + q < H) {
      db[k0 + q] = bs_i; db[H + k0 + q] = bs_f; db[2 * H + k0 + q] = bs_g; db[3 * H + k0 + q] = bs_o;
    }
  }
  cluster_sync_all();   // no CTA exits with multicast writes or remote arrives into it still in flight
}

static size_t g_fwd_mma_attr_dev[64] = {0}, g_bwd_mma_attr_dev[64] = {0};

// one decision for a (B, H) pair, used identically by forward and backward (the backward consumes the bf16
// masked-h buffer only the tensor-core forward writes)
static bool mma_recurrence_applicable(int64_t B, int H) {
  if (B > 32 || H > 624) return false;  // tile copy: <= 5 x 16 B chunks per thread
  const int Hq = mma_hq(H);
  dim3 grid((H + kStepUnits - 1) / kStepUnits, 1), gridb((H + kBwdCols - 1) / kBwdCols, 1);
  return coop_fit(lstm_fwd_persistent_mma_kernel, grid, size_t(32) * Hq * 2, kStepThreads, per_device(g_fwd_mma_attr_dev)) &&
         coop_fit(lstm_bwd_persistent_mma_kernel, gridb, size_t(4) * 32 * Hq * 2, kStepThreads, per_device(g_bwd_mma_attr_dev));
}

static int lstm_fwd_persistent_mma(const LstmLayerWs& L, const float* w_hh, float* hs, const float* notdone, int64_t T1,
                                   int64_t B, int H, unsigned* counter, cudaStream_t st) {
  const int Hq = mma_hq(H);
  const size_t smem = size_t(32) * Hq * 2;
  dim3 grid((H + kStepUnits - 1) / kStepUnits, 1);
  if (!coop_fit(lstm_fwd_persistent_mma_kernel, grid, smem, kStepThreads, per_device(g_fwd_mma_attr_dev))) return -1;
  cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned), st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  PersistFwdMmaArgs a;
  a.w_hh = w_hh; a.gates = L.gates; a.hs = hs; a.cs = L.cs; a.cm = L.cm; a.nd = notdone;
  a.hmq = static_cast<__nv_bfloat16*>(L.hmq); a.counter = counter;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hq = Hq; a.nctas = grid.x;
  void* args[] = {&a};
  e = cudaLaunchCooperativeKernel((const void*)lstm_fwd_persistent_mma_kernel, grid, dim3(kStepThreads), args, smem, st);
  TB_REQUIRE(e == cudaSuccess, "lstm_fwd_persistent_mma_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm_fwd_persistent_mma_kernel");
}

static size_t g_fwd_wave_attr_dev[64] = {0};
static size_t wave_fwd_smem(int Hq) { return size_t(2) * 32 * Hq * 2 + sizeof(float) * 16 * 2 * 16 * 33; }
static bool wave_fwd_applicable(int64_t B, int H) {
  if (!mma_recurrence_applicable(B, H)) return false;
  if (((H + 15) / 16 + 15) / 16 > kWaveK) return false;
  dim3 grid((H + kStepUnits - 1) / kStepUnits, 1);
  return coop_fit(lstm2_fwd_wave_mma_kernel, grid, wave_fwd_smem(mma_hq(H)), kStepThreads, per_device(g_fwd_wave_attr_dev));
}

static int lstm2_fwd_wave(LstmWs& ws, const LstmParams& p, float* y, const float* notdone, int64_t T1, int64_t B, int H,
                          cudaStream_t st) {
  const int Hq = mma_hq(H);
  const size_t smem = wave_fwd_smem(Hq);
  dim3 grid((H + kStepUnits - 1) / kStepUnits, 1);
  cudaError_t e = cudaMemsetAsync(ws.sync, 0, sizeof(unsigned), st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  WaveFwdArgs a;
  a.w_hh0 = p.w_hh[0]; a.w_ih1 = p.w_ih[1]; a.w_hh1 = p.w_hh[1]; a.bias1 = ws.layer[1].bsum;
  for (int l = 0; l < 2; ++l) {
    const LstmLayerWs& L = ws.layer[l];
    a.gates[l] = L.gates; a.hs[l] = (l == 1) ? y : L.hs; a.cs[l] = L.cs; a.cm[l] = L.cm;
    a.hq[l] = static_cast<__nv_bfloat16*>(L.hq); a.hmq[l] = static_cast<__nv_bfloat16*>(L.hmq);
  }
  a.nd = notdone; a.counter = ws.sync;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hq = Hq; a.nctas = grid.x;
  void* args[] = {&a};
  e = cudaLaunchCooperativeKernel((const void*)lstm2_fwd_wave_mma_kernel, grid, dim3(kStepThreads), args, smem, st);
  TB_REQUIRE(e == cudaSuccess, "lstm2_fwd_wave_mma_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm2_fwd_wave_mma_kernel");
}

// slot 0 of the split recurrence's planes: hq = split(h0) (raw), hmq = split(h0 * nd_0); row padding zero
__global__ void lstm_init_state_split_kernel(const float* __restrict__ h0, const float* __restrict__ nd,
                                             __nv_bfloat16* __restrict__ hq, int64_t hq_lo, __nv_bfloat16* __restrict__ hmq,
                                             int64_t hmq_lo, int B, int H, int Hq) {
  const int64_t total = int64_t(B) * Hq;
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = int(i / Hq), k = int(i % Hq);
  const float h = k < H ? h0[int64_t(b) * H + k] : 0.f;
  const float hm = h * nd[b];
  const __nv_bfloat16 a = __float2bfloat16_rn(h), m = __float2bfloat16_rn(hm);
  hq[i] = a; hq[hq_lo + i] = __float2bfloat16_rn(h - __bfloat162float(a));
  hmq[i] = m; hmq[hmq_lo + i] = __float2bfloat16_rn(hm - __bfloat162float(m));
}

// The split kernels run as one cooperative grid of 2-CTA clusters: launch configuration with both attributes
struct ClusterCoopLaunch {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[2];
  ClusterCoopLaunch(dim3 grid, size_t smem, cudaStream_t st) {
    cfg.gridDim = grid; cfg.blockDim = dim3(kSplitThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeCooperative; attr[1].val.cooperative = 1;
    cfg.attrs = attr; cfg.numAttrs = 2;
  }
};
// coop_fit for a grid of 2-CTA clusters: every cluster of the grid must be co-resident (the kernels spin on flags
// written by other CTAs)
template <typename Kernel>
static int cluster_coop_fit(Kernel kernel, dim3 grid, size_t smem, size_t* attr_smem) {
  int dev = 0, coop = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  if (!coop) return 0;
  if (*attr_smem < smem) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) {
      cudaGetLastError();
      return 0;
    }
    *attr_smem = smem;
  }
  ClusterCoopLaunch l(grid, smem, nullptr);
  int clusters = 0;
  if (cudaOccupancyMaxActiveClusters(&clusters, kernel, &l.cfg) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return int64_t(clusters) * 2 >= int64_t(grid.x);
}

static size_t g_fwd_split_attr_dev[64] = {0};
static size_t wave_fwd_split_smem() {   // tiles + partial sums + alignment slack
  return size_t(kSplitWarps) * 2 * kSlotBytes + sizeof(float) * kSplitWarps * 2 * 16 * 33 + 128;
}
// forward CTAs: kStepUnits units each, padded to whole clusters
static dim3 wave_fwd_split_grid(int H) { return dim3(((H + kStepUnits - 1) / kStepUnits + 1) & ~1, 1); }
// precision 2, two layers: the split-bf16 wavefront kernel (other shapes run the exact-fp32 recurrence kernels)
static bool wave_fwd_split_applicable(int64_t B, int In, int H) {
  if (B > 32 || In != H || (H + 15) / 16 > kSplitWarps * kSplitK) return false;
  const dim3 grid = wave_fwd_split_grid(H);
  if (int(grid.x) > kSplitThreads || grid.x > 512) return false;
  return cluster_coop_fit(lstm2_fwd_wave_split_kernel, grid, wave_fwd_split_smem(), per_device(g_fwd_split_attr_dev));
}

static int lstm2_fwd_wave_split(LstmWs& ws, const LstmParams& p, float* y, const float* notdone, const float* c0, float* hN,
                                float* cN, int64_t T1, int64_t B, int H, cudaStream_t st) {
  const int Hq = mma_hq(H);
  const dim3 grid = wave_fwd_split_grid(H);
  cudaError_t e = cudaMemsetAsync(ws.flags, 0, sizeof(unsigned) * 512 * kFlagStride, st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  WaveFwdSplitArgs a;
  a.w_hh0 = p.w_hh[0]; a.w_ih1 = p.w_ih[1]; a.w_hh1 = p.w_hh[1]; a.bias1 = ws.layer[1].bsum; a.c0 = c0;
  a.xproj = ws.layer[0].gates; a.y = y; a.hN = hN; a.cN = cN;
  for (int l = 0; l < 2; ++l) {
    const LstmLayerWs& L = ws.layer[l];
    a.gact[l] = L.gact; a.csb[l] = L.csb;
    TB_REQUIRE(L.gact && L.csb, "lstm: blocked save buffers missing");
    a.hq[l] = static_cast<__nv_bfloat16*>(L.hq); a.hmq[l] = static_cast<__nv_bfloat16*>(L.hmq);
  }
  a.hq_lo = ws.layer[0].hq_lo; a.hmq_lo = ws.layer[0].hmq_lo;
  TB_REQUIRE(ws.layer[1].hq_lo == a.hq_lo && ws.layer[1].hmq_lo == a.hmq_lo && a.hq_lo > 0, "lstm: split planes missing");
  a.nd = notdone; a.flags = ws.flags;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hq = Hq; a.nctas = unsigned((H + kStepUnits - 1) / kStepUnits);
  CUtensorMap maps[2];
  for (int l = 0; l < 2; ++l) {
    const uint64_t dims[4] = {uint64_t(Hq), uint64_t(B), uint64_t(T1 + 1), 2};
    const uint64_t strides[3] = {uint64_t(Hq) * 2, uint64_t(B) * Hq * 2, uint64_t(a.hq_lo) * 2};
    const uint32_t box[4] = {kTileRowE, 16, 1, 2};
    tcd::make_map_nd(&maps[l], a.hq[l], 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  ClusterCoopLaunch l(grid, wave_fwd_split_smem(), st);
  e = cudaLaunchKernelEx(&l.cfg, lstm2_fwd_wave_split_kernel, maps[0], maps[1], a);
  TB_REQUIRE(e == cudaSuccess, "lstm2_fwd_wave_split_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm2_fwd_wave_split_kernel");
}

// =========================================================================================
// Single-layer recurrence on ONE thread-block cluster (precision 2, H = 256: the IMPALA ResNet's LSTM).
// The cooperative kernels above pay a grid-wide barrier through L2 per step although a [B, 256] x [256, 1024]
// product is a small fraction of that in tensor-core time.  Here the 16 CTAs of one cluster own 16 hidden units x 4 gates each (64 gate
// rows of W_hh as hi / lo mma.sync B fragments in registers for all steps), h is exchanged through DISTRIBUTED SHARED
// MEMORY (every CTA stores its 16 units of h_t - bf16 hi / lo - into the A tile of all 16 CTAs) and the step barrier is the
// hardware cluster barrier.  Warp w multiplies k16 steps {2w, 2w+1} for all 8 n8 tiles (A is read once per CTA), partial
// sums meet in shared memory; thread (row, unit) finishes the four gates, keeps c in a register.
// Same buffers as lstm_fwd_persistent_kernel: gates (pre-activations in, activated out), hs, cs, cm / hm rows t+1.
// =========================================================================================
namespace cg = cooperative_groups;
constexpr int kClN = 16;            // CTAs per cluster
constexpr int kClH = 256;
constexpr int kClU = kClH / kClN;   // hidden units per CTA
constexpr int kClHq = kClH + 8;     // A tile row pitch (bf16): 528 B, conflict-free ldmatrix
constexpr int kClThreads = 256;

struct ClusterFwdArgs {
  const float* w_hh; float* gates; float* hs; float* cs; float* hm; float* cm; const float* nd;
  int T1, B, Hp;
};

template <int MT>   // m16 tiles of batch rows (B <= 16*MT)
__global__ void __launch_bounds__(kClThreads, 1) lstm_fwd_cluster_kernel(ClusterFwdArgs a) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = int(cluster.block_rank());
  constexpr int R = MT * 16;
  extern __shared__ __align__(128) unsigned char cl_smem[];
  typedef __nv_bfloat16 ATile[2][R][kClHq];                        // [hi / lo][row][k]
  ATile* A_s = reinterpret_cast<ATile*>(cl_smem);                  // [2 buffers]
  typedef float PartT[R][65];                                      // [row][gate*16 + unit]
  PartT* part = reinterpret_cast<PartT*>(cl_smem + 2 * sizeof(ATile));   // [8 warps]
  typedef __nv_bfloat16 StageT[R][kClU];                           // this CTA's h_t as hi / lo, before the broadcast
  StageT* stage = reinterpret_cast<StageT*>(cl_smem + 2 * sizeof(ATile) + 8 * sizeof(PartT));
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int B = a.B, H = kClH;
  // B fragments: n tile nt = local gate rows [8 nt, 8 nt + 8), local row lr = gate*16 + unit -> W_hh row gate*H + 16*rank + unit
  uint32_t bh[2][8][2], bl[2][8][2];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int lr = nt * 8 + (lane >> 2);
      const float* wr = a.w_hh + (int64_t(lr >> 4) * H + rank * kClU + (lr & 15)) * H;
      const int k = (2 * wrp + ks) * 16 + (lane & 3) * 2;
      split_pack(wr[k], wr[k + 1], bh[ks][nt][0], bl[ks][nt][0]);
      split_pack(wr[k + 8], wr[k + 9], bh[ks][nt][1], bl[ks][nt][1]);
    }
  // initial masked state: every CTA loads the whole h tile (rows >= B are zero)
  for (int i = tid; i < R * H; i += kClThreads) {
    const int r = i / H, k = i - r * H;
    const float v = r < B ? a.hm[int64_t(r) * a.Hp + k] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    A_s[0][0][r][k] = h;
    A_s[0][1][r][k] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
  // pointwise role: RP rows per thread, unit u
  constexpr int RP = R / 16;
  const int u = tid & 15, r0 = tid >> 4;
  const int ug = rank * kClU + u;
  float c_prev[RP];
#pragma unroll
  for (int q = 0; q < RP; ++q) { const int r = r0 + 16 * q; c_prev[q] = r < B ? a.cm[int64_t(r) * H + ug] : 0.f; }
  // inputs of the pointwise phase that do not depend on the recurrence (input projection, next step's notdone) are loaded one
  // step ahead, right before the cluster barrier, so their L2 / HBM latency hides behind it
  float pre[RP][4], ndn[RP];
  auto load_inputs = [&](int t) {
#pragma unroll
    for (int q = 0; q < RP; ++q) {
      const int r = r0 + 16 * q;
      ndn[q] = (r < B && t + 1 < a.T1) ? __ldg(a.nd + int64_t(t + 1) * B + r) : 0.f;
#pragma unroll
      for (int g = 0; g < 4; ++g) pre[q][g] = (r < B && t < a.T1) ? __ldcg(a.gates + (int64_t(t) * B + r) * 4 * H + g * H + ug) : 0.f;
    }
  };
  load_inputs(0);
  cluster.sync();
  for (int t = 0; t < a.T1; ++t) {
    const int cur = t & 1;
    const bool last = (t == a.T1 - 1);
    float acc[MT][8][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        uint32_t ah[4], al[4];
        const __nv_bfloat16* ap = &A_s[cur][0][mt * 16 + (lane & 15)][(2 * wrp + ks) * 16 + (lane >> 4) * 8];
        ldmatrix_x4(ah, ap);
        ldmatrix_x4(al, ap + R * kClHq);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) mma3(acc[mt][nt], ah, al, bh[ks][nt][0], bh[ks][nt][1], bl[ks][nt][0], bl[ks][nt][1]);
      }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int r = mt * 16 + (lane >> 2), c = nt * 8 + (lane & 3) * 2;
        part[wrp][r][c] = acc[mt][nt][0]; part[wrp][r][c + 1] = acc[mt][nt][1];
        part[wrp][r + 8][c] = acc[mt][nt][2]; part[wrp][r + 8][c + 1] = acc[mt][nt][3];
      }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < RP; ++q) {
      const int r = r0 + 16 * q;
      float gv[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float d = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) d += part[w][r][g * 16 + u];   // fixed order
        const float x = pre[q][g] + d;
        gv[g] = (g == 2) ? tanhf(x) : sigmoidf_(x);
      }
      const float c_new = gv[1] * c_prev[q] + gv[0] * gv[2];
      const float h_new = gv[3] * tanhf(c_new);
      const float hm_next = h_new * ndn[q];
      c_prev[q] = c_new * ndn[q];
      const __nv_bfloat16 hh = __float2bfloat16_rn(hm_next);
      stage[0][r][u] = hh;
      stage[1][r][u] = __float2bfloat16_rn(hm_next - __bfloat162float(hh));
      if (r < B) {   // saved for the backward pass / the weight-gradient GEMMs: off the critical path
        const int64_t row = int64_t(t) * B + r;
#pragma unroll
        for (int g = 0; g < 4; ++g) a.gates[row * 4 * H + g * H + ug] = gv[g];
        a.cs[row * H + ug] = c_new;
        a.hs[row * H + ug] = h_new;
        if (!last) {
          a.cm[(row + B) * H + ug] = c_prev[q];
          a.hm[(row + B) * a.Hp + ug] = hm_next;
        }
      }
    }
    __syncthreads();
    if (!last) {
      // broadcast this CTA's 16 units (32 B per row and plane) into the next A tile of every CTA: thread (row, d) serves CTA d
#pragma unroll
      for (int q = 0; q < RP; ++q) {
        const int r = r0 + 16 * q;
        __nv_bfloat16* dst0 = cluster.map_shared_rank(&A_s[cur ^ 1][0][r][rank * kClU], u);
        __nv_bfloat16* dst1 = cluster.map_shared_rank(&A_s[cur ^ 1][1][r][rank * kClU], u);
        const uint4* s0 = reinterpret_cast<const uint4*>(&stage[0][r][0]);
        const uint4* s1 = reinterpret_cast<const uint4*>(&stage[1][r][0]);
        reinterpret_cast<uint4*>(dst0)[0] = s0[0]; reinterpret_cast<uint4*>(dst0)[1] = s0[1];
        reinterpret_cast<uint4*>(dst1)[0] = s1[0]; reinterpret_cast<uint4*>(dst1)[1] = s1[1];
      }
    }
    load_inputs(t + 1);
    cluster.sync();   // release / acquire at cluster scope: every CTA's tile of step t+1 is complete and visible
  }
}

static size_t cluster_fwd_smem(int MT) {
  const size_t R = size_t(MT) * 16;
  return 2 * (2 * R * kClHq * 2) + 8 * (R * 65 * 4) + 2 * R * kClU * 2;
}

static int lstm_fwd_cluster(const LstmLayerWs& L, const float* w_hh, float* hs, const float* notdone, int64_t T1, int64_t B, int H,
                            cudaStream_t st) {
  if (H != kClH || B > 32 || B < 1) return -1;
  static int attr_ok[64] = {0};   // per device: 0 unknown, 1 ok, -1 unavailable
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr_ok[dev & 63] == 0) {
    cudaError_t e1 = cudaFuncSetAttribute(lstm_fwd_cluster_kernel<1>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaError_t e2 = cudaFuncSetAttribute(lstm_fwd_cluster_kernel<2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e1 == cudaSuccess) e1 = cudaFuncSetAttribute(lstm_fwd_cluster_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(cluster_fwd_smem(1)));
    if (e2 == cudaSuccess) e2 = cudaFuncSetAttribute(lstm_fwd_cluster_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(cluster_fwd_smem(2)));
    attr_ok[dev & 63] = (e1 == cudaSuccess && e2 == cudaSuccess) ? 1 : -1;
    if (attr_ok[dev & 63] < 0) cudaGetLastError();
  }
  if (attr_ok[dev & 63] < 0) return -1;
  ClusterFwdArgs a;
  a.w_hh = w_hh; a.gates = L.gates; a.hs = hs; a.cs = L.cs; a.hm = L.hm; a.cm = L.cm; a.nd = notdone;
  a.T1 = int(T1); a.B = int(B); a.Hp = padded_h(H);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kClN);
  cfg.blockDim = dim3(kClThreads);
  cfg.dynamicSmemBytes = cluster_fwd_smem(B <= 16 ? 1 : 2);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kClN; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = (B <= 16) ? cudaLaunchKernelEx(&cfg, lstm_fwd_cluster_kernel<1>, a) : cudaLaunchKernelEx(&cfg, lstm_fwd_cluster_kernel<2>, a);
  if (e != cudaSuccess) {   // a 16-CTA cluster cannot be placed here: the cooperative kernel takes over
    cudaGetLastError();
    return -1;
  }
  return check_launch("lstm_fwd_cluster_kernel");
}

// ---- backward on the same cluster ---------------------------------------------------------------------------------
// dL/dh_t needs dgates_{t+1} . W_hh over ALL 1024 gate rows.  Broadcasting the gate gradients (64 KB per CTA and step) would sit
// on the DSMEM links; instead every CTA multiplies ITS 64 gate gradients (local, bf16 hi / lo
// in shared memory) with ITS 64 rows of W_hh (B fragments in registers) into a partial dh[rows, 256], and the partials are
// reduce-scattered: the 16 columns of destination CTA d go into slot [source] of d's receive buffer (16 KB per CTA and
// step), summed by d in source order (deterministic) at the start of the next step.  Buffers as lstm_bwd_persistent_kernel:
// reads dy / gates (activated) / cs / cm / nd, writes dgates [N, 4H] fp32 for the weight-gradient GEMMs.
struct ClusterBwdArgs {
  const float* w_hh; const float* dy; const float* nd; const float* gates; const float* cs; const float* cm; float* dgates;
  int T1, B;
};

template <int MT>
__global__ void __launch_bounds__(kClThreads, 1) lstm_bwd_cluster_kernel(ClusterBwdArgs a) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = int(cluster.block_rank());
  constexpr int R = MT * 16, PQ = 64 + 8;
  extern __shared__ __align__(128) unsigned char cl_smem[];
  typedef __nv_bfloat16 PTile[R][PQ];                              // gate gradients of this CTA [row][gate*16 + unit]
  PTile* P_s = reinterpret_cast<PTile*>(cl_smem);                  // [hi / lo]
  typedef float RecvT[kClN][R][kClU];                              // [source CTA][row][unit]
  RecvT* recv = reinterpret_cast<RecvT*>(cl_smem + 2 * sizeof(PTile));   // [2 buffers]
  const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
  const int B = a.B, H = kClH;
  // B fragments: reduction index = local gate row lg (k16 steps 0..3), n = output column (hidden unit) 32*wrp + 8*ntl + lane/4
  uint32_t bh[4][4][2], bl[4][4][2];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int ntl = 0; ntl < 4; ++ntl) {
      const int n = wrp * 32 + ntl * 8 + (lane >> 2);
      const int lg = ks * 16 + (lane & 3) * 2;
      auto wv = [&](int l) { return a.w_hh[(int64_t(l >> 4) * H + rank * kClU + (l & 15)) * H + n]; };
      split_pack(wv(lg), wv(lg + 1), bh[ks][ntl][0], bl[ks][ntl][0]);
      split_pack(wv(lg + 8), wv(lg + 9), bh[ks][ntl][1], bl[ks][ntl][1]);
    }
  constexpr int RP = R / 16;
  const int u = tid & 15, r0 = tid >> 4;
  const int ug = rank * kClU + u;
  float dc_carry[RP];
#pragma unroll
  for (int q = 0; q < RP; ++q) dc_carry[q] = 0.f;
  // per-step inputs, loaded one step ahead (before the cluster barrier)
  float in_dy[RP], in_g[RP][4], in_cs[RP], in_cm[RP], in_nd[RP], in_ndn[RP];
  auto load_inputs = [&](int t) {
#pragma unroll
    for (int q = 0; q < RP; ++q) {
      const int r = r0 + 16 * q;
      const bool ok = r < B && t >= 0;
      const int64_t row = int64_t(t) * B + r;
      in_dy[q] = ok ? __ldg(a.dy + row * H + ug) : 0.f;
      in_cs[q] = ok ? __ldg(a.cs + row * H + ug) : 0.f;
      in_cm[q] = ok ? __ldg(a.cm + row * H + ug) : 0.f;
      in_nd[q] = ok ? __ldg(a.nd + row) : 0.f;
      in_ndn[q] = (ok && t + 1 < a.T1) ? __ldg(a.nd + row + B) : 0.f;
#pragma unroll
      for (int g = 0; g < 4; ++g) in_g[q][g] = ok ? __ldg(a.gates + row * 4 * H + g * H + ug) : 0.f;
    }
  };
  load_inputs(a.T1 - 1);
  cluster.sync();
  int buf = 0;
  for (int t = a.T1 - 1, it = 0; t >= 0; --t, ++it) {
#pragma unroll
    for (int q = 0; q < RP; ++q) {
      const int r = r0 + 16 * q;
      float dh = in_dy[q], dc = 0.f;
      if (it > 0) {
        float rec = 0.f;
#pragma unroll
        for (int sidx = 0; sidx < kClN; ++sidx) rec += recv[buf][sidx][r][u];   // fixed order
        dh += rec * in_ndn[q];
        dc = dc_carry[q];
      }
      const float ig = in_g[q][0], fg = in_g[q][1], gg = in_g[q][2], og = in_g[q][3];
      const float tc = tanhf(in_cs[q]);
      const float d_o = dh * tc;
      dc += dh * og * (1.0f - tc * tc);
      const float d_i = dc * gg, d_f = dc * in_cm[q], d_g = dc * ig;
      float pv[4];
      pv[0] = d_i * ig * (1.0f - ig); pv[1] = d_f * fg * (1.0f - fg);
      pv[2] = d_g * (1.0f - gg * gg); pv[3] = d_o * og * (1.0f - og);
      dc_carry[q] = dc * fg * in_nd[q];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const __nv_bfloat16 hh = __float2bfloat16_rn(pv[g]);
        P_s[0][r][g * 16 + u] = hh;
        P_s[1][r][g * 16 + u] = __float2bfloat16_rn(pv[g] - __bfloat162float(hh));
        if (r < B) a.dgates[(int64_t(t) * B + r) * 4 * H + g * H + ug] = pv[g];
      }
    }
    if (t == 0) break;   // uniform: no earlier step needs dh
    __syncthreads();
    float acc[MT][4][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int ntl = 0; ntl < 4; ++ntl)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][ntl][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        uint32_t ah[4], al[4];
        const __nv_bfloat16* ap = &P_s[0][mt * 16 + (lane & 15)][ks * 16 + (lane >> 4) * 8];
        ldmatrix_x4(ah, ap);
        ldmatrix_x4(al, ap + R * PQ);
#pragma unroll
        for (int ntl = 0; ntl < 4; ++ntl) mma3(acc[mt][ntl], ah, al, bh[ks][ntl][0], bh[ks][ntl][1], bl[ks][ntl][0], bl[ks][ntl][1]);
      }
    // reduce-scatter: this warp's 32 columns belong to CTAs 2*wrp (n tiles 0, 1) and 2*wrp + 1 (n tiles 2, 3)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int ntl = 0; ntl < 4; ++ntl) {
        const int dest = 2 * wrp + (ntl >> 1);
        const int col = (ntl & 1) * 8 + (lane & 3) * 2, row = mt * 16 + (lane >> 2);
        float* d0 = cluster.map_shared_rank(&recv[buf ^ 1][rank][row][col], dest);
        float* d1 = cluster.map_shared_rank(&recv[buf ^ 1][rank][row + 8][col], dest);
        *reinterpret_cast<float2*>(d0) = make_float2(acc[mt][ntl][0], acc[mt][ntl][1]);
        *reinterpret_cast<float2*>(d1) = make_float2(acc[mt][ntl][2], acc[mt][ntl][3]);
      }
    load_inputs(t - 1);
    cluster.sync();
    buf ^= 1;
  }
  cluster.sync();   // nobody leaves while a peer may still address its shared memory
}

static size_t cluster_bwd_smem(int MT) {
  const size_t R = size_t(MT) * 16;
  return 2 * (R * 72 * 2) + 2 * (size_t(kClN) * R * kClU * 4);
}

static int lstm_bwd_cluster(const LstmLayerWs& L, const float* w_hh, const float* dy, const float* notdone, int64_t T1, int64_t B,
                            int H, cudaStream_t st) {
  if (H != kClH || B > 32 || B < 1) return -1;
  static int attr_ok[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr_ok[dev & 63] == 0) {
    cudaError_t e1 = cudaFuncSetAttribute(lstm_bwd_cluster_kernel<1>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaError_t e2 = cudaFuncSetAttribute(lstm_bwd_cluster_kernel<2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e1 == cudaSuccess) e1 = cudaFuncSetAttribute(lstm_bwd_cluster_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(cluster_bwd_smem(1)));
    if (e2 == cudaSuccess) e2 = cudaFuncSetAttribute(lstm_bwd_cluster_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(cluster_bwd_smem(2)));
    attr_ok[dev & 63] = (e1 == cudaSuccess && e2 == cudaSuccess) ? 1 : -1;
    if (attr_ok[dev & 63] < 0) cudaGetLastError();
  }
  if (attr_ok[dev & 63] < 0) return -1;
  ClusterBwdArgs a;
  a.w_hh = w_hh; a.dy = dy; a.nd = notdone; a.gates = L.gates; a.cs = L.cs; a.cm = L.cm; a.dgates = L.dgates;
  a.T1 = int(T1); a.B = int(B);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kClN);
  cfg.blockDim = dim3(kClThreads);
  cfg.dynamicSmemBytes = cluster_bwd_smem(B <= 16 ? 1 : 2);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kClN; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = (B <= 16) ? cudaLaunchKernelEx(&cfg, lstm_bwd_cluster_kernel<1>, a) : cudaLaunchKernelEx(&cfg, lstm_bwd_cluster_kernel<2>, a);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return check_launch("lstm_bwd_cluster_kernel");
}

static int lstm_bwd_persistent_mma(const LstmLayerWs& L, const float* w_hh, const float* dy, const float* notdone,
                                   int64_t T1, int64_t B, int H, float* db, unsigned* counter, cudaStream_t st) {
  const int Hq = mma_hq(H);
  const size_t smem = size_t(4) * 32 * Hq * 2;
  dim3 grid((H + kBwdCols - 1) / kBwdCols, 1);
  if (!coop_fit(lstm_bwd_persistent_mma_kernel, grid, smem, kStepThreads, per_device(g_bwd_mma_attr_dev))) return -1;
  cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(L.dgq, 0, size_t(2) * 4 * B * Hq * 2, st);  // zero the row padding
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  PersistBwdMmaArgs a;
  a.w_hh = w_hh; a.dy = dy; a.nd = notdone; a.gates = L.gates; a.cs = L.cs; a.cm = L.cm;
  a.dgb = static_cast<__nv_bfloat16*>(L.dgb); a.lg = int(ld16(4 * H)); a.db = db;
  a.dgq = static_cast<__nv_bfloat16*>(L.dgq); a.counter = counter;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hq = Hq; a.nctas = grid.x;
  void* args[] = {&a};
  e = cudaLaunchCooperativeKernel((const void*)lstm_bwd_persistent_mma_kernel, grid, dim3(kStepThreads), args, smem, st);
  TB_REQUIRE(e == cudaSuccess, "lstm_bwd_persistent_mma_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm_bwd_persistent_mma_kernel");
}

static size_t g_bwd_wave_attr_dev[64] = {0};
static size_t wave_bwd_smem(int H) {
  const int kper = (4 * ((H + 15) / 16) + 15) / 16;
  return size_t(4) * 32 * mma_hq(H) * 2 + size_t(16) * kper * 32 * 8;
}
static bool wave_bwd_applicable(int64_t B, int H) {
  if (!mma_recurrence_applicable(B, H)) return false;
  dim3 grid(2 * ((H + kBwdCols - 1) / kBwdCols), 1);
  return coop_fit(lstm2_bwd_wave_mma_kernel, grid, wave_bwd_smem(H), kStepThreads, per_device(g_bwd_wave_attr_dev));
}

// both layers' backward recurrences in one launch; leaves dgb / bias gradients of both layers and
// ws.dx_mid = dL/d(lower layer output)
static int lstm2_bwd_wave(LstmWs& ws, const LstmParams& p, const LstmGrads& g, const float* dy, const float* notdone, int64_t T1,
                          int64_t B, int H, cudaStream_t st) {
  const int Hq = mma_hq(H);
  const unsigned nc = unsigned((H + kBwdCols - 1) / kBwdCols);
  const LstmLayerWs& U = ws.layer[1];
  const LstmLayerWs& L = ws.layer[0];
  unsigned* counter = ws.sync + 32;
  cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(U.dgq, 0, size_t(2) * 4 * B * Hq * 2, st);  // zero the row padding
  if (e == cudaSuccess) e = cudaMemsetAsync(L.dgq, 0, size_t(2) * 4 * B * Hq * 2, st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  WaveBwdArgs a;
  a.w_hh_up = p.w_hh[1]; a.w_hh_lo = p.w_hh[0]; a.w_ih_up = p.w_ih[1];
  a.dy = dy; a.nd = notdone;
  a.gates_up = U.gates; a.cs_up = U.cs; a.cm_up = U.cm;
  a.gates_lo = L.gates; a.cs_lo = L.cs; a.cm_lo = L.cm;
  a.dgb_up = static_cast<__nv_bfloat16*>(U.dgb); a.dgb_lo = static_cast<__nv_bfloat16*>(L.dgb); a.lg = int(ld16(4 * H));
  a.db_up = g.b_ih[1]; a.db_lo = g.b_ih[0];
  a.dgq_up = static_cast<__nv_bfloat16*>(U.dgq); a.dgq_lo = static_cast<__nv_bfloat16*>(L.dgq);
  a.dxm = ws.dx_mid; a.counter = counter;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hq = Hq; a.nc = nc;
  void* args[] = {&a};
  e = cudaLaunchCooperativeKernel((const void*)lstm2_bwd_wave_mma_kernel, dim3(2 * nc), dim3(kStepThreads), args,
                                  wave_bwd_smem(H), st);
  TB_REQUIRE(e == cudaSuccess, "lstm2_bwd_wave_mma_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm2_bwd_wave_mma_kernel");
}

static size_t g_bwd_split_attr_dev[64] = {0};
static size_t wave_bwd_split_smem() {   // tile rings + partial sums + prefetched pointwise operands + alignment slack
  return size_t(kSplitWarps) * 2 * kSlotBytes + sizeof(float) * kSplitWarps * 2 * kBwdCols * 33 + sizeof(float) * 9 * 256 + 128;
}
// CTAs per role: kBwdCols columns each, padded to whole clusters (a cluster never straddles the two roles)
static unsigned wave_bwd_split_role_ctas(int H) { return unsigned(((H + kBwdCols - 1) / kBwdCols + 1) & ~1); }
static bool wave_bwd_split_applicable(int64_t B, int In, int H) {
  if (!wave_fwd_split_applicable(B, In, H)) return false;  // consumes the planes the split forward leaves behind
  dim3 grid(2 * wave_bwd_split_role_ctas(H), 1);
  if (int(grid.x / 2) + 1 > kSplitThreads || grid.x > 512) return false;
  return cluster_coop_fit(lstm2_bwd_wave_split_kernel, grid, wave_bwd_split_smem(), per_device(g_bwd_split_attr_dev));
}

static int lstm2_bwd_wave_split(LstmWs& ws, const LstmParams& p, const LstmGrads& g, const float* dy, const float* notdone,
                                int64_t T1, int64_t B, int H, cudaStream_t st) {
  const int Hq = mma_hq(H);
  const unsigned nc = wave_bwd_split_role_ctas(H);
  const LstmLayerWs& U = ws.layer[1];
  const LstmLayerWs& L = ws.layer[0];
  unsigned* flags = ws.flags + 512 * kFlagStride;
  cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(unsigned) * 512 * kFlagStride, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(U.dgq, 0, size_t(U.dgq_lo + int64_t(2) * 4 * B * Hq) * 2, st);  // zero the row padding
  if (e == cudaSuccess) e = cudaMemsetAsync(L.dgq, 0, size_t(L.dgq_lo + int64_t(2) * 4 * B * Hq) * 2, st);
  TB_REQUIRE(e == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(e));
  TB_REQUIRE(U.dgq_lo > 0 && U.dgq_lo == L.dgq_lo && U.dgb_lo > 0 && U.dgb_lo == L.dgb_lo, "lstm: split planes missing");
  WaveBwdSplitArgs a;
  a.w_hh_up = p.w_hh[1]; a.w_hh_lo = p.w_hh[0]; a.w_ih_up = p.w_ih[1];
  a.dy = dy; a.nd = notdone;
  a.gact_up = U.gact; a.csb_up = U.csb; a.gact_lo = L.gact; a.csb_lo = L.csb; a.nfwd = (H + kStepUnits - 1) / kStepUnits;
  TB_REQUIRE(U.gact && U.csb && L.gact && L.csb && ws.dxb, "lstm: blocked save buffers missing");
  a.dgb_up = static_cast<__nv_bfloat16*>(U.dgb); a.dgb_lo = static_cast<__nv_bfloat16*>(L.dgb); a.lg = int(ld16(4 * H));
  a.dgb_lo_off = U.dgb_lo;
  a.db_up = g.b_ih[1]; a.db_lo = g.b_ih[0];
  a.dgq_up = static_cast<__nv_bfloat16*>(U.dgq); a.dgq_lo = static_cast<__nv_bfloat16*>(L.dgq); a.dgq_lo_off = U.dgq_lo;
  a.dxb = ws.dxb; a.flags = flags;
  a.T1 = int(T1); a.B = int(B); a.H = H; a.Hq = Hq; a.nc = nc; a.ncol = unsigned((H + kBwdCols - 1) / kBwdCols);
  CUtensorMap maps[2];
  for (int r = 0; r < 2; ++r) {
    const uint64_t dims[5] = {uint64_t(Hq), uint64_t(B), 4, 2, 2};
    const uint64_t strides[4] = {uint64_t(Hq) * 2, uint64_t(B) * Hq * 2, uint64_t(4) * B * Hq * 2, uint64_t(a.dgq_lo_off) * 2};
    const uint32_t box[5] = {kTileRowE, 16, 1, 1, 2};
    tcd::make_map_nd(&maps[r], r == 0 ? a.dgq_up : a.dgq_lo, 5, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  ClusterCoopLaunch l(dim3(2 * nc), wave_bwd_split_smem(), st);
  e = cudaLaunchKernelEx(&l.cfg, lstm2_bwd_wave_split_kernel, maps[0], maps[1], a);
  TB_REQUIRE(e == cudaSuccess, "lstm2_bwd_wave_split_kernel: %s", cudaGetErrorString(e));
  return check_launch("lstm2_bwd_wave_split_kernel");
}

// Side stream for work that can run beside a recurrence kernel (which occupies only H/8 = 65 of the 132 SMs):
// forked from / joined into the caller's stream with events, so it is captured into the learner's CUDA graph.
struct SideStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
};
// A caller-owned side stream (tb_set_aux_stream): data-parallel learners pass the stream they will enqueue the all-reduce of
// the LSTM gradient slice on, so that it is ordered behind the weight-gradient GEMMs forked onto it.
static thread_local cudaStream_t g_aux_stream = nullptr;

static SideStream* side_stream() {
  static thread_local SideStream per_dev[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  SideStream& s = per_dev[dev];
  if (g_aux_stream) {
    static thread_local SideStream aux[64];
    SideStream& x = aux[dev];
    x.stream = g_aux_stream;
    if (!x.fork && (cudaEventCreateWithFlags(&x.fork, cudaEventDisableTiming) != cudaSuccess ||
                    cudaEventCreateWithFlags(&x.join, cudaEventDisableTiming) != cudaSuccess)) {
      cudaGetLastError();
      return nullptr;
    }
    return &x;
  }
  if (!s.stream) {
    if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      s.stream = nullptr;
      return nullptr;
    }
  }
  return &s;
}

#define TB_TRY(expr)        \
  do {                      \
    int _rc = (expr);       \
    if (_rc) return _rc;    \
  } while (0)

int lstm_forward(const float* x, const float* notdone, const float* h0, const float* c0, const LstmParams& p,
                 int64_t T1, int64_t B, int In, int H, int layers, LstmWs& ws, float* y, float* hN, float* cN,
                 float* splitk, int precision, cudaStream_t st) {
  TB_REQUIRE(layers >= 1 && layers <= kLstmMaxLayers, "lstm: 1..%d layers", kLstmMaxLayers);
  const int64_t N = T1 * B;
  const float* xin = x;
  int in_dim = In;
  if (precision == 1 && layers == 2 && wave_fwd_applicable(B, H)) {
    // both layers in one wavefront kernel: only layer 0's input projection is hoisted
    const int Hq = mma_hq(H);
    for (int l = 0; l < 2; ++l) {
      LstmLayerWs& L = ws.layer[l];
      const int in_l = (l == 0) ? In : H;
      const int64_t l16 = ld16(in_l);
      add2_kernel<<<(4 * H + 255) / 256, 256, 0, st>>>(p.b_ih[l], p.b_hh[l], L.bsum, 4 * H);
      TB_TRY(check_launch("add2_kernel"));
      TB_TRY(pack_weights_bf16(p.w_ih[l], L.wihb, 4 * H, 1, in_l, l16, st));  // layer 1's is used by the backward
      if (l == 0) {
        TB_TRY(f32_to_bf16(x, L.xb, N, In, In, l16, st));
        TcEpilogue te; te.C = L.gates; te.ldc = 4 * H; te.bias = L.bsum; te.tag = "lstm_xproj_fwd";
        TB_TRY(gemm_tc_bf16(L.xb, L.wihb, N, 4 * H, In, l16, l16, te, st));
      }
      cudaError_t eq = cudaMemsetAsync(L.hmq, 0, size_t(N) * Hq * 2, st);
      if (eq == cudaSuccess) eq = cudaMemsetAsync(L.hq, 0, size_t(N + B) * Hq * 2, st);
      TB_REQUIRE(eq == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(eq));
      lstm_init_state_q_kernel<<<(unsigned)((B * Hq + 255) / 256), 256, 0, st>>>(
          h0 + int64_t(l) * B * H, c0 + int64_t(l) * B * H, notdone, static_cast<__nv_bfloat16*>(L.hmq), L.cm, int(B), H,
          Hq, static_cast<__nv_bfloat16*>(L.hq));
      TB_TRY(check_launch("lstm_init_state_q_kernel"));
    }
    {
      ProfScope prof("lstm_recurrence_fwd", st);
      TB_TRY(lstm2_fwd_wave(ws, p, y, notdone, T1, B, H, st));
    }
    TB_TRY(f32_to_bf16(ws.layer[0].hs, ws.layer[1].xb, N, H, H, ld16(H), st));  // layer 1's input, for its dW_ih GEMM
    for (int l = 0; l < 2; ++l) {
      const float* hs = (l == 1) ? y : ws.layer[0].hs;
      cudaError_t e = cudaMemcpyAsync(hN + int64_t(l) * B * H, hs + (T1 - 1) * B * H, sizeof(float) * B * H,
                                      cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(cN + int64_t(l) * B * H, ws.layer[l].cs + (T1 - 1) * B * H, sizeof(float) * B * H,
                            cudaMemcpyDeviceToDevice, st);
      TB_REQUIRE(e == cudaSuccess, "lstm: state copy: %s", cudaGetErrorString(e));
    }
    return 0;
  }
  // (forward and backward are decided together: the split backward consumes the blocked saves only the split forward writes)
  if (precision == 2 && layers == 2 && wave_bwd_split_applicable(B, In, H)) {
    // split-bf16 wavefront: layer 0's input projection is one split wgmma GEMM, everything sequential is ONE kernel
    const int Hq = mma_hq(H);
    for (int l = 0; l < 2; ++l) {
      LstmLayerWs& L = ws.layer[l];
      const int in_l = (l == 0) ? In : H;
      const int64_t l16 = ld16(in_l);
      add2_kernel<<<(4 * H + 255) / 256, 256, 0, st>>>(p.b_ih[l], p.b_hh[l], L.bsum, 4 * H);
      TB_TRY(check_launch("add2_kernel"));
      TB_TRY(pack_weights_bf16(p.w_ih[l], L.wihb, 4 * H, 1, in_l, l16, st, L.wihb_lo));  // layer 1's: backward (dx)
      if (l == 0) {
        TB_TRY(f32_to_bf16(x, L.xb, N, In, In, l16, st, L.xb_lo));
        TcEpilogue te; te.C = L.gates; te.ldc = 4 * H; te.bias = L.bsum; te.tag = "lstm_xproj_fwd";
        te.a_lo = L.xb_lo; te.b_lo = L.wihb_lo;
        TB_TRY(gemm_tc_bf16(L.xb, L.wihb, N, 4 * H, In, l16, l16, te, st));
      }
      // zero the row padding (columns [H, Hq)) of every slot of both planes; the kernels only write [0, 4*ceil(H/4))
      cudaError_t eq = cudaMemsetAsync(L.hmq, 0, size_t(L.hmq_lo + N * Hq) * 2, st);
      if (eq == cudaSuccess) eq = cudaMemsetAsync(L.hq, 0, size_t(L.hq_lo + (N + B) * Hq) * 2, st);
      TB_REQUIRE(eq == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(eq));
      lstm_init_state_split_kernel<<<(unsigned)((B * Hq + 255) / 256), 256, 0, st>>>(
          h0 + int64_t(l) * B * H, notdone, static_cast<__nv_bfloat16*>(L.hq), L.hq_lo, static_cast<__nv_bfloat16*>(L.hmq), L.hmq_lo,
          int(B), H, Hq);
      TB_TRY(check_launch("lstm_init_state_split_kernel"));
    }
    {
      ProfScope prof("lstm_recurrence_fwd", st);
      TB_TRY(lstm2_fwd_wave_split(ws, p, y, notdone, c0, hN, cN, T1, B, H, st));  // writes hN / cN itself
    }
    return 0;
  }
  for (int l = 0; l < layers; ++l) {
    LstmLayerWs& L = ws.layer[l];
    float* hs = (l == layers - 1) ? y : L.hs;
    add2_kernel<<<(4 * H + 255) / 256, 256, 0, st>>>(p.b_ih[l], p.b_hh[l], L.bsum, 4 * H);
    TB_TRY(check_launch("add2_kernel"));
    if (precision) {
      const int64_t l16 = ld16(in_dim);
      TB_TRY(f32_to_bf16(xin, L.xb, N, in_dim, in_dim, l16, st, L.xb_lo));
      TB_TRY(pack_weights_bf16(p.w_ih[l], L.wihb, 4 * H, 1, in_dim, l16, st, L.wihb_lo));
      TcEpilogue te; te.C = L.gates; te.ldc = 4 * H; te.bias = L.bsum; te.tag = "lstm_xproj_fwd";
      te.a_lo = L.xb_lo; te.b_lo = L.wihb_lo;
      TB_TRY(gemm_tc_bf16(L.xb, L.wihb, N, 4 * H, in_dim, l16, l16, te, st));
    } else {
      GemmEpilogue ep; ep.bias = L.bsum; ep.tag = "lstm_xproj_fwd";
      TB_TRY((gemm_simt<float, float, false, true>(xin, p.w_ih[l], L.gates, N, 4 * H, in_dim, in_dim, in_dim, 4 * H, ep, 1,
                                                    nullptr, st)));
    }
    const int Hp = padded_h(H);
    // precision 2 (split-bf16 GEMMs) keeps the recurrence itself in exact fp32 (lstm_*_persistent_kernel)
    const bool use_mma = precision == 1 && mma_recurrence_applicable(B, H);
    if (!use_mma) {  // operands of the fp32 recurrence kernels
      const int64_t tot = int64_t(4 * H + 4) * Hp;
      lstm_pack_whh_kernel<<<(unsigned)((tot + 255) / 256 > 1184 ? 1184 : (tot + 255) / 256), 256, 0, st>>>(p.w_hh[l], L.wp, H, Hp);
      TB_TRY(check_launch("lstm_pack_whh_kernel"));
      cudaError_t em = cudaMemsetAsync(L.hm, 0, sizeof(float) * N * Hp, st);  // zero the row padding
      TB_REQUIRE(em == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(em));
      lstm_init_state_kernel<<<(unsigned)((B * Hp + 255) / 256), 256, 0, st>>>(
          h0 + int64_t(l) * B * H, c0 + int64_t(l) * B * H, notdone, L.hm, L.cm, int(B), H, Hp);
      TB_TRY(check_launch("lstm_init_state_kernel"));
    }
    ProfScope prof("lstm_recurrence_fwd", st);
    int prc = -1;
    if (use_mma) {
      const int Hq = mma_hq(H);
      cudaError_t eq = cudaMemsetAsync(L.hmq, 0, size_t(N) * Hq * 2, st);
      TB_REQUIRE(eq == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(eq));
      lstm_init_state_q_kernel<<<(unsigned)((B * Hq + 255) / 256), 256, 0, st>>>(
          h0 + int64_t(l) * B * H, c0 + int64_t(l) * B * H, notdone, static_cast<__nv_bfloat16*>(L.hmq), L.cm, int(B), H, Hq);
      TB_TRY(check_launch("lstm_init_state_q_kernel"));
      prc = lstm_fwd_persistent_mma(L, p.w_hh[l], hs, notdone, T1, B, H, ws.sync, st);
      TB_REQUIRE(prc >= 0, "lstm: tensor-core recurrence kernel does not fit (B=%lld H=%d)", (long long)B, H);
    }
    if (prc < 0 && precision == 2) prc = lstm_fwd_cluster(L, p.w_hh[l], hs, notdone, T1, B, H, st);   // H = 256, B <= 32
    if (prc < 0) prc = lstm_fwd_persistent(L, hs, notdone, T1, B, H, ws.sync, st);
    if (prc > 0) return prc;
    for (int64_t t = 0; prc < 0 && t < T1; ++t) {
      StepArgs a;
      a.hm = L.hm + t * B * Hp;
      a.cm = L.cm + t * B * H;
      const bool last = (t == T1 - 1);
      a.nd_next = last ? nullptr : notdone + (t + 1) * B;
      a.wp = L.wp;
      a.gates = L.gates + t * B * 4 * H;
      a.hs = hs + t * B * H; a.cs = L.cs + t * B * H;
      a.hm_next = last ? nullptr : L.hm + (t + 1) * B * Hp;
      a.cm_next = last ? nullptr : L.cm + (t + 1) * B * H;
      a.B = int(B); a.H = H; a.Hp = Hp;
      TB_TRY(launch_step_fwd(a, st));
    }
    cudaError_t e = cudaMemcpyAsync(hN + int64_t(l) * B * H, hs + (T1 - 1) * B * H, sizeof(float) * B * H,
                                    cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(cN + int64_t(l) * B * H, L.cs + (T1 - 1) * B * H, sizeof(float) * B * H,
                          cudaMemcpyDeviceToDevice, st);
    TB_REQUIRE(e == cudaSuccess, "lstm: state copy: %s", cudaGetErrorString(e));
    xin = hs;
    in_dim = H;
  }
  (void)splitk;
  return 0;
}

static int splits_for(int64_t M, int64_t N, int64_t K, int64_t scratch_floats) {
  const int64_t bm = (N <= 32) ? 128 : (M <= 64 ? 64 : 128), bn = (N <= 32) ? 32 : 64;
  const int64_t tiles = ((M + bm - 1) / bm) * ((N + bn - 1) / bn);
  int64_t s = (2 * kNumSMs + tiles - 1) / tiles;
  const int64_t ktiles = (K + kGemmBK - 1) / kGemmBK;
  if (s > ktiles / 4) s = ktiles / 4;
  if (s * M * N > scratch_floats) s = scratch_floats / (M * N);
  if (s > 64) s = 64;
  if (s < 1) s = 1;
  return int(s);
}

static thread_local SideStream* g_pending_join = nullptr;

int lstm_backward_join(cudaStream_t st) {
  if (!g_pending_join) return 0;
  cudaError_t e = cudaStreamWaitEvent(st, g_pending_join->join, 0);
  g_pending_join = nullptr;
  TB_REQUIRE(e == cudaSuccess, "lstm: side stream join: %s", cudaGetErrorString(e));
  return 0;
}

int lstm_backward(const float* dy, const float* x, const float* notdone, const LstmParams& p, const LstmGrads& g,
                  int64_t T1, int64_t B, int In, int H, int layers, LstmWs& ws, float* dx, float* splitk,
                  float* colsum_scratch, int precision, cudaStream_t st) {
  const int64_t N = T1 * B;
  const int64_t scratch = int64_t(8) << 20;  // == kSplitKScratchFloats (atarinet.cu)
  const float* dyl = dy;
  bool forked = false;
  // two layers on the tensor-core backend: ONE wavefront kernel runs both recurrences (and the upper layer's
  // input-gradient product); only the hoisted weight-gradient GEMMs and the lower layer's dx remain per layer
  bool wave_done = false;
  const bool split_fwd = precision == 2 && layers == 2 && wave_bwd_split_applicable(B, In, H);  // same predicate as the forward
  bool split_bwd = false;  // the split wavefront kernel ran: gate gradients are already bf16 hi/lo planes, bias gradients summed
  if (precision == 1 && layers == 2 && In <= H && wave_bwd_applicable(B, H)) {
    ProfScope prof("lstm_recurrence_bwd", st);
    TB_TRY(lstm2_bwd_wave(ws, p, g, dy, notdone, T1, B, H, st));
    wave_done = true;
  } else if (split_fwd) {
    // (the 4 padding columns of the [N, ld16(4H)] gate-gradient planes are never read as data: the GEMMs' tensor maps
    //  end at column 4H)
    ProfScope prof("lstm_recurrence_bwd", st);
    TB_TRY(lstm2_bwd_wave_split(ws, p, g, dy, notdone, T1, B, H, st));
    wave_done = true;
    split_bwd = true;
  }
  // After the wavefront kernel only the hoisted weight-gradient GEMMs of both layers (and the lower layer's dx) remain.
  // The GEMMs feed nothing downstream in this backward pass: fork them onto the side stream (own split-K scratch); the
  // caller joins with lstm_backward_join().
  SideStream* tail = (wave_done && ws.wg_scratch) ? side_stream() : nullptr;
  if (tail) {
    TB_TRY(lstm_backward_join(st));  // a previous call's fork must be joined before its event is reused
    cudaError_t ee = cudaEventRecord(tail->fork, st);
    if (ee == cudaSuccess) ee = cudaStreamWaitEvent(tail->stream, tail->fork, 0);
    TB_REQUIRE(ee == cudaSuccess, "lstm: side stream fork: %s", cudaGetErrorString(ee));
  }
  for (int l = layers - 1; l >= 0; --l) {
    LstmLayerWs& L = ws.layer[l];
    const float* xin = (l == 0) ? x : ws.layer[l - 1].hs;
    const int in_dim = (l == 0) ? In : H;
    float* dxl = (l == 0) ? dx : ws.dx_mid;
    const int Hp = padded_h(H);
    const bool use_mma = precision == 1 && mma_recurrence_applicable(B, H);
    if (!use_mma && !split_bwd) {  // operands of the fp32 recurrence kernels
      const int64_t tot = int64_t(H + 4) * 4 * Hp;
      lstm_pack_whh_t_kernel<<<(unsigned)((tot + 255) / 256 > 1184 ? 1184 : (tot + 255) / 256), 256, 0, st>>>(p.w_hh[l], L.w_hh_t, H, Hp);
      TB_TRY(check_launch("lstm_pack_whh_t_kernel"));
      cudaError_t em = cudaMemsetAsync(ws.dgp, 0, sizeof(float) * 4 * B * Hp, st);  // zero the row padding
      TB_REQUIRE(em == cudaSuccess, "lstm: memset: %s", cudaGetErrorString(em));
    }
    if (!wave_done) {
    ProfScope prof("lstm_recurrence_bwd", st);
    int prc = -1;
    if (use_mma) {
      prc = lstm_bwd_persistent_mma(L, p.w_hh[l], dyl, notdone, T1, B, H, g.b_ih[l], ws.sync + 16, st);
      TB_REQUIRE(prc >= 0, "lstm: tensor-core recurrence kernel does not fit (B=%lld H=%d)", (long long)B, H);
    }
    if (prc < 0 && precision == 2 && layers == 1) prc = lstm_bwd_cluster(L, p.w_hh[l], dyl, notdone, T1, B, H, st);   // H = 256, B <= 32
    if (prc < 0) prc = lstm_bwd_persistent(L, ws, dyl, notdone, T1, B, H, ws.sync + 16, st);
    if (prc > 0) return prc;
    for (int64_t t = T1 - 1; prc < 0 && t >= 0; --t) {
      BwdPointArgs a;
      a.dy = dyl + t * B * H;
      a.first = (t == T1 - 1);
      a.dh_raw = ws.dh; a.nd_next = a.first ? nullptr : notdone + (t + 1) * B;
      a.nd = notdone + t * B;
      a.gates = L.gates + t * B * 4 * H; a.cs = L.cs + t * B * H; a.cm = L.cm + t * B * H;
      a.dc = ws.dc; a.dgates = L.dgates + t * B * 4 * H; a.B = int(B); a.H = H; a.dgp = ws.dgp; a.Hp = Hp;
      const int64_t total = B * H;
      lstm_step_bwd_point_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a);
      TB_TRY(check_launch("lstm_step_bwd_point_kernel"));
      if (t > 0) {
        // dh_raw[B,H] = dgates_t[B,4H] . W_hh[4H,H]   (masked by notdone_t when consumed at t-1)
        DhArgs d;
        d.dgp = ws.dgp; d.wtp = L.w_hh_t; d.dh_raw = ws.dh; d.B = int(B); d.H = H; d.Hp = Hp;
        TB_TRY(launch_step_bwd_dh(d, st));
      }
    }
    }
    // parameter gradients over all steps at once
    if (precision) {
      const int64_t lg = ld16(4 * H), lh = ld16(H), li = ld16(in_dim);
      if (forked) {  // the upper layer's side-stream GEMMs used the split-K scratch: join before reusing it
        cudaError_t ej = cudaStreamWaitEvent(st, side_stream()->join, 0);
        TB_REQUIRE(ej == cudaSuccess, "lstm: side stream join: %s", cudaGetErrorString(ej));
        forked = false;
      }
      // the tensor-core recurrence wrote the gate gradients in bf16 and summed the bias gradients itself
      if (!use_mma && !split_bwd) TB_TRY(f32_to_bf16(L.dgates, L.dgb, N, 4 * H, 4 * H, lg, st, L.dgb_lo));
      const void* hm_b = L.hmb;
      int64_t hm_ld = lh, hm_lo = L.hmb_lo;
      const void* x_b = L.xb;
      int64_t x_ld = li, x_lo = L.xb_lo;
      if (use_mma) {  // the tensor-core forward recurrence already left the masked h in bf16
        hm_b = L.hmq; hm_ld = mma_hq(H); hm_lo = 0;
      } else if (split_fwd) {
        // the split wavefront forward left the masked h as hi / lo planes, and layer 1's input (= layer 0's raw h_t) is
        // slot t+1 of layer 0's exchange planes
        hm_b = L.hmq; hm_ld = mma_hq(H); hm_lo = L.hmq_lo;
        if (l == 1) {
          x_b = static_cast<const __nv_bfloat16*>(ws.layer[0].hq) + B * mma_hq(H); x_ld = mma_hq(H); x_lo = ws.layer[0].hq_lo;
        }
      } else {
        TB_TRY(f32_to_bf16(L.hm, L.hmb, N, H, padded_h(H), lh, st, L.hmb_lo));
      }
      const int64_t kb = (N + 63) / 64;
      int sp = int(kb / 8); if (sp < 1) sp = 1; if (sp > 4) sp = 4;
      // The weight-gradient GEMMs of the UPPER layer do not feed the lower layer's recurrence (only dx does), and that
      // recurrence occupies 65 SMs: run them on a side stream with a grid capped to the idle SMs and join before the
      // split-K scratch is needed again.
      SideStream* side = (use_mma && l == 1 && layers == 2 && !wave_done) ? side_stream() : nullptr;
      cudaStream_t gs = st;
      float* wscr = splitk;
      TcEpilogue te; te.tag = "lstm_wgrad";
      if (tail) {
        gs = tail->stream; wscr = ws.wg_scratch;
      }
      if (side) {
        cudaError_t ee = cudaEventRecord(side->fork, st);
        if (ee == cudaSuccess) ee = cudaStreamWaitEvent(side->stream, side->fork, 0);
        TB_REQUIRE(ee == cudaSuccess, "lstm: side stream fork: %s", cudaGetErrorString(ee));
        gs = side->stream;
        te.max_ctas = kNumSMs - int((H + kBwdCols - 1) / kBwdCols) - 2;
        forked = true;
      }
      te.C = g.w_hh[l]; te.ldc = H;      // dW_hh[4H,H] = dgates^T . hm   (both operands stored [N, .]: MN-major)
      te.a_lo = L.dgb_lo; te.b_lo = hm_lo;
      TB_TRY(gemm_tc_bf16_ex(L.dgb, hm_b, 4 * H, H, N, lg, hm_ld, true, true, te, sp, wscr, gs));
      te.C = g.w_ih[l]; te.ldc = in_dim;  // dW_ih[4H,in] = dgates^T . x
      te.b_lo = x_lo;
      TB_TRY(gemm_tc_bf16_ex(L.dgb, x_b, 4 * H, in_dim, N, lg, x_ld, true, true, te, sp, wscr, gs));
      if (!use_mma && !split_bwd) TB_TRY(colsum(L.dgates, g.b_ih[l], N, 4 * H, 4 * H, colsum_scratch, st));
      cudaError_t e = cudaMemcpyAsync(g.b_hh[l], g.b_ih[l], sizeof(float) * 4 * H, cudaMemcpyDeviceToDevice, gs);
      TB_REQUIRE(e == cudaSuccess, "lstm: bias grad copy: %s", cudaGetErrorString(e));
      if (side) {
        e = cudaEventRecord(side->join, side->stream);
        TB_REQUIRE(e == cudaSuccess, "lstm: side stream join: %s", cudaGetErrorString(e));
      }
      // dx[N,in] = dgates[N,4H] . W_ih[4H,in]   (W_ih as stored: reduction index is its row index)
      if (!(wave_done && l == 1)) {  // the wavefront kernel already produced the upper layer's dx (= ws.dx_mid)
        TcEpilogue td; td.tag = "lstm_xproj_dgrad"; td.C = dxl; td.ldc = in_dim;
        td.a_lo = L.dgb_lo; td.b_lo = L.wihb_lo;
        TB_TRY(gemm_tc_bf16_ex(L.dgb, L.wihb, N, in_dim, 4 * H, lg, li, false, true, td, 1, nullptr, st));
      }
    } else {
    GemmEpilogue ep; ep.tag = "lstm_wgrad";
    int s = splits_for(4 * H, H, N, scratch);
    TB_TRY((gemm_simt<float, float, true, false>(L.dgates, L.hm, g.w_hh[l], 4 * H, H, N, 4 * H, padded_h(H), H, ep, s, splitk,
                                                  st)));
    s = splits_for(4 * H, in_dim, N, scratch);
    TB_TRY((gemm_simt<float, float, true, false>(L.dgates, xin, g.w_ih[l], 4 * H, in_dim, N, 4 * H, in_dim, in_dim, ep, s,
                                                  splitk, st)));
    TB_TRY(colsum(L.dgates, g.b_ih[l], N, 4 * H, 4 * H, colsum_scratch, st));
    cudaError_t e = cudaMemcpyAsync(g.b_hh[l], g.b_ih[l], sizeof(float) * 4 * H, cudaMemcpyDeviceToDevice, st);
    TB_REQUIRE(e == cudaSuccess, "lstm: bias grad copy: %s", cudaGetErrorString(e));
    // gradient w.r.t. this layer's input: dx[N,in] = dgates[N,4H] . W_ih[4H,in]
    ep.tag = "lstm_xproj_dgrad";
    TB_TRY((gemm_simt<float, float, false, false>(L.dgates, p.w_ih[l], dxl, N, in_dim, 4 * H, 4 * H, in_dim, in_dim, ep, 1,
                                                   nullptr, st)));
    }
    dyl = dxl;
  }
  if (tail) {
    cudaError_t e = cudaEventRecord(tail->join, tail->stream);
    TB_REQUIRE(e == cudaSuccess, "lstm: side stream join: %s", cudaGetErrorString(e));
    g_pending_join = tail;
  }
  return 0;
}

}  // namespace tb

// =======================================================================================
// C ABI: the stacked LSTM on its own, hidden size / layers / batch as parameters (SURVEY 8(b) B3 tb_lstm_{fwd,bwd};
// BASELINE configs[4]: "long-unroll stress T=600 B=128, LSTM hidden=512")
// =======================================================================================
using namespace tb;

namespace {
constexpr int64_t kLstmAbiSplitK = int64_t(8) << 20;  // floats, == kSplitKScratchFloats of the network entry points

struct LstmAbiWs { LstmWs ws; float* splitk; float* colsum; size_t bytes; };

LstmAbiWs lstm_abi_ws(void* base, int64_t T1, int64_t B, int In, int H, int layers, int precision) {
  LstmAbiWs w;
  const size_t lbytes = lstm_ws_bytes(T1, B, In, H, layers, precision);
  size_t off = (lbytes + 255) & ~size_t(255);
  w.ws = lstm_ws(base, T1, B, In, H, layers, precision);
  w.splitk = base ? reinterpret_cast<float*>(static_cast<char*>(base) + off) : nullptr;
  off += size_t(kLstmAbiSplitK) * sizeof(float);
  w.colsum = base ? reinterpret_cast<float*>(static_cast<char*>(base) + off) : nullptr;
  off += size_t(colsum_scratch_floats(4 * int64_t(H) > 512 ? 4 * int64_t(H) : 512)) * sizeof(float);
  w.bytes = off;
  return w;
}

int lstm_abi_check(int64_t T1, int64_t B, int In, int H, int layers, int precision) {
  TB_REQUIRE(T1 >= 1 && B >= 1 && In >= 1 && H >= 1, "tb_lstm: bad sizes T1=%lld B=%lld In=%d H=%d", (long long)T1, (long long)B, In, H);
  TB_REQUIRE(layers >= 1 && layers <= kLstmMaxLayers, "tb_lstm: 1..%d layers", kLstmMaxLayers);
  TB_REQUIRE(precision >= 0 && precision <= 2, "tb_lstm: precision must be 0 (fp32), 1 (bf16) or 2 (split-bf16)");
  TB_REQUIRE(precision == 0 || ((In % 1) == 0), "tb_lstm: bad precision");
  return 0;
}
}  // namespace

extern "C" {

int tb_set_aux_stream(void* stream) {
  g_aux_stream = (cudaStream_t)stream;
  return 0;
}

size_t tb_lstm_workspace_bytes(int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision) {
  if (T1 < 1 || B < 1 || input_size < 1 || hidden_size < 1 || layers < 1 || layers > kLstmMaxLayers) return 0;
  return lstm_abi_ws(nullptr, T1, B, input_size, hidden_size, layers, precision).bytes;
}

int tb_lstm_forward(const float* x, const float* notdone, const float* h0, const float* c0, const float* const* params,
                    int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision, void* workspace,
                    float* y, float* hN, float* cN, void* stream) {
  if (lstm_abi_check(T1, B, input_size, hidden_size, layers, precision)) return 1;
  TB_REQUIRE(x && notdone && h0 && c0 && params && workspace && y && hN && cN, "tb_lstm_forward: null pointer");
  LstmParams p;
  for (int l = 0; l < layers; ++l) {
    p.w_ih[l] = params[4 * l]; p.w_hh[l] = params[4 * l + 1]; p.b_ih[l] = params[4 * l + 2]; p.b_hh[l] = params[4 * l + 3];
    TB_REQUIRE(p.w_ih[l] && p.w_hh[l] && p.b_ih[l] && p.b_hh[l], "tb_lstm_forward: null parameter pointer (layer %d)", l);
  }
  LstmAbiWs w = lstm_abi_ws(workspace, T1, B, input_size, hidden_size, layers, precision);
  return lstm_forward(x, notdone, h0, c0, p, T1, B, input_size, hidden_size, layers, w.ws, y, hN, cN, w.splitk, precision,
                      (cudaStream_t)stream);
}

int tb_lstm_backward(const float* dy, const float* x, const float* notdone, const float* const* params, float* const* grads,
                     int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision, void* workspace,
                     float* dx, void* stream) {
  if (lstm_abi_check(T1, B, input_size, hidden_size, layers, precision)) return 1;
  TB_REQUIRE(dy && x && notdone && params && grads && workspace && dx, "tb_lstm_backward: null pointer");
  LstmParams p; LstmGrads g;
  for (int l = 0; l < layers; ++l) {
    p.w_ih[l] = params[4 * l]; p.w_hh[l] = params[4 * l + 1]; p.b_ih[l] = params[4 * l + 2]; p.b_hh[l] = params[4 * l + 3];
    g.w_ih[l] = grads[4 * l]; g.w_hh[l] = grads[4 * l + 1]; g.b_ih[l] = grads[4 * l + 2]; g.b_hh[l] = grads[4 * l + 3];
    TB_REQUIRE(p.w_ih[l] && p.w_hh[l] && g.w_ih[l] && g.w_hh[l] && g.b_ih[l] && g.b_hh[l], "tb_lstm_backward: null pointer (layer %d)", l);
  }
  LstmAbiWs w = lstm_abi_ws(workspace, T1, B, input_size, hidden_size, layers, precision);
  int rc = lstm_backward(dy, x, notdone, p, g, T1, B, input_size, hidden_size, layers, w.ws, dx, w.splitk, w.colsum, precision,
                         (cudaStream_t)stream);
  if (rc) return rc;
  return lstm_backward_join((cudaStream_t)stream);
}

}  // extern "C"

