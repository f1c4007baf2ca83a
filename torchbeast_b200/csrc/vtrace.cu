// V-trace + IMPALA loss kernels for sm_90a (H100).
//
// Replaces the device-side work of (paths under /root/reference/torchbeast/):
//   core/vtrace.py:50-55    action_log_probs           -> action_log_probs_kernel
//   core/vtrace.py:91-139   from_importance_weights    -> vtrace_scan_kernel
//   core/vtrace.py:58-88 + monobeast.py:107-125,245-277 (== polybeast_learner.py:113-131,332-361)
//                           from_logits + 3 losses + their backward -> impala_loss_kernel
//
// Data layout: time-major [T,B] / [T,B,A], element (t,b) at t*B+b.  A CTA owns a tile of 32
// adjacent batch columns (one 128-byte row segment per time step, fully coalesced) and W warps
// split the unroll T into W contiguous chunks.  The recurrence
//     acc_t = delta_t + (gamma_t c_t) acc_{t+1},  acc_T = 0               (vtrace.py:116-120)
// is first-order linear, so each warp reduces its chunk to an affine map acc_in -> a*acc_in + b
// (pass 1), the W maps are composed through shared memory (pass 2, O(W)), and each warp then
// replays its chunk with the right carry-in and emits vs / pg_advantages / loss terms / grads
// (pass 3; re-reads hit L1/L2, HBM traffic stays the algorithmic 24*T*B+4*B bytes).  When the
// batch is wide enough to fill the chip W=1 and pass 3 alone runs (single streaming pass).
// This kernel is HBM-/latency-bound integer-free fp32 work: no tensor cores by design.
#include <cooperative_groups.h>
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace tb {

static int g_sm_count = 0;
static int sm_count() {
  if (g_sm_count == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      g_sm_count = n;
    else
      g_sm_count = kNumSMs;
  }
  return g_sm_count;
}

// Pick the number of T-chunks (warps per CTA) so that tiles*W warps roughly fill the chip.
static int pick_warps(int64_t T, int64_t tiles) {
  const int64_t target = int64_t(sm_count()) * 16;  // ~16 resident warps per SM
  int64_t w = target / (tiles > 0 ? tiles : 1);
  int64_t wmax = (T + 3) / 4;  // at least 4 time steps per chunk
  if (wmax > 16) wmax = 16;  // 512 threads per CTA
  if (w > wmax) w = wmax;
  if (w < 1) w = 1;
  return int(w);
}

constexpr int kWideWarps = 8;

static int pick_grid(int64_t tiles) {
  int64_t g = int64_t(sm_count()) * 8;
  if (g > kMaxPartialCtas) g = kMaxPartialCtas;
  if (tiles < g) g = tiles;
  return int(g < 1 ? 1 : g);
}

// ----------------------------------------------------------------------------------------
// scan only: from_importance_weights
// ----------------------------------------------------------------------------------------
template <typename F>
struct ScanArgs {
  const F* log_rhos; const F* discounts; const F* rewards; const F* values; const F* bootstrap;
  int64_t T, B;
  F clip_rho, clip_pg; int has_clip_rho, has_clip_pg;
  F* vs; F* pg_adv;
  int wide;  // 1: every warp owns its own column tile and the whole unroll (no T split, no smem)
};

template <typename F, int U>
__global__ void __launch_bounds__(512) vtrace_scan_kernel(ScanArgs<F> p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  F* sA = reinterpret_cast<F*>(smem_raw);
  F* sB = sA + blockDim.y * kWarp;
  const int lane = threadIdx.x;
  const int w = p.wide ? 0 : threadIdx.y, W = p.wide ? 1 : blockDim.y;
  const int64_t T = p.T, B = p.B;
  const int64_t tiles = (B + kWarp - 1) / kWarp;
  const int64_t chunk = (T + W - 1) / W;
  const int64_t t0 = (int64_t(w) * chunk < T) ? int64_t(w) * chunk : T;
  const int64_t t1 = (t0 + chunk < T) ? t0 + chunk : T;
  const int64_t tile0 = p.wide ? int64_t(blockIdx.x) * blockDim.y + threadIdx.y : blockIdx.x;
  const int64_t tile_step = p.wide ? int64_t(gridDim.x) * blockDim.y : gridDim.x;

  for (int64_t tile = tile0; tile < tiles; tile += tile_step) {
    const int64_t b = tile * kWarp + lane;
    const bool active = b < B;
    F acc_in = F(0);
    if (W > 1) {
      // pass 1: chunk -> affine map (a, bb)
      F a = F(1), bb = F(0);
      if (active && t1 > t0) {
        F v_next = (t1 < T) ? p.values[t1 * B + b] : p.bootstrap[b];
        for (int64_t te = t1; te > t0; te -= U) {
          F lr[U], g[U], r[U], v[U];
#pragma unroll
          for (int k = 0; k < U; ++k) {
            const int64_t t = te - 1 - k;
            if (t >= t0) {
              const int64_t i = t * B + b;
              lr[k] = p.log_rhos[i]; g[k] = p.discounts[i]; r[k] = p.rewards[i]; v[k] = p.values[i];
            }
          }
#pragma unroll
          for (int k = 0; k < U; ++k) {
            const int64_t t = te - 1 - k;
            if (t >= t0) {
              const F rho = M<F>::exp(lr[k]);
              const F c = M<F>::min(rho, F(1));
              const F rb = p.has_clip_rho ? M<F>::min(rho, p.clip_rho) : rho;
              const F delta = rb * (r[k] + g[k] * v_next - v[k]);
              const F dc = g[k] * c;
              bb = delta + dc * bb;
              a = dc * a;
              v_next = v[k];
            }
          }
        }
      }
      __syncthreads();  // previous tile's pass-2 reads are done
      sA[w * kWarp + lane] = a;
      sB[w * kWarp + lane] = bb;
      __syncthreads();
      // pass 2: carry-in of this chunk = composition of all later chunks applied to 0
      for (int w2 = W - 1; w2 > w; --w2) acc_in = sB[w2 * kWarp + lane] + sA[w2 * kWarp + lane] * acc_in;
    }
    if (!active || t1 <= t0) continue;
    // pass 3: replay with carry-in, emit outputs
    F v_next = (t1 < T) ? p.values[t1 * B + b] : p.bootstrap[b];
    F vs_next = (t1 < T) ? acc_in + v_next : v_next;
    F acc = acc_in;
    for (int64_t te = t1; te > t0; te -= U) {
      F lr[U], g[U], r[U], v[U];
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const int64_t t = te - 1 - k;
        if (t >= t0) {
          const int64_t i = t * B + b;
          lr[k] = p.log_rhos[i]; g[k] = p.discounts[i]; r[k] = p.rewards[i]; v[k] = p.values[i];
        }
      }
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const int64_t t = te - 1 - k;
        if (t >= t0) {
          const int64_t i = t * B + b;
          const F rho = M<F>::exp(lr[k]);
          const F c = M<F>::min(rho, F(1));
          const F rb = p.has_clip_rho ? M<F>::min(rho, p.clip_rho) : rho;
          const F rp = p.has_clip_pg ? M<F>::min(rho, p.clip_pg) : rho;
          const F delta = rb * (r[k] + g[k] * v_next - v[k]);
          acc = delta + (g[k] * c) * acc;
          const F vst = acc + v[k];
          p.pg_adv[i] = rp * (r[k] + g[k] * vs_next - v[k]);
          p.vs[i] = vst;
          vs_next = vst;
          v_next = v[k];
        }
      }
    }
  }
}

// Long unrolls on few columns (BASELINE configs[4]: T = 600, B = 128 -> 4 column tiles): one CTA per tile leaves the unroll to
// 16 warps x 38 dependent steps.  Here a thread-block CLUSTER of C CTAs owns the tile: 16*C warps split T (5 steps per warp at
// T = 600, C = 8), every warp folds its chunk into an affine map (pass 1), a CTA composes its 16 maps into one, the cluster
// exchanges the C per-CTA maps through DISTRIBUTED SHARED MEMORY (cluster.sync + map_shared_rank reads of 2 x 32 floats per later
// CTA), and every warp replays its chunk with the right carry-in (pass 3).  Same arithmetic and summation order as the
// single-CTA kernel within a chunk; the chunk boundaries differ, which moves results by fp32 rounding of the affine composition
// (covered by the same tolerances: tests/test_vtrace_gpu.py).
template <typename F, int U>
__global__ void __launch_bounds__(512) vtrace_scan_cluster_kernel(ScanArgs<F> p) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int W = blockDim.y, C = int(cluster.num_blocks()), rank = int(cluster.block_rank());
  F* sA = reinterpret_cast<F*>(smem_raw);      // [W][32] per-warp maps
  F* sB = sA + W * kWarp;
  F* sCA = sB + W * kWarp;                     // [32] this CTA's composed map (read by the other CTAs of the cluster)
  F* sCB = sCA + kWarp;
  const int lane = threadIdx.x, w = threadIdx.y;
  const int64_t T = p.T, B = p.B;
  const int64_t tile = blockIdx.x / C;
  const int64_t b = tile * kWarp + lane;
  const bool active = b < B;
  const int64_t chunk = (T + int64_t(W) * C - 1) / (int64_t(W) * C);
  const int64_t gw = int64_t(rank) * W + w;    // chunk index along T (rank-major: a CTA owns W consecutive chunks)
  const int64_t t0 = (gw * chunk < T) ? gw * chunk : T;
  const int64_t t1 = (t0 + chunk < T) ? t0 + chunk : T;
  // pass 1: chunk -> affine map (a, bb); the chunk's operands stay in registers for pass 3 (chunk <= U)
  F lr[U], g[U], r[U], v[U];
  F a = F(1), bb = F(0);
  F v_last = F(0);
  if (active && t1 > t0) {
    v_last = (t1 < T) ? p.values[t1 * B + b] : p.bootstrap[b];
    F v_next = v_last;
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t t = t1 - 1 - k;
      if (t >= t0) {
        const int64_t i = t * B + b;
        lr[k] = p.log_rhos[i]; g[k] = p.discounts[i]; r[k] = p.rewards[i]; v[k] = p.values[i];
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t t = t1 - 1 - k;
      if (t >= t0) {
        const F rho = M<F>::exp(lr[k]);
        const F c = M<F>::min(rho, F(1));
        const F rb = p.has_clip_rho ? M<F>::min(rho, p.clip_rho) : rho;
        const F delta = rb * (r[k] + g[k] * v_next - v[k]);
        const F dc = g[k] * c;
        bb = delta + dc * bb;
        a = dc * a;
        v_next = v[k];
      }
    }
  }
  sA[w * kWarp + lane] = a;
  sB[w * kWarp + lane] = bb;
  __syncthreads();
  if (w == 0) {  // this CTA's W maps composed (latest chunk applied first)
    F ca = F(1), cb = F(0);
    for (int w2 = W - 1; w2 >= 0; --w2) { cb = sB[w2 * kWarp + lane] + sA[w2 * kWarp + lane] * cb; ca = sA[w2 * kWarp + lane] * ca; }
    sCA[lane] = ca; sCB[lane] = cb;
  }
  cluster.sync();
  // carry-in: all later CTAs (through DSMEM), then the later warps of this CTA
  F acc_in = F(0);
  for (int r2 = C - 1; r2 > rank; --r2) {
    const F* ra = cluster.map_shared_rank(sCA, r2);
    const F* rb2 = cluster.map_shared_rank(sCB, r2);
    acc_in = rb2[lane] + ra[lane] * acc_in;
  }
  for (int w2 = W - 1; w2 > w; --w2) acc_in = sB[w2 * kWarp + lane] + sA[w2 * kWarp + lane] * acc_in;
  if (active && t1 > t0) {  // pass 3: replay from registers
    F v_next = v_last;
    F vs_next = (t1 < T) ? acc_in + v_next : v_next;
    F acc = acc_in;
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t t = t1 - 1 - k;
      if (t >= t0) {
        const int64_t i = t * B + b;
        const F rho = M<F>::exp(lr[k]);
        const F c = M<F>::min(rho, F(1));
        const F rb = p.has_clip_rho ? M<F>::min(rho, p.clip_rho) : rho;
        const F rp = p.has_clip_pg ? M<F>::min(rho, p.clip_pg) : rho;
        const F delta = rb * (r[k] + g[k] * v_next - v[k]);
        acc = delta + (g[k] * c) * acc;
        const F vst = acc + v[k];
        p.pg_adv[i] = rp * (r[k] + g[k] * vs_next - v[k]);
        p.vs[i] = vst;
        vs_next = vst;
        v_next = v[k];
      }
    }
  }
  cluster.sync();  // no CTA may exit while another still reads its shared memory
}

// cluster size for the T-split across CTAs: the largest power of two <= 8 that leaves >= 4 time steps per warp (0: not worth it)
static int pick_cluster(int64_t T, int64_t tiles, int W) {
  if (W < 16 || tiles * 16 > int64_t(sm_count()) * 2) return 0;  // enough tiles to fill the chip without it
  int c = 8;
  while (c > 1 && (T < int64_t(16) * c * 4 || (T + int64_t(16) * c - 1) / (int64_t(16) * c) > 8)) c >>= 1;
  if (c > 1 && (T + int64_t(16) * c - 1) / (int64_t(16) * c) > 8) return 0;  // chunk must fit the register window (U = 8)
  return c > 1 ? c : 0;
}

template <typename F>
static int launch_scan(const F* log_rhos, const F* discounts, const F* rewards, const F* values,
                       const F* bootstrap, int64_t T, int64_t B, F clip_rho, F clip_pg, F* vs,
                       F* pg_adv, void* stream) {
  TB_REQUIRE(T >= 0 && B >= 0, "vtrace scan: negative size T=%lld B=%lld", (long long)T, (long long)B);
  if (T == 0 || B == 0) return 0;
  TB_REQUIRE(log_rhos && discounts && rewards && values && bootstrap && vs && pg_adv,
             "vtrace scan: null pointer");
  ScanArgs<F> a;
  a.log_rhos = log_rhos; a.discounts = discounts; a.rewards = rewards; a.values = values;
  a.bootstrap = bootstrap; a.T = T; a.B = B;
  a.has_clip_rho = (clip_rho >= F(0));  // NaN compares false -> None
  a.has_clip_pg = (clip_pg >= F(0));
  a.clip_rho = clip_rho; a.clip_pg = clip_pg; a.vs = vs; a.pg_adv = pg_adv;
  const int64_t tiles = (B + kWarp - 1) / kWarp;
  int W = pick_warps(T, tiles);
  a.wide = (W == 1);
  dim3 grid(pick_grid(tiles));
  if (a.wide) {  // wide batch: 8 warps per CTA, one column tile each, enough CTAs for every tile
    W = kWideWarps;
    int64_t g = (tiles + W - 1) / W;
    grid = dim3((unsigned)(g < 1 ? 1 : g));
  }
  dim3 block(kWarp, W);
  size_t smem = size_t(2) * W * kWarp * sizeof(F);
  ProfScope prof("vtrace_scan", (cudaStream_t)stream);
  const int C = a.wide ? 0 : pick_cluster(T, tiles, W);
  if (C > 1) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(tiles * C));
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem + 2 * kWarp * sizeof(F);
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = unsigned(C); attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, vtrace_scan_cluster_kernel<F, 8>, a);
    if (e == cudaSuccess) return check_launch("vtrace_scan_cluster_kernel");
    cudaGetLastError();  // cluster launch not possible here: fall through to the single-CTA kernel
  }
  vtrace_scan_kernel<F, 8><<<grid, block, smem, (cudaStream_t)stream>>>(a);
  return check_launch("vtrace_scan_kernel");
}

// ----------------------------------------------------------------------------------------
// log-softmax helpers (row in registers, A compile-time; A==0 -> runtime loop over global)
// ----------------------------------------------------------------------------------------
template <typename F, int A>
struct RowOps {
  // returns log(sum exp(x - m)) and m; x loaded into registers
  static __device__ __forceinline__ void load(const F* __restrict__ row, int64_t, F (&x)[A]) {
#pragma unroll
    for (int j = 0; j < A; ++j) x[j] = row[j];
  }
  static __device__ __forceinline__ void lse(const F (&x)[A], F& m, F& logs) {
    m = x[0];
#pragma unroll
    for (int j = 1; j < A; ++j) m = M<F>::max(m, x[j]);
    F s = F(0);
#pragma unroll
    for (int j = 0; j < A; ++j) s += M<F>::exp(x[j] - m);
    logs = M<F>::log(s);
  }
  static __device__ __forceinline__ F pick(const F (&x)[A], int64_t a) {
    F r = x[0];
#pragma unroll
    for (int j = 1; j < A; ++j) r = (a == j) ? x[j] : r;
    return r;
  }
};

// log pi(a) for one row of runtime length A (global re-reads; used when A has no instantiation)
template <typename F>
__device__ __forceinline__ F alp_dyn(const F* __restrict__ row, int64_t A, int64_t a, F* m_out, F* logs_out) {
  F m = row[0];
  for (int64_t j = 1; j < A; ++j) m = M<F>::max(m, row[j]);
  F s = F(0);
  for (int64_t j = 0; j < A; ++j) s += M<F>::exp(row[j] - m);
  const F logs = M<F>::log(s);
  if (m_out) { *m_out = m; *logs_out = logs; }
  // an action index outside [0, A) is a caller bug (the reference's nll_loss raises "Target out of bounds"); a kernel
  // cannot raise, so it must neither read out of bounds nor silently pick a logit: the result is NaN, which poisons the
  // loss and is caught by the caller's finiteness checks
  if (a < 0 || a >= A) return F(NAN);
  return (row[a] - m) - logs;
}

template <typename F, int A>
__device__ __forceinline__ F alp_row(const F* __restrict__ row, int64_t Adyn, int64_t a, F* m_out, F* logs_out) {
  if constexpr (A == 0) {
    return alp_dyn<F>(row, Adyn, a, m_out, logs_out);
  } else {
    F x[A];
    RowOps<F, A>::load(row, Adyn, x);
    F m, logs;
    RowOps<F, A>::lse(x, m, logs);
    if (m_out) { *m_out = m; *logs_out = logs; }
    if (a < 0 || a >= A) return F(NAN);  // see alp_dyn
    return (RowOps<F, A>::pick(x, a) - m) - logs;
  }
}

template <typename F, int A>
__global__ void action_log_probs_kernel(const F* __restrict__ logits, const int64_t* __restrict__ actions,
                                        int64_t N, int64_t Adyn, F* __restrict__ out) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const int64_t Ause = A ? A : Adyn;
    out[i] = alp_row<F, A>(logits + i * Ause, Adyn, actions[i], nullptr, nullptr);
  }
}

#define TB_DISPATCH_A(Aval, CALL)                          \
  switch (Aval) {                                          \
    case 2: { constexpr int kA = 2; CALL; } break;         \
    case 3: { constexpr int kA = 3; CALL; } break;         \
    case 4: { constexpr int kA = 4; CALL; } break;         \
    case 5: { constexpr int kA = 5; CALL; } break;         \
    case 6: { constexpr int kA = 6; CALL; } break;         \
    case 7: { constexpr int kA = 7; CALL; } break;         \
    case 8: { constexpr int kA = 8; CALL; } break;         \
    case 9: { constexpr int kA = 9; CALL; } break;         \
    case 10: { constexpr int kA = 10; CALL; } break;       \
    case 12: { constexpr int kA = 12; CALL; } break;       \
    case 14: { constexpr int kA = 14; CALL; } break;       \
    case 16: { constexpr int kA = 16; CALL; } break;       \
    case 18: { constexpr int kA = 18; CALL; } break;       \
    default: { constexpr int kA = 0; CALL; } break;        \
  }

template <typename F>
static int launch_alp(const F* logits, const int64_t* actions, int64_t N, int64_t A, F* out, void* stream) {
  TB_REQUIRE(N >= 0 && A >= 1, "action_log_probs: bad sizes N=%lld A=%lld", (long long)N, (long long)A);
  if (N == 0) return 0;
  TB_REQUIRE(logits && actions && out, "action_log_probs: null pointer");
  const int threads = 256;
  int64_t blocks = (N + threads - 1) / threads;
  const int64_t cap = int64_t(sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  TB_DISPATCH_A(A, (action_log_probs_kernel<F, kA><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
                       logits, actions, N, A, out)));
  return check_launch("action_log_probs_kernel");
}

// ----------------------------------------------------------------------------------------
// fused from_logits + losses + backward
// ----------------------------------------------------------------------------------------
struct LossArgs {
  const float* blogits; const float* tlogits; const int64_t* actions; const float* rewards;
  const uint8_t* done; const float* discounts; const float* values; const float* bootstrap;
  int64_t T, B, A;
  float discounting, baseline_cost, entropy_cost;
  int clip_rewards; float clip_rho, clip_pg; int has_clip_rho, has_clip_pg;
  float* vs; float* pg_adv; float* log_rhos; float* balp; float* talp; float* losses;
  float* grad_logits; float* grad_values; int zero_tail;
  void* workspace;
  int wide;  // see ScanArgs
  const tb_hparams* hp;  // nullable: overrides the scalars above when the kernel runs
  // PopArt (impala_loss_kernel<A, true> only): `values` holds the normalised value head [T+1,B,K] (bootstrap row
  // included, `bootstrap` unused), row (t,b) uses task[t*B+b]; grad_values is [T+1,B,K]
  const int64_t* task; const double* pa_mu; const double* pa_nu; int K;
  // importance weights (impala_loss_kernel<A, false, true> only): column b's pg, baseline and entropy terms, in the
  // losses and the gradients, are multiplied by column_weights[b]
  const float* column_weights;
  // trust region (impala_loss_kernel<A, *, *, true> only): beta read from *trust_beta when the kernel runs, kl [T,B]
  // out, trust_out [2] = {trusted rows, sum kl}
  const float* trust_beta; float* kl; float* trust_out;
  // factored action space (impala_loss_kernel<0, *, *, *, true> only): actions are [T,B,D], row segments as in seg
  ActionSegments seg;
  // A diagonal-Gaussian policy (impala_loss_kernel<kGaussianRows, ...>) adds no field: its rows are (mu, log sigma)
  // of width A = 2D, and `actions` carries the address of its float32 [T,B,D] actions (gaussian_actions), so the
  // struct, and every kernel that takes it, keeps the layout it had before Gaussian rows existed.
};

// ---- continuous (diagonal-Gaussian) action spaces (impala_loss_kernel<kGaussianRows, ...>) ---------------------------
// A row of width A = 2D is (mu_0 .. mu_{D-1}, l_0 .. l_{D-1}), sigma_k = expf(l_k).  Every sum over k runs in index
// order and starts from the k = 0 term; a non-finite input makes the quantity NaN (include/torchbeast_b200.h,
// "continuous (diagonal-Gaussian) action spaces").
constexpr float kHalfLog2Pi = TB_GAUSSIAN_HALF_LOG_2PI;
constexpr int kGaussianRows = -1;  // impala_loss_kernel's row-width argument for Gaussian rows

__device__ __forceinline__ const float* gaussian_actions(const LossArgs& p) {
  return reinterpret_cast<const float*>(p.actions);
}

__device__ __forceinline__ bool gaussian_finite(float mu, float l) { return isfinite(mu) && isfinite(l); }

// log pi(a) = sum_k (-0.5 z_k^2 - l_k - c), z_k = (a_k - mu_k) expf(-l_k)
__device__ __forceinline__ float alp_gaussian(const float* __restrict__ row, int D, const float* __restrict__ act) {
  float lp = 0.0f;
  bool ok = true;
  for (int k = 0; k < D; ++k) {
    const float mu = row[k], l = row[D + k], a = act[k];
    ok = ok && gaussian_finite(mu, l) && isfinite(a);
    const float z = (a - mu) * expf(-l);
    const float term = (-0.5f * (z * z) - l) - kHalfLog2Pi;
    lp = k == 0 ? term : lp + term;
  }
  return ok ? lp : __int_as_float(0x7fffffff);
}

// KL(pi || mu_b) of row i: sum_k ((lb_k - l_k) + 0.5 (expf(2 (l_k - lb_k)) + ((mu_k - mub_k) expf(-lb_k))^2) - 0.5)
__device__ __forceinline__ float trust_kl_gaussian(const LossArgs& p, int64_t i) {
  const int D = int(p.A / 2);
  const float* trow = p.tlogits + i * p.A;
  const float* brow = p.blogits + i * p.A;
  float kl = 0.0f;
  bool ok = true;
  for (int k = 0; k < D; ++k) {
    const float mu = trow[k], l = trow[D + k], mub = brow[k], lb = brow[D + k];
    ok = ok && gaussian_finite(mu, l) && gaussian_finite(mub, lb);
    const float dm = (mu - mub) * expf(-lb);
    const float term = ((lb - l) + 0.5f * (expf(2.0f * (l - lb)) + dm * dm)) - 0.5f;
    kl = k == 0 ? term : kl + term;
  }
  return ok ? kl : __int_as_float(0x7fffffff);
}

// The entropy term ent = sum_k -(l_k + 0.5 + c) of row i, and with grad_logits its gradient row: mu_k gets
// -adv z_k expf(-l_k), l_k gets adv (1 - z_k^2) - entropy_cost, each times column_weights[b] when kWeighted.  A row or
// action with a non-finite entry gets NaN for the term and the whole gradient row.
template <bool kWeighted>
__device__ __forceinline__ float gaussian_entropy_grad(const LossArgs& p, int64_t i, int64_t b, float adv) {
  const int D = int(p.A / 2);
  const float* row = p.tlogits + i * p.A;
  const float* act = gaussian_actions(p) + i * D;
  float ent = 0.0f;
  bool ok = true;
  for (int k = 0; k < D; ++k) {
    const float l = row[D + k];
    ok = ok && gaussian_finite(row[k], l) && isfinite(act[k]);
    const float term = -((l + 0.5f) + kHalfLog2Pi);
    ent = k == 0 ? term : ent + term;
  }
  const float nan = __int_as_float(0x7fffffff);
  if (p.grad_logits) {
    float* g = p.grad_logits + i * p.A;
    const float wb = kWeighted ? __ldg(p.column_weights + b) : 1.0f;
    for (int k = 0; k < D; ++k) {
      const float mu = row[k], l = row[D + k];
      const float s = expf(-l), z = (act[k] - mu) * s;
      float gm = ((-adv) * z) * s, gl = adv * (1.0f - z * z) - p.entropy_cost;
      if (!ok) gm = gl = nan;
      if constexpr (kWeighted) { gm *= wb; gl *= wb; }
      g[k] = gm;
      g[D + k] = gl;
    }
  }
  return ok ? ent : nan;
}

// ---- factored action spaces (impala_loss_kernel<0, *, *, *, true>) -----------------------------------------------------
// Each segment is a row of its own for alp_dyn, the code the flat rows use; the sums over segments run in index order from
// segment 0 (include/torchbeast_b200.h, "multi-discrete (factored) action spaces").

// log pi(a) = sum_k log pi_k(a_k) of the row at `row`, actions act[0..D)
__device__ __forceinline__ float alp_factored(const ActionSegments& seg, const float* __restrict__ row,
                                              const int64_t* __restrict__ act) {
  float lp = alp_dyn<float>(row, seg.off[1], act[0], nullptr, nullptr);
  for (int k = 1; k < seg.D; ++k)
    lp += alp_dyn<float>(row + seg.off[k], seg.off[k + 1] - seg.off[k], act[k], nullptr, nullptr);
  return lp;
}

// sum_k KL(pi_k || mu_k) of row i in fp32, each segment as trust_kl forms a whole row
__device__ __forceinline__ float trust_kl_factored(const LossArgs& p, int64_t i) {
  const float* trow = p.tlogits + i * p.A;
  const float* brow = p.blogits + i * p.A;
  float kl = 0.0f;
  for (int k = 0; k < p.seg.D; ++k) {
    const int o = p.seg.off[k], Ak = p.seg.off[k + 1] - o;
    float mt, logst, mb, logsb;
    alp_dyn<float>(trow + o, Ak, 0, &mt, &logst);
    alp_dyn<float>(brow + o, Ak, 0, &mb, &logsb);
    float klk = 0.0f;
    for (int j = o; j < o + Ak; ++j) {
      const float lt = (trow[j] - mt) - logst, lb = (brow[j] - mb) - logsb;
      klk += expf(lt) * (lt - lb);
    }
    kl = k == 0 ? klk : kl + klk;
  }
  return kl;
}

// The entropy term sum_k ent_k of row i, and with grad_logits its gradient row: segment k gets
// adv * (p - onehot(a_k)) + entropy_cost * p * (lp - ent_k), times column_weights[b] when kWeighted.
template <bool kWeighted>
__device__ __forceinline__ float factored_entropy_grad(const LossArgs& p, int64_t i, int64_t b, float adv) {
  const float* trow = p.tlogits + i * p.A;
  const int64_t* act = p.actions + i * p.seg.D;
  float ent_row = 0.0f;
  for (int k = 0; k < p.seg.D; ++k) {
    const int o = p.seg.off[k], Ak = p.seg.off[k + 1] - o;
    const float* srow = trow + o;
    const int64_t ak = act[k];
    float m, logs;
    alp_dyn<float>(srow, Ak, 0, &m, &logs);
    float ent = 0.0f;
    for (int j = 0; j < Ak; ++j) {
      const float lp = (srow[j] - m) - logs;
      ent += expf(lp) * lp;
    }
    if (p.grad_logits) {
      float* g = p.grad_logits + i * p.A + o;
      for (int j = 0; j < Ak; ++j) {
        const float lp = (srow[j] - m) - logs, pr = expf(lp);
        const float gl = adv * (pr - (ak == j ? 1.0f : 0.0f)) + p.entropy_cost * pr * (lp - ent);
        if constexpr (kWeighted) g[j] = gl * __ldg(p.column_weights + b); else g[j] = gl;
      }
    }
    ent_row = k == 0 ? ent : ent_row + ent;
  }
  return ent_row;
}

// ---- trust region (impala_loss_kernel<A, *, *, true>) ----------------------------------------------------------------
// The kernel reaches the trust region only through the three helpers below, so the instantiations without it compile
// to the same code as before the trust region existed.

// KL(pi || mu) of row i in fp32.  Each row's max and log-sum-exp come from alp_row, the code that forms the action
// log-probabilities, so both log-softmaxes are the ones behind target_alp / behavior_alp; identical rows give 0.
template <int A>
__device__ __forceinline__ float trust_kl(const LossArgs& p, int64_t i, int64_t Ause) {
  const float* trow = p.tlogits + i * Ause;
  const float* brow = p.blogits + i * Ause;
  float mt, logst, mb, logsb;
  alp_row<float, A>(trow, Ause, 0, &mt, &logst);
  alp_row<float, A>(brow, Ause, 0, &mb, &logsb);
  float kl = 0.0f;
  if constexpr (A == 0) {
    for (int64_t j = 0; j < Ause; ++j) {
      const float lt = (trow[j] - mt) - logst, lb = (brow[j] - mb) - logsb;
      kl += expf(lt) * (lt - lb);
    }
  } else {
    float xt[A], xb[A];
    RowOps<float, A>::load(trow, Ause, xt);
    RowOps<float, A>::load(brow, Ause, xb);
#pragma unroll
    for (int j = 0; j < A; ++j) {
      const float lt = (xt[j] - mt) - logst, lb = (xb[j] - mb) - logsb;
      kl += expf(lt) * (lt - lb);
    }
  }
  return kl;
}

// rho of row i under the trust region: expf(lr) where kl_i <= beta, else 0 (a NaN kl too).  kl_i is formed and written
// to p.kl here, or, with `written`, read back from there (pass 1 of the split layout wrote it in this thread).
template <int A, bool kFactored = false, bool kGaussian = false>
__device__ __forceinline__ float trust_rho(const LossArgs& p, int64_t i, int64_t Ause, float lr, bool written) {
  float kl;
  if (written) {
    kl = p.kl[i];
  } else {
    if constexpr (kGaussian) kl = trust_kl_gaussian(p, i);
    else if constexpr (kFactored) kl = trust_kl_factored(p, i);
    else kl = trust_kl<A>(p, i, Ause);
    p.kl[i] = kl;
  }
  const float rho = expf(lr);
  return kl <= *p.trust_beta ? rho : 0.0f;
}

// The end of the trust-region kernel: the trusted rows and the sum of kl over this thread's rows, read back from p.kl
// in the order pass 3 walked them, then one five-value grid sum.  The loss values are those grid_sum3 would give.
__device__ __forceinline__ void trust_finish(const LossArgs& p, double s_pg, double s_bl, double s_en, int64_t tile0,
                                             int64_t tile_step, int64_t t0, int64_t t1) {
  const int64_t tiles = (p.B + kWarp - 1) / kWarp;
  const float beta = *p.trust_beta;
  double rows = 0.0, kl_sum = 0.0;
  for (int64_t tile = tile0; tile < tiles; tile += tile_step) {
    const int64_t b = tile * kWarp + threadIdx.x;
    if (b >= p.B) continue;
    for (int64_t t = t1 - 1; t >= t0; --t) {
      const float kl = p.kl[t * p.B + b];
      rows += (kl <= beta) ? 1.0 : 0.0;
      kl_sum += double(kl);
    }
  }
  double s[5] = {s_pg, s_bl, s_en, rows, kl_sum}, tot[5];
  if (grid_sum<5>(s, p.workspace, tot)) {
    const double pg = tot[0], bl = double(p.baseline_cost) * tot[1], en = double(p.entropy_cost) * tot[2];
    p.losses[0] = float(pg); p.losses[1] = float(bl); p.losses[2] = float(en); p.losses[3] = float(pg + bl + en);
    p.trust_out[0] = float(tot[3]); p.trust_out[1] = float(tot[4]);
  }
}

constexpr int kPopArtMaxTasks = 64;

// PopArt sigma of one task from its first and second moments (include/torchbeast_b200.h)
__host__ __device__ __forceinline__ double popart_sigma(double mu, double nu) {
  const double s = sqrt(fmax(nu - mu * mu, 0.0));
  return fmin(fmax(s, 1e-4), 1e6);
}

// The scalars of a tb_hparams block, with has_clip_* derived as the float-argument entry point derives them.
__device__ __forceinline__ void load_hparams(LossArgs& p) {
  const tb_hparams* h = p.hp;
  p.discounting = h->discounting; p.baseline_cost = h->baseline_cost; p.entropy_cost = h->entropy_cost;
  p.clip_rewards = h->clip_rewards; p.clip_rho = h->clip_rho; p.clip_pg = h->clip_pg_rho;
  p.has_clip_rho = (p.clip_rho >= 0.0f); p.has_clip_pg = (p.clip_pg >= 0.0f);
}

__device__ __forceinline__ float reward_of(const LossArgs& p, int64_t i) {
  float r = p.rewards[i];
  if (p.clip_rewards) r = fminf(fmaxf(r, -1.0f), 1.0f);
  return r;
}
__device__ __forceinline__ float discount_of(const LossArgs& p, int64_t i) {
  return p.discounts ? p.discounts[i] : (p.done[i] ? 0.0f : p.discounting);
}

// kPopArt: the value input is PopArt-normalised (LossArgs::task / pa_mu / pa_nu / K); the non-PopArt instantiations
// compile none of that code.  kWeighted: every term of column b is multiplied by LossArgs::column_weights[b], after the
// unweighted term is formed, so a weight of 1.0f gives the unweighted bits; the other instantiations compile no weight
// code.  kTrust: row (t, b) with kl_t = KL(pi_t || mu_t) > beta (or NaN) runs the V-trace and the policy gradient with
// rho_t = 0 (include/torchbeast_b200.h, tb_impala_loss_f32); the other instantiations compile no trust code.  kFactored
// (with A = 0 only): actions are [T,B,D] and every row quantity is formed per segment (LossArgs::seg); the other
// instantiations compile none of that code.  AT = kGaussianRows: diagonal-Gaussian rows (mu, log sigma) on the
// dynamic-A path (A = 0 below), whose actions are float32 [T,B,D] (gaussian_actions); the other instantiations compile
// none of that code.  The row kind rides on AT rather than on a sixth flag so that the categorical instantiations keep
// the names they had before Gaussian rows existed.
template <int AT, bool kPopArt = false, bool kWeighted = false, bool kTrust = false, bool kFactored = false>
__global__ void __launch_bounds__(512) impala_loss_kernel(LossArgs p) {
  constexpr bool kGaussian = AT == kGaussianRows;
  constexpr int A = kGaussian ? 0 : AT;
  static_assert(!kFactored || A == 0, "factored rows take the dynamic-A path");
  static_assert(!kGaussian || !kFactored, "a row is factored or Gaussian");
  if (p.hp) load_hparams(p);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sA = reinterpret_cast<float*>(smem_raw);
  float* sB = sA + blockDim.y * kWarp;
  float* sMu = sB + blockDim.y * kWarp;  // PopArt: per-task mu and sigma in fp32, [K] each
  float* sSig = sMu + kPopArtMaxTasks;
  if constexpr (kPopArt) {
    for (int k = threadIdx.x + threadIdx.y * blockDim.x; k < p.K; k += blockDim.x * blockDim.y) {
      const double mu = p.pa_mu[k];
      sMu[k] = float(mu);
      sSig[k] = float(popart_sigma(mu, p.pa_nu[k]));
    }
    __syncthreads();
  }
  // PopArt: the unnormalised value of row t of column b (t == T: the bootstrap value); an out-of-range task id reads 0
  auto pop_value = [&](int64_t t, int64_t b) -> float {
    const int64_t k = p.task[t * p.B + b];
    return (k >= 0 && k < p.K) ? sSig[k] * p.values[(t * p.B + b) * p.K + k] + sMu[k] : 0.0f;
  };
  const int lane = threadIdx.x;
  const int w = p.wide ? 0 : threadIdx.y, W = p.wide ? 1 : blockDim.y;
  const int64_t T = p.T, B = p.B;
  const int64_t Ause = A ? A : p.A;
  const int64_t tiles = (B + kWarp - 1) / kWarp;
  const int64_t chunk = (T + W - 1) / W;
  const int64_t t0 = (int64_t(w) * chunk < T) ? int64_t(w) * chunk : T;
  const int64_t t1 = (t0 + chunk < T) ? t0 + chunk : T;
  const int64_t tile0 = p.wide ? int64_t(blockIdx.x) * blockDim.y + threadIdx.y : blockIdx.x;
  const int64_t tile_step = p.wide ? int64_t(gridDim.x) * blockDim.y : gridDim.x;
  double s_pg = 0.0, s_bl = 0.0, s_en = 0.0;

  for (int64_t tile = tile0; tile < tiles; tile += tile_step) {
    const int64_t b = tile * kWarp + lane;
    const bool active = b < B;
    float acc_in = 0.0f;
    if (W > 1) {
      float a = 1.0f, bb = 0.0f;
      if (active && t1 > t0) {
        float v_next = kPopArt ? pop_value(t1, b) : (t1 < T) ? p.values[t1 * B + b] : p.bootstrap[b];
        for (int64_t t = t1 - 1; t >= t0; --t) {
          const int64_t i = t * B + b;
          float tlp, blp;
          if constexpr (kGaussian) {
            tlp = alp_gaussian(p.tlogits + i * Ause, int(Ause / 2), gaussian_actions(p) + i * (Ause / 2));
            blp = alp_gaussian(p.blogits + i * Ause, int(Ause / 2), gaussian_actions(p) + i * (Ause / 2));
          } else if constexpr (kFactored) {
            tlp = alp_factored(p.seg, p.tlogits + i * Ause, p.actions + i * p.seg.D);
            blp = alp_factored(p.seg, p.blogits + i * Ause, p.actions + i * p.seg.D);
          } else {
            const int64_t act = p.actions[i];
            tlp = alp_row<float, A>(p.tlogits + i * Ause, Ause, act, nullptr, nullptr);
            blp = alp_row<float, A>(p.blogits + i * Ause, Ause, act, nullptr, nullptr);
          }
          const float lr = tlp - blp;
          p.talp[i] = tlp; p.balp[i] = blp; p.log_rhos[i] = lr;
          const float rho = kTrust ? trust_rho<A, kFactored, kGaussian>(p, i, Ause, lr, false) : expf(lr);  // kl read back in pass 3
          const float g = discount_of(p, i), r = reward_of(p, i), v = kPopArt ? pop_value(t, b) : p.values[i];
          const float rb = p.has_clip_rho ? fminf(rho, p.clip_rho) : rho;
          const float delta = rb * (r + g * v_next - v);
          const float dc = g * fminf(rho, 1.0f);
          bb = delta + dc * bb;
          a = dc * a;
          v_next = v;
        }
      }
      __syncthreads();
      sA[w * kWarp + lane] = a;
      sB[w * kWarp + lane] = bb;
      __syncthreads();
      for (int w2 = W - 1; w2 > w; --w2) acc_in = sB[w2 * kWarp + lane] + sA[w2 * kWarp + lane] * acc_in;
    }
    if (!active) continue;
    if (p.zero_tail && w == 0) {  // bootstrap row of the learner outputs gets no gradient
      if (p.grad_values) {
        if constexpr (kPopArt) {
          for (int j = 0; j < p.K; ++j) p.grad_values[(T * B + b) * p.K + j] = 0.0f;
        } else {
          p.grad_values[T * B + b] = 0.0f;
        }
      }
      if (p.grad_logits)
        for (int64_t j = 0; j < Ause; ++j) p.grad_logits[(T * B + b) * Ause + j] = 0.0f;
    }
    if (t1 <= t0) continue;
    float v_next = kPopArt ? pop_value(t1, b) : (t1 < T) ? p.values[t1 * B + b] : p.bootstrap[b];
    float vs_next = (t1 < T) ? acc_in + v_next : v_next;
    float acc = acc_in;
    for (int64_t t = t1 - 1; t >= t0; --t) {
      const int64_t i = t * B + b;
      const int64_t act = (kFactored || kGaussian) ? 0 : p.actions[i];
      const float* trow = p.tlogits + i * Ause;
      float m, logs;
      float tlp;
      if constexpr (kGaussian) tlp = alp_gaussian(trow, int(Ause / 2), gaussian_actions(p) + i * (Ause / 2));
      else if constexpr (kFactored) tlp = alp_factored(p.seg, trow, p.actions + i * p.seg.D);
      else tlp = alp_row<float, A>(trow, Ause, act, &m, &logs);
      float lr;
      if (W > 1) {
        lr = p.log_rhos[i];  // written by this same thread in pass 1
      } else {
        float blp;
        if constexpr (kGaussian) blp = alp_gaussian(p.blogits + i * Ause, int(Ause / 2), gaussian_actions(p) + i * (Ause / 2));
        else if constexpr (kFactored) blp = alp_factored(p.seg, p.blogits + i * Ause, p.actions + i * p.seg.D);
        else blp = alp_row<float, A>(p.blogits + i * Ause, Ause, act, nullptr, nullptr);
        lr = tlp - blp;
        p.talp[i] = tlp; p.balp[i] = blp; p.log_rhos[i] = lr;
      }
      const float rho = kTrust ? trust_rho<A, kFactored, kGaussian>(p, i, Ause, lr, W > 1) : expf(lr);
      const float g = discount_of(p, i), r = reward_of(p, i), v = kPopArt ? pop_value(t, b) : p.values[i];
      const float rb = p.has_clip_rho ? fminf(rho, p.clip_rho) : rho;
      const float rp = p.has_clip_pg ? fminf(rho, p.clip_pg) : rho;
      const float delta = rb * (r + g * v_next - v);
      acc = delta + (g * fminf(rho, 1.0f)) * acc;
      const float vst = acc + v;
      float adv = rp * (r + g * vs_next - v);
      p.vs[i] = vst;
      p.pg_adv[i] = adv;
      vs_next = vst;
      v_next = v;
      // losses (monobeast.py:107-125) and closed-form backward (SURVEY 8(a) A4)
      float d;
      if constexpr (kPopArt) {
        // normalised space: the policy gradient scales by 1/sigma_k, the baseline regresses n_k onto (vs - mu_k)/sigma_k;
        // a row of an out-of-range task adds no loss and gets zero gradient rows
        const int64_t k = p.task[i];
        if (k < 0 || k >= p.K) {
          if (p.grad_logits)
            for (int64_t j = 0; j < Ause; ++j) p.grad_logits[i * Ause + j] = 0.0f;
          if (p.grad_values)
            for (int j = 0; j < p.K; ++j) p.grad_values[i * p.K + j] = 0.0f;
          continue;
        }
        adv = adv / sSig[k];
        d = (vst - sMu[k]) / sSig[k] - p.values[i * p.K + k];
      } else {
        d = vst - v;
      }
      if constexpr (kWeighted) {
        const double wd = double(__ldg(p.column_weights + b));  // column b's weight, read where it is used (L1)
        s_pg += double(-tlp * adv) * wd;
        s_bl += 0.5 * double(d * d) * wd;
      } else {
        s_pg += double(-tlp * adv);
        s_bl += 0.5 * double(d * d);
      }
      float ent_row = 0.0f;
      if constexpr (kGaussian) {
        ent_row = gaussian_entropy_grad<kWeighted>(p, i, b, adv);
      } else if constexpr (kFactored) {
        ent_row = factored_entropy_grad<kWeighted>(p, i, b, adv);
      } else if constexpr (A != 0) {
        float lp[A], pr[A];
#pragma unroll
        for (int j = 0; j < A; ++j) {
          lp[j] = (trow[j] - m) - logs;
          pr[j] = expf(lp[j]);
          ent_row += pr[j] * lp[j];
        }
        if (p.grad_logits) {
#pragma unroll
          for (int j = 0; j < A; ++j) {
            const float gl = adv * (pr[j] - (act == j ? 1.0f : 0.0f)) + p.entropy_cost * pr[j] * (lp[j] - ent_row);
            if constexpr (kWeighted) p.grad_logits[i * A + j] = gl * __ldg(p.column_weights + b); else p.grad_logits[i * A + j] = gl;
          }
        }
      } else {
        for (int64_t j = 0; j < Ause; ++j) {
          const float lp = (trow[j] - m) - logs;
          ent_row += expf(lp) * lp;
        }
        if (p.grad_logits) {
          for (int64_t j = 0; j < Ause; ++j) {
            const float lp = (trow[j] - m) - logs, pr = expf(lp);
            const float gl = adv * (pr - (act == j ? 1.0f : 0.0f)) + p.entropy_cost * pr * (lp - ent_row);
            if constexpr (kWeighted) p.grad_logits[i * Ause + j] = gl * __ldg(p.column_weights + b); else p.grad_logits[i * Ause + j] = gl;
          }
        }
      }
      if constexpr (kWeighted) s_en += double(ent_row) * double(__ldg(p.column_weights + b)); else s_en += double(ent_row);
      if (p.grad_values) {
        if constexpr (kPopArt) {
          const int64_t k = p.task[i];
          for (int j = 0; j < p.K; ++j) p.grad_values[i * p.K + j] = (j == k) ? -p.baseline_cost * d : 0.0f;
        } else if constexpr (kWeighted) {
          p.grad_values[i] = (-p.baseline_cost * d) * __ldg(p.column_weights + b);
        } else {
          p.grad_values[i] = -p.baseline_cost * d;
        }
      }
    }
  }
  if constexpr (kTrust) {
    trust_finish(p, s_pg, s_bl, s_en, tile0, tile_step, t0, t1);
    return;
  }
  double tot[3];
  if (grid_sum3(s_pg, s_bl, s_en, p.workspace, tot)) {
    const double pg = tot[0], bl = double(p.baseline_cost) * tot[1], en = double(p.entropy_cost) * tot[2];
    p.losses[0] = float(pg); p.losses[1] = float(bl); p.losses[2] = float(en); p.losses[3] = float(pg + bl + en);
  }
}

// ----------------------------------------------------------------------------------------
// UPGO: upgoing policy gradient (tb_upgo_loss_f32), a second launch after impala_loss_kernel
// ----------------------------------------------------------------------------------------
// The loss's arguments (so reward_of, discount_of and load_hparams apply unchanged) plus UPGO's own.  log_rhos and kl are
// the loss launch's outputs, read here.
struct UpgoArgs : LossArgs {
  const float* upgo_cost;  // f32 [1], read when the kernel runs; 0: grad_logits and losses are not written
  float* upgo_adv;         // [T,B] out
  float* upgo_out;         // [1] out: the weighted loss
};

// The return is carried backwards as X_t = lambda_t ? G_t : V_t, X_T = V_T, so G_t = r_t + g_t X_{t+1}.  A chunk of rows
// is the affine map X_t0 = a X_t1 + bb, which is the select above when composed row by row (a = 0 after a lambda of 0),
// so the split-T layout composes it across warps as the loss kernel composes its V-trace maps.
// __maxnreg__(128) is the register ceiling of a 512-thread block, as __launch_bounds__(512) would give; under the
// latter ptxas settled on 64 registers and spilled in some instantiations.
template <int A, bool kPopArt = false, bool kWeighted = false, bool kTrust = false>
__global__ void __maxnreg__(128) upgo_loss_kernel(UpgoArgs p) {
  if (p.hp) load_hparams(p);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sA = reinterpret_cast<float*>(smem_raw);
  float* sB = sA + blockDim.y * kWarp;
  float* sMu = sB + blockDim.y * kWarp;
  float* sSig = sMu + kPopArtMaxTasks;
  if constexpr (kPopArt) {
    for (int k = threadIdx.x + threadIdx.y * blockDim.x; k < p.K; k += blockDim.x * blockDim.y) {
      const double mu = p.pa_mu[k];
      sMu[k] = float(mu);
      sSig[k] = float(popart_sigma(mu, p.pa_nu[k]));
    }
    __syncthreads();
  }
  const int64_t T = p.T, B = p.B;
  // V_t of column b, t == T: the bootstrap value (PopArt: unnormalised as in impala_loss_kernel's pop_value)
  auto value_of = [&](int64_t t, int64_t b) -> float {
    if constexpr (kPopArt) {
      const int64_t k = p.task[t * B + b];
      return (k >= 0 && k < p.K) ? sSig[k] * p.values[(t * B + b) * p.K + k] + sMu[k] : 0.0f;
    } else {
      return t < T ? p.values[t * B + b] : p.bootstrap[b];
    }
  };
  const float cost = *p.upgo_cost;
  const int lane = threadIdx.x;
  const int w = p.wide ? 0 : threadIdx.y, W = p.wide ? 1 : blockDim.y;
  const int64_t Ause = A ? A : p.A;
  const int64_t tiles = (B + kWarp - 1) / kWarp;
  const int64_t chunk = (T + W - 1) / W;
  const int64_t t0 = (int64_t(w) * chunk < T) ? int64_t(w) * chunk : T;
  const int64_t t1 = (t0 + chunk < T) ? t0 + chunk : T;
  const int64_t tile0 = p.wide ? int64_t(blockIdx.x) * blockDim.y + threadIdx.y : blockIdx.x;
  const int64_t tile_step = p.wide ? int64_t(gridDim.x) * blockDim.y : gridDim.x;
  double s_up = 0.0;

  for (int64_t tile = tile0; tile < tiles; tile += tile_step) {
    const int64_t b = tile * kWarp + lane;
    const bool active = b < B;
    float x_in = active ? value_of(T, b) : 0.0f;  // X_T = V_T
    if (W > 1) {
      float a = 1.0f, bb = 0.0f;
      if (active && t1 > t0) {
        float v_next = value_of(t1, b);
        for (int64_t t = t1 - 1; t >= t0; --t) {
          const int64_t i = t * B + b;
          const float g = discount_of(p, i), r = reward_of(p, i), v = value_of(t, b);
          if (r + g * v_next >= v) {  // lambda_t = 1
            bb = r + g * bb;
            a = g * a;
          } else {
            bb = v;
            a = 0.0f;
          }
          v_next = v;
        }
      }
      __syncthreads();
      sA[w * kWarp + lane] = a;
      sB[w * kWarp + lane] = bb;
      __syncthreads();
      for (int w2 = W - 1; w2 > w; --w2) x_in = sB[w2 * kWarp + lane] + sA[w2 * kWarp + lane] * x_in;
    }
    if (!active || t1 <= t0) continue;
    float v_next = value_of(t1, b);
    float x = x_in;  // X_{t+1}
    for (int64_t t = t1 - 1; t >= t0; --t) {
      const int64_t i = t * B + b;
      const float g = discount_of(p, i), r = reward_of(p, i), v = value_of(t, b);
      const float G = r + g * x;
      x = (r + g * v_next >= v) ? G : v;
      v_next = v;
      float rho = expf(p.log_rhos[i]);
      if constexpr (kTrust) rho = p.kl[i] <= *p.trust_beta ? rho : 0.0f;
      const float rp = p.has_clip_pg ? fminf(rho, p.clip_pg) : rho;
      float adv = rp * (G - v);
      if constexpr (kPopArt) {
        const int64_t k = p.task[i];
        if (k < 0 || k >= p.K) {  // adds nothing
          p.upgo_adv[i] = 0.0f;
          continue;
        }
        adv = adv / sSig[k];
      }
      p.upgo_adv[i] = adv;
      const int64_t act = p.actions[i];
      const float* trow = p.tlogits + i * Ause;
      float m, logs;
      const float tlp = alp_row<float, A>(trow, Ause, act, &m, &logs);
      float scale = cost * adv;  // d loss / d logits = cost * w_b * adv * (pi - onehot)
      if constexpr (kWeighted) {
        const float wb = __ldg(p.column_weights + b);
        s_up += double(-tlp * adv) * double(wb);
        scale *= wb;
      } else {
        s_up += double(-tlp * adv);
      }
      if (p.grad_logits && cost != 0.0f) {
        // the row is re-read (L1) rather than kept in registers from alp_row
        float* grow = p.grad_logits + i * Ause;
#pragma unroll
        for (int64_t j = 0; j < Ause; ++j) grow[j] += scale * (expf((trow[j] - m) - logs) - (act == j ? 1.0f : 0.0f));
      }
    }
  }
  double tot[3];
  if (grid_sum3(s_up, 0.0, 0.0, p.workspace, tot)) {
    const float up = float(double(cost) * tot[0]);
    p.upgo_out[0] = up;
    if (cost != 0.0f) p.losses[3] = float(double(p.losses[3]) + double(up));
  }
}

// ----------------------------------------------------------------------------------------
// Kickstarting: KL(teacher || learner) per row (tb_kickstart_loss_f32), a launch after the loss (and UPGO)
// ----------------------------------------------------------------------------------------
struct KickstartArgs {
  const float* teacher; const float* target;  // [T,B,A] each
  int64_t T, B, A;
  const float* column_weights;                // [B] or NULL (kickstart_loss_kernel<A, true> only)
  const float* cost;                          // f32 [1], read when the kernel runs; 0: grad and losses not written
  float* out;                                 // [2] out: {cost * sum w_b KL_t, sum KL_t}
  float* losses;                              // [4]: losses[3] += out[0]
  float* grad;                                // [T(+1),B,A] or NULL: rows t < T += cost w_b (p_S - p_T)
  void* workspace;
};

// KL_t = sum_a p_T(a) (log p_T(a) - log p_S(a)) of one row in fp32, with both log-softmaxes from the max / log-sum-exp
// the loss uses; a term with p_T(a) == 0 adds exactly 0 (a -inf teacher logit), a NaN one propagates.  With `grow` the
// gradient scale * (p_S - p_T) is added into it.
template <int A>
__device__ __forceinline__ float kickstart_row(const float* __restrict__ trow, const float* __restrict__ srow,
                                               int64_t Ause, float* __restrict__ grow, float scale) {
  float kl = 0.0f;
  if constexpr (A == 0) {
    float mt, logst, ms, logss;
    alp_dyn<float>(trow, Ause, 0, &mt, &logst);
    alp_dyn<float>(srow, Ause, 0, &ms, &logss);
    for (int64_t j = 0; j < Ause; ++j) {
      const float lt = (trow[j] - mt) - logst, ls = (srow[j] - ms) - logss, pt = expf(lt);
      kl += pt == 0.0f ? 0.0f : pt * (lt - ls);
      if (grow) grow[j] += scale * (expf(ls) - pt);
    }
  } else {
    float xt[A], xs[A], mt, logst, ms, logss;
    RowOps<float, A>::load(trow, Ause, xt);
    RowOps<float, A>::load(srow, Ause, xs);
    RowOps<float, A>::lse(xt, mt, logst);
    RowOps<float, A>::lse(xs, ms, logss);
#pragma unroll
    for (int j = 0; j < A; ++j) {
      const float lt = (xt[j] - mt) - logst, ls = (xs[j] - ms) - logss, pt = expf(lt);
      kl += pt == 0.0f ? 0.0f : pt * (lt - ls);
      if (grow) grow[j] += scale * (expf(ls) - pt);
    }
  }
  return kl;
}

// Rows are independent: a grid-stride loop over the T*B rows, then one grid_sum3 of {sum w_b KL_t, sum KL_t}.
// kWeighted: row (t, b)'s loss and gradient are multiplied by column_weights[b]; the other instantiations compile none.
template <int A, bool kWeighted>
__global__ void __launch_bounds__(256) kickstart_loss_kernel(KickstartArgs p) {
  const float cost = *p.cost;
  const int64_t Ause = A ? A : p.A;
  const int64_t N = p.T * p.B;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  double s_w = 0.0, s_kl = 0.0;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    float scale = cost;
    if constexpr (kWeighted) scale *= __ldg(p.column_weights + i % p.B);
    float* grow = (p.grad && cost != 0.0f) ? p.grad + i * Ause : nullptr;
    const float kl = kickstart_row<A>(p.teacher + i * Ause, p.target + i * Ause, Ause, grow, scale);
    s_kl += double(kl);
    if constexpr (kWeighted) s_w += double(kl) * double(__ldg(p.column_weights + i % p.B)); else s_w += double(kl);
  }
  double tot[3];
  if (grid_sum3(s_w, s_kl, 0.0, p.workspace, tot)) {
    const float ks = float(double(cost) * tot[0]);
    p.out[0] = ks;
    p.out[1] = float(tot[1]);
    if (cost != 0.0f) p.losses[3] = float(double(p.losses[3]) + double(ks));
  }
}

// ----------------------------------------------------------------------------------------
// PopArt statistics
// ----------------------------------------------------------------------------------------
// sums[k] = count, sums[K+k] = sum vs, sums[2K+k] = sum vs^2 over the rows t < T of task k.  CTA k owns task k and
// walks every row in a fixed pattern (thread j takes rows j, j+256, ...; warps then CTA folded in index order), so the
// sums are bit-identical from run to run without atomics.  The rows are the loss kernel's vs output, still in L2.
constexpr int kPopArtStatsThreads = 256;
__global__ void __launch_bounds__(kPopArtStatsThreads) popart_task_sums_kernel(const float* __restrict__ vs,
                                                                                const int64_t* __restrict__ task,
                                                                                int64_t N, int K, double* __restrict__ sums) {
  __shared__ double sm[kPopArtStatsThreads / kWarp][3];
  const int k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double c = 0.0, s = 0.0, s2 = 0.0;
  for (int64_t i = tid; i < N; i += kPopArtStatsThreads) {
    if (__ldg(task + i) == k) {
      const double x = double(__ldg(vs + i));
      c += 1.0; s += x; s2 += x * x;
    }
  }
  c = warp_sum(c); s = warp_sum(s); s2 = warp_sum(s2);
  if (lane == 0) { sm[warp][0] = c; sm[warp][1] = s; sm[warp][2] = s2; }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0, d = 0.0;
    for (int w = 0; w < kPopArtStatsThreads / kWarp; ++w) { a += sm[w][0]; b += sm[w][1]; d += sm[w][2]; }
    sums[k] = a; sums[K + k] = b; sums[2 * K + k] = d;
  }
}

// Statistics update and output-preserving rescale of the value head, CTA k for task k.  A task without rows keeps
// its statistics and its head row.
__global__ void popart_update_kernel(const double* __restrict__ sums, const double* __restrict__ beta, double* mu,
                                     double* nu, int K, float* __restrict__ weight, float* __restrict__ bias, int64_t F) {
  __shared__ double s_scale, s_mu, s_mu_new, s_sig, s_sig_new;
  __shared__ bool s_skip;
  const int k = blockIdx.x;
  if (threadIdx.x == 0) {
    const double n = sums[k];
    s_skip = !(n > 0.0);
    if (!s_skip) {
      const double b = *beta, m = mu[k], v = nu[k];
      const double m2 = (1.0 - b) * m + b * (sums[K + k] / n);
      const double v2 = (1.0 - b) * v + b * (sums[2 * K + k] / n);
      s_mu = m; s_mu_new = m2;
      s_sig = popart_sigma(m, v); s_sig_new = popart_sigma(m2, v2);
      s_scale = s_sig / s_sig_new;
      mu[k] = m2; nu[k] = v2;
    }
  }
  __syncthreads();
  if (s_skip) return;
  float* row = weight + int64_t(k) * F;
  for (int64_t f = threadIdx.x; f < F; f += blockDim.x) row[f] = float(double(row[f]) * s_scale);
  if (threadIdx.x == 0) bias[k] = float((s_sig * double(bias[k]) + s_mu - s_mu_new) / s_sig_new);
}

// ----------------------------------------------------------------------------------------
// stand-alone loss functions (API mirror of compute_*_loss; F = float or double)
// ----------------------------------------------------------------------------------------
template <typename F>
__global__ void baseline_loss_kernel(const F* __restrict__ adv, int64_t N, F* out, F* grad, void* ws) {
  double s = 0.0;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const F a = adv[i];
    s += 0.5 * double(a) * double(a);
    if (grad) grad[i] = a;
  }
  double tot[3];
  if (grid_sum3(s, 0.0, 0.0, ws, tot)) out[0] = F(tot[0]);
}

template <typename F>
__global__ void entropy_loss_kernel(const F* __restrict__ logits, int64_t N, int64_t A, F* out, F* grad, void* ws) {
  double s = 0.0;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const F* row = logits + i * A;
    F m, logs;
    alp_dyn<F>(row, A, 0, &m, &logs);
    F ent = F(0);
    for (int64_t j = 0; j < A; ++j) { const F lp = (row[j] - m) - logs; ent += M<F>::exp(lp) * lp; }
    s += double(ent);
    if (grad)
      for (int64_t j = 0; j < A; ++j) { const F lp = (row[j] - m) - logs; grad[i * A + j] = M<F>::exp(lp) * (lp - ent); }
  }
  double tot[3];
  if (grid_sum3(s, 0.0, 0.0, ws, tot)) out[0] = F(tot[0]);
}

template <typename F>
__global__ void pg_loss_kernel(const F* __restrict__ logits, const int64_t* __restrict__ actions,
                               const F* __restrict__ adv, int64_t N, int64_t A, F* out, F* grad, void* ws) {
  double s = 0.0;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const F* row = logits + i * A;
    const int64_t a = actions[i];
    F m, logs;
    const F lpa = alp_dyn<F>(row, A, a, &m, &logs);
    const F ad = adv[i];
    s += double(-lpa * ad);
    if (grad)
      for (int64_t j = 0; j < A; ++j) grad[i * A + j] = ad * (M<F>::exp((row[j] - m) - logs) - (j == a ? F(1) : F(0)));
  }
  double tot[3];
  if (grid_sum3(s, 0.0, 0.0, ws, tot)) out[0] = F(tot[0]);
}

// What a loss row means: a flat categorical, a factored one (p.seg) or a diagonal Gaussian (gaussian_actions).
enum class RowKind { kFlat, kFactored, kGaussian };

// One fused-loss launch: the flat kernel of the row width p.A (TB_DISPATCH_A), or the dynamic-A kernel of a factored or
// Gaussian row.
template <bool kPopArt, bool kWeighted, bool kTrust>
static void launch_loss_kernel(const LossArgs& p, RowKind kind, dim3 grid, dim3 block, size_t smem, cudaStream_t st) {
  if (kind == RowKind::kFactored)
    impala_loss_kernel<0, kPopArt, kWeighted, kTrust, true><<<grid, block, smem, st>>>(p);
  else if (kind == RowKind::kGaussian)
    impala_loss_kernel<kGaussianRows, kPopArt, kWeighted, kTrust><<<grid, block, smem, st>>>(p);
  else
    TB_DISPATCH_A(p.A, (impala_loss_kernel<kA, kPopArt, kWeighted, kTrust><<<grid, block, smem, st>>>(p)));
}

// tb_impala_loss_f32, with seg non-NULL tb_impala_loss_factored_f32, and with gactions non-NULL (actions then NULL)
// tb_impala_loss_gaussian_f32.  The kernel instantiation follows from which of column_weights, task and trust_beta are
// non-NULL.
static int impala_loss(const float* blogits, const float* tlogits, const int64_t* actions, const float* rewards,
                       const uint8_t* done, const float* discounts, const float* values, const float* bootstrap,
                       int64_t T, int64_t B, int64_t A, float discounting, float baseline_cost, float entropy_cost,
                       int clip_rewards, float clip_rho, float clip_pg_rho, const tb_hparams* hp,
                       const float* column_weights, const int64_t* task, const double* mu, const double* nu,
                       int64_t K, double* task_sums, const float* trust_beta, float* kl_out, float* trust_out,
                       float* vs, float* pg_adv, float* log_rhos, float* behavior_alp, float* target_alp,
                       float* losses_out, float* grad_logits, float* grad_values, int zero_tail, void* workspace,
                       void* stream, const ActionSegments* seg, const float* gactions = nullptr) {

  if (task) {
    TB_REQUIRE(!column_weights, "impala_loss_popart: column_weights are not supported with PopArt (task)");
    TB_REQUIRE(T >= 1 && B >= 1 && A >= 1, "impala_loss_popart: bad sizes T=%lld B=%lld A=%lld", (long long)T,
               (long long)B, (long long)A);
    TB_REQUIRE(K >= 1 && K <= kPopArtMaxTasks, "impala_loss_popart: num_tasks %lld outside [1, %d]", (long long)K,
               kPopArtMaxTasks);
    TB_REQUIRE(values && mu && nu && task_sums, "impala_loss_popart: null PopArt pointer");
    TB_REQUIRE(zero_tail == 1, "impala_loss_popart: zero_tail must be 1");
    bootstrap = values;  // not read: the bootstrap row is row T of values
  }
  TB_REQUIRE(T >= 0 && B >= 0 && A >= 1, "impala_loss: bad sizes T=%lld B=%lld A=%lld", (long long)T,
             (long long)B, (long long)A);
  TB_REQUIRE(losses_out && workspace, "impala_loss: losses_out/workspace must not be null");
  TB_REQUIRE(!trust_beta || (kl_out && trust_out), "impala_loss_trust: kl_out/trust_out must not be null");
  if (T == 0 || B == 0) {
    cudaError_t e = cudaMemsetAsync(losses_out, 0, 4 * sizeof(float), (cudaStream_t)stream);
    TB_REQUIRE(e == cudaSuccess, "impala_loss: memset: %s", cudaGetErrorString(e));
    if (trust_beta) {
      e = cudaMemsetAsync(trust_out, 0, 2 * sizeof(float), (cudaStream_t)stream);
      TB_REQUIRE(e == cudaSuccess, "impala_loss_trust: memset: %s", cudaGetErrorString(e));
    }
    if (B > 0 && zero_tail) {
      if (grad_values) cudaMemsetAsync(grad_values, 0, B * sizeof(float), (cudaStream_t)stream);
      if (grad_logits) cudaMemsetAsync(grad_logits, 0, B * A * sizeof(float), (cudaStream_t)stream);
    }
    return 0;
  }
  TB_REQUIRE(blogits && tlogits && (actions || gactions) && rewards && (done || discounts) && values && bootstrap,
             "impala_loss: null input pointer");
  TB_REQUIRE(vs && pg_adv && log_rhos && behavior_alp && target_alp, "impala_loss: null output pointer");
  LossArgs p;
  p.blogits = blogits; p.tlogits = tlogits; p.rewards = rewards; p.done = done;
  p.actions = gactions ? reinterpret_cast<const int64_t*>(gactions) : actions;
  p.discounts = discounts; p.values = values; p.bootstrap = bootstrap; p.T = T; p.B = B; p.A = A;
  p.discounting = discounting; p.baseline_cost = baseline_cost; p.entropy_cost = entropy_cost;
  p.clip_rewards = clip_rewards; p.clip_rho = clip_rho; p.clip_pg = clip_pg_rho;
  p.has_clip_rho = (clip_rho >= 0.0f); p.has_clip_pg = (clip_pg_rho >= 0.0f);
  p.vs = vs; p.pg_adv = pg_adv; p.log_rhos = log_rhos; p.balp = behavior_alp; p.talp = target_alp;
  p.losses = losses_out; p.grad_logits = grad_logits; p.grad_values = grad_values; p.zero_tail = zero_tail;
  p.workspace = workspace;
  p.hp = hp;
  p.task = task; p.pa_mu = mu; p.pa_nu = nu; p.K = int(K);
  p.column_weights = column_weights;
  p.trust_beta = trust_beta; p.kl = kl_out; p.trust_out = trust_out;
  if (seg) p.seg = *seg;
  const RowKind kind = seg ? RowKind::kFactored : gactions ? RowKind::kGaussian : RowKind::kFlat;
  const int64_t tiles = (B + kWarp - 1) / kWarp;
  int W = pick_warps(T, tiles);
  p.wide = (W == 1);
  dim3 grid(pick_grid(tiles));
  if (p.wide) {
    W = kWideWarps;
    int64_t g = (tiles + W - 1) / W;
    if (g > kMaxPartialCtas) g = kMaxPartialCtas;  // per-CTA loss partials live in the workspace
    grid = dim3((unsigned)(g < 1 ? 1 : g));
  }
  dim3 block(kWarp, W);
  const size_t smem = size_t(2) * W * kWarp * sizeof(float);
  if (task) {
    ProfScope prof(trust_beta ? "impala_loss_popart_trust" : "impala_loss_popart", (cudaStream_t)stream);
    const size_t pop_smem = smem + size_t(2) * kPopArtMaxTasks * sizeof(float);
    if (trust_beta) {
      launch_loss_kernel<true, false, true>(p, kind, grid, block, pop_smem, (cudaStream_t)stream);
      TB_TRY(check_launch("impala_loss_kernel<popart, trust>"));
    } else {
      launch_loss_kernel<true, false, false>(p, kind, grid, block, pop_smem, (cudaStream_t)stream);
      TB_TRY(check_launch("impala_loss_kernel<popart>"));
    }
    popart_task_sums_kernel<<<unsigned(K), kPopArtStatsThreads, 0, (cudaStream_t)stream>>>(vs, task, T * B, int(K),
                                                                                       task_sums);
    return check_launch("popart_task_sums_kernel");
  }
  if (trust_beta) {
    ProfScope prof("impala_loss_trust", (cudaStream_t)stream);
    if (column_weights) {
      launch_loss_kernel<false, true, true>(p, kind, grid, block, smem, (cudaStream_t)stream);
      return check_launch("impala_loss_kernel<weighted, trust>");
    }
    launch_loss_kernel<false, false, true>(p, kind, grid, block, smem, (cudaStream_t)stream);
    return check_launch("impala_loss_kernel<trust>");
  }
  if (column_weights) {
    ProfScope prof("impala_loss_weighted", (cudaStream_t)stream);
    launch_loss_kernel<false, true, false>(p, kind, grid, block, smem, (cudaStream_t)stream);
    return check_launch("impala_loss_kernel<weighted>");
  }
  ProfScope prof("impala_loss_fwd_bwd", (cudaStream_t)stream);
  launch_loss_kernel<false, false, false>(p, kind, grid, block, smem, (cudaStream_t)stream);
  return check_launch("impala_loss_kernel");
}

static int reduce_grid(int64_t N, int threads) {
  int64_t blocks = (N + threads - 1) / threads;
  const int64_t cap = int64_t(sm_count()) * 4;
  if (blocks > cap) blocks = cap;
  if (blocks > kMaxPartialCtas) blocks = kMaxPartialCtas;
  return int(blocks < 1 ? 1 : blocks);
}

}  // namespace tb

// ========================================================================================
// C ABI
// ========================================================================================
using namespace tb;

extern "C" {

int tb_action_log_probs_f32(const float* l, const int64_t* a, int64_t N, int64_t A, float* o, void* s) {
  return launch_alp<float>(l, a, N, A, o, s);
}
int tb_action_log_probs_f64(const double* l, const int64_t* a, int64_t N, int64_t A, double* o, void* s) {
  return launch_alp<double>(l, a, N, A, o, s);
}

int tb_vtrace_from_importance_weights_f32(const float* lr, const float* d, const float* r, const float* v,
                                          const float* bs, int64_t T, int64_t B, float c1, float c2,
                                          float* vs, float* pg, void* s) {
  return launch_scan<float>(lr, d, r, v, bs, T, B, c1, c2, vs, pg, s);
}
int tb_vtrace_from_importance_weights_f64(const double* lr, const double* d, const double* r, const double* v,
                                          const double* bs, int64_t T, int64_t B, double c1, double c2,
                                          double* vs, double* pg, void* s) {
  return launch_scan<double>(lr, d, r, v, bs, T, B, c1, c2, vs, pg, s);
}

int tb_impala_loss_f32(const float* blogits, const float* tlogits, const int64_t* actions, const float* rewards,
                       const uint8_t* done, const float* discounts, const float* values, const float* bootstrap,
                       int64_t T, int64_t B, int64_t A, float discounting, float baseline_cost, float entropy_cost,
                       int clip_rewards, float clip_rho, float clip_pg_rho, const tb_hparams* hp,
                       const float* column_weights, const int64_t* task, const double* mu, const double* nu,
                       int64_t K, double* task_sums, const float* trust_beta, float* kl_out, float* trust_out,
                       float* vs, float* pg_adv, float* log_rhos, float* behavior_alp, float* target_alp,
                       float* losses_out, float* grad_logits, float* grad_values, int zero_tail, void* workspace,
                       void* stream) {
  return impala_loss(blogits, tlogits, actions, rewards, done, discounts, values, bootstrap, T, B, A, discounting,
                     baseline_cost, entropy_cost, clip_rewards, clip_rho, clip_pg_rho, hp, column_weights, task, mu, nu,
                     K, task_sums, trust_beta, kl_out, trust_out, vs, pg_adv, log_rhos, behavior_alp, target_alp,
                     losses_out, grad_logits, grad_values, zero_tail, workspace, stream, nullptr);
}

int tb_impala_loss_factored_f32(const float* blogits, const float* tlogits, const int64_t* actions,
                                const float* rewards, const uint8_t* done, const float* discounts, const float* values,
                                const float* bootstrap, int64_t T, int64_t B, int64_t A, float discounting,
                                float baseline_cost, float entropy_cost, int clip_rewards, float clip_rho,
                                float clip_pg_rho, const tb_hparams* hp, const float* column_weights,
                                const int64_t* task, const double* mu, const double* nu, int64_t K, double* task_sums,
                                const float* trust_beta, float* kl_out, float* trust_out, float* vs, float* pg_adv,
                                float* log_rhos, float* behavior_alp, float* target_alp, float* losses_out,
                                float* grad_logits, float* grad_values, int zero_tail, const tb_action_space* space,
                                void* workspace, void* stream) {
  ActionSegments seg;
  TB_TRY(action_segments(space, A, "impala_loss_factored", &seg));
  return impala_loss(blogits, tlogits, actions, rewards, done, discounts, values, bootstrap, T, B, A, discounting,
                     baseline_cost, entropy_cost, clip_rewards, clip_rho, clip_pg_rho, hp, column_weights, task, mu, nu,
                     K, task_sums, trust_beta, kl_out, trust_out, vs, pg_adv, log_rhos, behavior_alp, target_alp,
                     losses_out, grad_logits, grad_values, zero_tail, workspace, stream, &seg);
}

int tb_impala_loss_gaussian_f32(const float* blogits, const float* tlogits, const float* actions, const float* rewards,
                                const uint8_t* done, const float* discounts, const float* values, const float* bootstrap,
                                int64_t T, int64_t B, int64_t A, float discounting, float baseline_cost,
                                float entropy_cost, int clip_rewards, float clip_rho, float clip_pg_rho,
                                const tb_hparams* hp, const float* column_weights, const int64_t* task, const double* mu,
                                const double* nu, int64_t K, double* task_sums, const float* trust_beta, float* kl_out,
                                float* trust_out, float* vs, float* pg_adv, float* log_rhos, float* behavior_alp,
                                float* target_alp, float* losses_out, float* grad_logits, float* grad_values,
                                int zero_tail, void* workspace, void* stream) {
  TB_REQUIRE(A >= 2 && A % 2 == 0 && A / 2 <= TB_MAX_CONTINUOUS_DIM,
             "impala_loss_gaussian: A = %lld must be 2D with 1 <= D <= %d", (long long)A, TB_MAX_CONTINUOUS_DIM);
  TB_REQUIRE(actions || T == 0 || B == 0, "impala_loss_gaussian: null actions");
  return impala_loss(blogits, tlogits, nullptr, rewards, done, discounts, values, bootstrap, T, B, A, discounting,
                     baseline_cost, entropy_cost, clip_rewards, clip_rho, clip_pg_rho, hp, column_weights, task, mu, nu,
                     K, task_sums, trust_beta, kl_out, trust_out, vs, pg_adv, log_rhos, behavior_alp, target_alp,
                     losses_out, grad_logits, grad_values, zero_tail, workspace, stream, nullptr, actions);
}

// The kernel instantiation follows from which of column_weights, task and trust_beta are non-NULL, as in the loss.
int tb_upgo_loss_f32(const float* tlogits, const int64_t* actions, const float* rewards, const uint8_t* done,
                     const float* discounts, const float* values, const float* bootstrap, int64_t T, int64_t B,
                     int64_t A, float discounting, int clip_rewards, float clip_pg_rho, const tb_hparams* hp,
                     const float* column_weights, const int64_t* task, const double* mu, const double* nu, int64_t K,
                     const float* log_rhos, const float* trust_beta, const float* kl, const float* upgo_cost,
                     float* upgo_adv, float* upgo_out, float* losses_out, float* grad_logits, void* workspace,
                     void* stream) {
  if (task) {
    TB_REQUIRE(!column_weights, "upgo_loss_popart: column_weights are not supported with PopArt (task)");
    TB_REQUIRE(T >= 1 && B >= 1, "upgo_loss_popart: bad sizes T=%lld B=%lld", (long long)T, (long long)B);
    TB_REQUIRE(K >= 1 && K <= kPopArtMaxTasks, "upgo_loss_popart: num_tasks %lld outside [1, %d]", (long long)K,
               kPopArtMaxTasks);
    TB_REQUIRE(values && mu && nu, "upgo_loss_popart: null PopArt pointer");
    bootstrap = values;  // not read: the bootstrap row is row T of values
  }
  TB_REQUIRE(T >= 0 && B >= 0 && A >= 1, "upgo_loss: bad sizes T=%lld B=%lld A=%lld", (long long)T, (long long)B,
             (long long)A);
  TB_REQUIRE(upgo_cost && upgo_out && losses_out && workspace,
             "upgo_loss: upgo_cost/upgo_out/losses_out/workspace must not be null");
  TB_REQUIRE(!trust_beta || kl, "upgo_loss_trust: kl must not be null");
  if (T == 0 || B == 0) {
    cudaError_t e = cudaMemsetAsync(upgo_out, 0, sizeof(float), (cudaStream_t)stream);
    TB_REQUIRE(e == cudaSuccess, "upgo_loss: memset: %s", cudaGetErrorString(e));
    return 0;
  }
  TB_REQUIRE(tlogits && actions && rewards && (done || discounts) && values && bootstrap && log_rhos,
             "upgo_loss: null input pointer");
  TB_REQUIRE(upgo_adv, "upgo_loss: upgo_adv must not be null");
  UpgoArgs p = {};
  p.tlogits = tlogits; p.actions = actions; p.rewards = rewards; p.done = done; p.discounts = discounts;
  p.values = values; p.bootstrap = bootstrap; p.T = T; p.B = B; p.A = A;
  p.discounting = discounting; p.clip_rewards = clip_rewards; p.clip_pg = clip_pg_rho;
  p.has_clip_pg = (clip_pg_rho >= 0.0f);
  p.log_rhos = const_cast<float*>(log_rhos);  // read only
  p.losses = losses_out; p.grad_logits = grad_logits; p.workspace = workspace; p.hp = hp;
  p.task = task; p.pa_mu = mu; p.pa_nu = nu; p.K = int(K);
  p.column_weights = column_weights;
  p.trust_beta = trust_beta; p.kl = const_cast<float*>(kl);  // read only
  p.upgo_cost = upgo_cost; p.upgo_adv = upgo_adv; p.upgo_out = upgo_out;
  const int64_t tiles = (B + kWarp - 1) / kWarp;
  int W = pick_warps(T, tiles);
  p.wide = (W == 1);
  dim3 grid(pick_grid(tiles));
  if (p.wide) {
    W = kWideWarps;
    int64_t g = (tiles + W - 1) / W;
    if (g > kMaxPartialCtas) g = kMaxPartialCtas;
    grid = dim3((unsigned)(g < 1 ? 1 : g));
  }
  dim3 block(kWarp, W);
  const size_t smem = size_t(2) * W * kWarp * sizeof(float);
  const cudaStream_t s = (cudaStream_t)stream;
  if (task) {
    ProfScope prof(trust_beta ? "upgo_loss_popart_trust" : "upgo_loss_popart", s);
    const size_t pop_smem = smem + size_t(2) * kPopArtMaxTasks * sizeof(float);
    if (trust_beta) {
      TB_DISPATCH_A(A, (upgo_loss_kernel<kA, true, false, true><<<grid, block, pop_smem, s>>>(p)));
      return check_launch("upgo_loss_kernel<popart, trust>");
    }
    TB_DISPATCH_A(A, (upgo_loss_kernel<kA, true><<<grid, block, pop_smem, s>>>(p)));
    return check_launch("upgo_loss_kernel<popart>");
  }
  if (trust_beta) {
    ProfScope prof("upgo_loss_trust", s);
    if (column_weights) {
      TB_DISPATCH_A(A, (upgo_loss_kernel<kA, false, true, true><<<grid, block, smem, s>>>(p)));
      return check_launch("upgo_loss_kernel<weighted, trust>");
    }
    TB_DISPATCH_A(A, (upgo_loss_kernel<kA, false, false, true><<<grid, block, smem, s>>>(p)));
    return check_launch("upgo_loss_kernel<trust>");
  }
  if (column_weights) {
    ProfScope prof("upgo_loss_weighted", s);
    TB_DISPATCH_A(A, (upgo_loss_kernel<kA, false, true><<<grid, block, smem, s>>>(p)));
    return check_launch("upgo_loss_kernel<weighted>");
  }
  ProfScope prof("upgo_loss", s);
  TB_DISPATCH_A(A, (upgo_loss_kernel<kA><<<grid, block, smem, s>>>(p)));
  return check_launch("upgo_loss_kernel");
}

// The kernel instantiation follows from whether column_weights is non-NULL.
int tb_kickstart_loss_f32(const float* teacher_logits, const float* target_logits, int64_t T, int64_t B, int64_t A,
                          const float* column_weights, const float* kickstart_cost, float* kickstart_out,
                          float* losses_out, float* grad_logits, void* workspace, void* stream) {
  TB_REQUIRE(T >= 1 && B >= 1 && A >= 1, "kickstart_loss: bad sizes T=%lld B=%lld A=%lld", (long long)T,
             (long long)B, (long long)A);
  TB_REQUIRE(teacher_logits && target_logits, "kickstart_loss: null input pointer");
  TB_REQUIRE(kickstart_cost && kickstart_out && losses_out && workspace,
             "kickstart_loss: kickstart_cost/kickstart_out/losses_out/workspace must not be null");
  KickstartArgs p;
  p.teacher = teacher_logits; p.target = target_logits; p.T = T; p.B = B; p.A = A;
  p.column_weights = column_weights; p.cost = kickstart_cost; p.out = kickstart_out; p.losses = losses_out;
  p.grad = grad_logits; p.workspace = workspace;
  const int threads = 256;
  int64_t blocks = (T * B + threads - 1) / threads;
  const int64_t cap = int64_t(sm_count()) * 8 < kMaxPartialCtas ? int64_t(sm_count()) * 8 : kMaxPartialCtas;
  if (blocks > cap) blocks = cap;
  const cudaStream_t s = (cudaStream_t)stream;
  if (column_weights) {
    ProfScope prof("kickstart_loss_weighted", s);
    TB_DISPATCH_A(A, (kickstart_loss_kernel<kA, true><<<unsigned(blocks), threads, 0, s>>>(p)));
    return check_launch("kickstart_loss_kernel<weighted>");
  }
  ProfScope prof("kickstart_loss", s);
  TB_DISPATCH_A(A, (kickstart_loss_kernel<kA, false><<<unsigned(blocks), threads, 0, s>>>(p)));
  return check_launch("kickstart_loss_kernel");
}

int tb_popart_update(const double* task_sums, const double* beta, double* mu, double* nu, int64_t K, float* weight,
                     float* bias, int64_t F, void* stream) {
  TB_REQUIRE(K >= 1 && K <= kPopArtMaxTasks && F >= 1, "popart_update: bad sizes K=%lld F=%lld", (long long)K,
             (long long)F);
  TB_REQUIRE(task_sums && beta && mu && nu && weight && bias, "popart_update: null pointer");
  ProfScope prof("popart_update", (cudaStream_t)stream);
  popart_update_kernel<<<unsigned(K), 128, 0, (cudaStream_t)stream>>>(task_sums, beta, mu, nu, int(K), weight, bias, F);
  return check_launch("popart_update_kernel");
}

#define TB_LOSS_ENTRY(NAME, F, KERNEL, ARGS_DECL, ARGS_CALL, NEXPR)                                     \
  int NAME ARGS_DECL {                                                                                  \
    TB_REQUIRE(out && workspace, #NAME ": out/workspace must not be null");                            \
    const int threads = 256;                                                                            \
    const int blocks = reduce_grid((NEXPR), threads);                                                   \
    KERNEL<F><<<blocks, threads, 0, (cudaStream_t)stream>>> ARGS_CALL;                                  \
    return check_launch(#NAME);                                                                         \
  }

TB_LOSS_ENTRY(tb_baseline_loss_f32, float, baseline_loss_kernel,
              (const float* adv, int64_t N, float* out, float* grad, void* workspace, void* stream),
              (adv, N, out, grad, workspace), N)
TB_LOSS_ENTRY(tb_baseline_loss_f64, double, baseline_loss_kernel,
              (const double* adv, int64_t N, double* out, double* grad, void* workspace, void* stream),
              (adv, N, out, grad, workspace), N)
TB_LOSS_ENTRY(tb_entropy_loss_f32, float, entropy_loss_kernel,
              (const float* logits, int64_t N, int64_t A, float* out, float* grad, void* workspace, void* stream),
              (logits, N, A, out, grad, workspace), N)
TB_LOSS_ENTRY(tb_entropy_loss_f64, double, entropy_loss_kernel,
              (const double* logits, int64_t N, int64_t A, double* out, double* grad, void* workspace, void* stream),
              (logits, N, A, out, grad, workspace), N)
TB_LOSS_ENTRY(tb_pg_loss_f32, float, pg_loss_kernel,
              (const float* logits, const int64_t* actions, const float* adv, int64_t N, int64_t A, float* out,
               float* grad, void* workspace, void* stream),
              (logits, actions, adv, N, A, out, grad, workspace), N)
TB_LOSS_ENTRY(tb_pg_loss_f64, double, pg_loss_kernel,
              (const double* logits, const int64_t* actions, const double* adv, int64_t N, int64_t A, double* out,
               double* grad, void* workspace, void* stream),
              (logits, actions, adv, N, A, out, grad, workspace), N)

}  // extern "C"
