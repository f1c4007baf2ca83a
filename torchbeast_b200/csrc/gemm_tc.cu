// bf16 tensor-core GEMM for sm_90a: wgmma.mma_async + register accumulators + TMA-staged operands.
//
//   C[M,N] = epilogue( sum_k A[m,k] * B[n,k] )     A [M,K], B [N,K] bf16, K contiguous ("K-major")
//
// One CTA computes a 128 x BLOCK_N tile.  Warp roles (160 threads):
//   warp 4     TMA producer : cp.async.bulk.tensor.2d (SWIZZLE_128B boxes of 64 bf16 = 128 B) into a
//                             shared-memory ring, mbarrier expect_tx / complete_tx
//   warps 0-3  consumer     : one warpgroup issues wgmma.m64nNk16 (N = BLOCK_N) for both 64-row halves of
//                             the tile, x4 per 64-wide k-block, keeping one wgmma group in flight; a ring slot
//                             is handed back once the group that read it has completed.  The accumulator
//                             fragments then go through a shared-memory staging tile so that each thread owns
//                             one output row for the epilogue: scale / bias / ReLU / ReLU-mask, fp32 and/or
//                             bf16 stores
// M/N/K tails are handled by TMA out-of-bounds zero fill plus guarded stores.  Shared-memory
// matrix descriptors: K-major, SWIZZLE_128B, SBO = 1024 B (8 rows x 128 B), advanced by 32 B per
// K=16 step inside the swizzle atom (the CUTLASS/DeepGEMM canonical layout).
// Operands may also be "MN-major" (the reduction index is the ROW index in memory, A_MN / B_MN):
// the tile is then loaded as 64(k) x 64(mn) boxes, described with LBO = 8192 B between 64-wide mn
// groups and SBO = 1024 B between 8-row k groups, advanced by 2048 B per K=16 step.  That gives
//   forward  act = col . W^T      : A K-major,  B K-major
//   dgrad    dcol = dY . W        : A K-major,  B MN-major (W [n', k'] as stored)
//   wgrad    dW   = dY^T . col    : A MN-major, B MN-major (no transposed copies), split-K over grid.z
#include <cuda.h>
#include <cuda_bf16.h>

#include "gemm_tc.cuh"

#include "gemm_simt.cuh"  // splitk_reduce_kernel / GemmEpilogue
#include "tc_common.cuh"

namespace tb {

using namespace tcd;

namespace {

// Persistent: each CTA walks the work list (m tile, n tile, k split) with stride gridDim.x; the producer runs
// ahead into the next work item while the consumers run the epilogue, and the per-CTA prologue is paid once.
// EPI: 0 = store the accumulator as is; 1 = scale / bias / ReLU; 2 = + ReLU-mask / residual loads.
// (compile-time so the common epilogues carry no predicated per-element loads - ncu showed the generic
//  epilogue, not the MMA pipe, bounding the K=64 dgrad products)
// IMPL (implicit-GEMM convolution, forward): the A operand is not a matrix in memory but the NHWC activation
// itself, addressed through a rank-4 tensor map {flat frame element, ox, oy, frame} whose dimensions overlap:
// M tile t = the `rows` = OW*OH*fpt patches of frames [t*fpt, (t+1)*fpt), k-block kb = 64 consecutive
// (kw, c) elements of kernel row kb / kbw starting at element e0 of the frame - one TMA box per stage lands
// as [patch][64 k] rows in the canonical SWIZZLE_128B layout, so no patch matrix is ever written.
//
// The same machinery runs the INPUT gradient (mode 1/2) as a gather-form transposed convolution, so that
// neither the [patches, KH*KW*C] gradient matrix nor a col2im pass exists:
//   mode 1 (stride 1): dX[n,y,x,c] = sum_{kh,kw,o} dY[n,y-kh,x-kw,o] W[o,kh,kw,c]; the A tile of k-block (kh,kw) is
//     the TMA box of dY at (x0,y0) = (-kw,-kh) - out-of-bounds rows/columns arrive as zeros (the "full" padding);
//   mode 2 (stride 2, even kernel): output pixels split by parity (py,px) = (y&1, x&1): each class is a stride-1
//     conv of dY with the (KH/2 x KW/2) sub-kernel W[o, py+2i, px+2j, c].  All classes read the SAME dY boxes, so
//     they are the N dimension of one GEMM: B = [(py,px,c), (i,j,o)], and the epilogue scatters the 32-column
//     chunk of class (py,px) to pixel (2u+py, 2v+px).
struct ImplicitConv {
  int rows = 0;       // valid rows per M tile (<= 128)
  int fpt = 1;        // frames per tile
  int kbw = 1;        // k-blocks per kernel row
  int row_elems = 0;  // mode 0: W*C
  int mode = 0;       // 0 forward, 1 input gradient stride 1, 2 input gradient stride 2 (parity classes)
  int tw = 0;         // mode 2: tile width (v range) = ceil(W_in / 2)
  int outH = 0, outW = 0;  // mode 2: input-gradient image size
};

// SPLIT (split-bf16, see TcEpilogue): a stage holds the hi AND lo plane tiles of both operands (tmAl / tmBl are the
// lo planes' tensor maps) and every k-step issues three MMAs (lo.hi, hi.lo, hi.hi) into the same accumulator; the
// epilogue can write its bf16 output as hi / lo planes.
template <int BLOCK_N, bool A_MN, bool B_MN, int kStages, int EPI, bool IMPL = false, bool SPLIT = false>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmAl, const __grid_constant__ CUtensorMap tmBl, TcEpilogue ep, int M,
               int N, int K, float* partial, int tiles_m, int tiles_n, int splits, int ldp = 0,
               ImplicitConv ic = ImplicitConv()) {
  constexpr uint32_t B_BYTES = BLOCK_N * kBlockK * 2;
  constexpr uint32_t A_STAGE = (SPLIT ? 2u : 1u) * kABytes, B_STAGE = (SPLIT ? 2u : 1u) * B_BYTES;  // [hi][lo]
  constexpr int LDS = BLOCK_N + 4;  // staging row pitch in floats (16-byte rows, conflict-free row reads)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024 B alignment
  const uint32_t sA = base, sB = base + kStages * A_STAGE;
  const uint32_t bars = sB + kStages * B_STAGE;  // full[kStages], empty[kStages], then the accumulator staging tile
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kStages + s); };
  // [128][LDS] fp32: the epilogue reads whole rows, the wgmma fragments are scattered over row pairs
  float* stg = reinterpret_cast<float*>(smem_raw + (bars + 16u * kStages - smem_addr(smem_raw)));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_kb = (K + kBlockK - 1) / kBlockK;
  const int per = (total_kb + splits - 1) / splits;
  const int tiles_mn = tiles_m * tiles_n;
  const int total_work = tiles_mn * splits;

  if (warp == 4 && lane == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // work item -> tile coordinates (n fastest so that co-running CTAs share A tiles in L2)
  auto decode = [&](int w, int& m0, int& n0, int& kb0, int& num_kb, int& z) {
    z = w / tiles_mn;
    const int rem = w - z * tiles_mn;
    m0 = (rem / tiles_n) * kBlockM;
    n0 = (rem % tiles_n) * BLOCK_N;
    kb0 = z * per;
    const int kb1 = (kb0 + per < total_kb) ? kb0 + per : total_kb;
    num_kb = kb1 > kb0 ? kb1 - kb0 : 0;
  };

  if (warp == 4) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        int m0, n0, kb0, num_kb, z;
        decode(w, m0, n0, kb0, num_kb, z);
        for (int i = 0; i < num_kb; ++i) {
          const int kc = (kb0 + i) * kBlockK;
          mbar_wait(empty(stage), phase ^ 1);
          mbar_expect_tx(full(stage), (SPLIT ? 2u : 1u) * ((IMPL ? uint32_t(ic.rows) * 128u : kABytes) + B_BYTES));
#pragma unroll
          for (int pl = 0; pl < (SPLIT ? 2 : 1); ++pl) {  // plane 0 = hi, plane 1 = lo
            const CUtensorMap* mA = pl ? &tmAl : &tmA;
            const CUtensorMap* mB = pl ? &tmBl : &tmB;
            const uint32_t dA = sA + stage * A_STAGE + pl * kABytes, dB = sB + stage * B_STAGE + pl * B_BYTES;
            if (IMPL) {
              const int kb = kb0 + i;
              if (ic.mode == 0)
                tma_load_4d(dA, mA, full(stage), (kb / ic.kbw) * ic.row_elems + (kb % ic.kbw) * kBlockK, 0, 0,
                            (m0 / kBlockM) * ic.fpt);
              else
                tma_load_4d(dA, mA, full(stage), 0, -(kb % ic.kbw), -(kb / ic.kbw), (m0 / kBlockM) * ic.fpt);
            } else if (A_MN) {  // two 64(k) x 64(m) boxes
              tma_load_2d(dA, mA, full(stage), m0, kc);
              tma_load_2d(dA + 8192, mA, full(stage), m0 + 64, kc);
            } else {
              tma_load_2d(dA, mA, full(stage), kc, m0);
            }
            if (B_MN) {
#pragma unroll
              for (int j = 0; j < BLOCK_N / 64; ++j) tma_load_2d(dB + j * 8192, mB, full(stage), n0 + 64 * j, kc);
            } else {
              tma_load_2d(dB, mB, full(stage), kc, n0);
            }
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < 4) {
    int stage = 0; uint32_t phase = 0;
    float acc[2][BLOCK_N / 2];  // rows [0, 64) and [64, 128) of the tile
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
      int m0, n0, kb0, num_kb, z;
      decode(w, m0, n0, kb0, num_kb, z);
      const int rl = threadIdx.x;
      const int64_t r = IMPL ? int64_t(m0 / kBlockM) * ic.rows + rl : int64_t(m0) + rl;
      const bool rvalid = r < M && (!IMPL || rl < ic.rows);
      // where this thread's 32 values of column chunk c0 live in memory: row pr, first column pc (== r, n0 + c0
      // except for the parity-class scatter of the stride-2 input gradient); false = nothing to store
      auto locate = [&](int c0, int64_t& pr, int& pc) -> bool {
        pr = r; pc = n0 + c0;
        if (IMPL && ic.mode == 2) {
          const int cls = (n0 + c0) >> 5, u = rl / ic.tw, v2 = rl - u * ic.tw;
          const int y = 2 * u + (cls >> 1), x = 2 * v2 + (cls & 1);
          if (y >= ic.outH || x >= ic.outW) return false;
          pr = (int64_t(m0 / kBlockM) * ic.outH + y) * ic.outW + x;
          pc = 0;
        }
        return true;
      };
      // EPI 2: pull the ReLU-mask / residual rows of the WHOLE tile into L2 before waiting for the accumulator, so
      // their DRAM latency hides behind the MMA main loop (fetching them chunk by chunk after the wait made the
      // stride-2 input gradient - 4 chunks, 4 k-blocks - epilogue-latency bound)
      if constexpr (EPI >= 2) {
        if (rvalid) {
#pragma unroll 1
          for (int c0 = 0; c0 < BLOCK_N && n0 + c0 < N; c0 += 32) {
            int64_t pr; int pc;
            if (!locate(c0, pr, pc)) continue;
            if (ep.mask16) asm volatile("prefetch.global.L2 [%0];" ::"l"(ep.mask16 + pr * ep.ldmask + pc));
            if (ep.addend16) asm volatile("prefetch.global.L2 [%0];" ::"l"(ep.addend16 + pr * ep.ldadd + pc));
          }
        }
      }
      // main loop: one k-block per stage; a stage is handed back once the wgmma group after it has been issued and
      // its own group has completed (one group in flight)
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(full(stage), phase);
        wgmma_fence();
        const uint32_t aA = sA + stage * A_STAGE, aB = sB + stage * B_STAGE;
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          const uint64_t db = B_MN ? make_smem_desc_mn(aB + k * 2048) : make_smem_desc(aB + k * 32);
#pragma unroll
          for (int h = 0; h < 2; ++h) {  // the two 64-row halves of the tile (8192 B apart in both layouts)
            const uint32_t ah = aA + h * 8192;
            const uint64_t da = A_MN ? make_smem_desc_mn(ah + k * 2048) : make_smem_desc(ah + k * 32);
            if constexpr (SPLIT) {  // small terms first: lo.hi, hi.lo, then hi.hi
              const uint64_t dal = A_MN ? make_smem_desc_mn(ah + kABytes + k * 2048) : make_smem_desc(ah + kABytes + k * 32);
              const uint64_t dbl = B_MN ? make_smem_desc_mn(aB + B_BYTES + k * 2048) : make_smem_desc(aB + B_BYTES + k * 32);
              wgmma_bf16<BLOCK_N, A_MN, B_MN>(acc[h], dal, db, (kb | k) != 0);
              wgmma_bf16<BLOCK_N, A_MN, B_MN>(acc[h], da, dbl, 1);
              wgmma_bf16<BLOCK_N, A_MN, B_MN>(acc[h], da, db, 1);
            } else {
              wgmma_bf16<BLOCK_N, A_MN, B_MN>(acc[h], da, db, (kb | k) != 0);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty(prev)); }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty(prev)); }
      if (num_kb == 0) {  // nothing was accumulated (empty split)
#pragma unroll
        for (int j = 0; j < BLOCK_N / 2; ++j) { acc[0][j] = 0.0f; acc[1][j] = 0.0f; }
      }
      named_sync(1, kConsumers);  // the previous tile's epilogue has read the staging tile
      {
        const int fr = warp * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            float* sp = stg + (h * 64 + fr) * LDS + 8 * j + fc;
            *reinterpret_cast<float2*>(sp) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
            *reinterpret_cast<float2*>(sp + 8 * LDS) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
          }
      }
      named_sync(1, kConsumers);
#pragma unroll 1
      for (int c0 = 0; c0 < BLOCK_N; c0 += 32) {
        uint32_t v[32];
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 t = *reinterpret_cast<const float4*>(stg + rl * LDS + c0 + j);
          v[j] = __float_as_uint(t.x); v[j + 1] = __float_as_uint(t.y); v[j + 2] = __float_as_uint(t.z); v[j + 3] = __float_as_uint(t.w);
        }
        if (partial) {  // split-K: raw partial tile [z][M][N]; splitk_reduce_kernel applies the epilogue
          if (rvalid) {
            // rows of the partial tiles are ldp floats apart, ldp = N rounded up to 32: every chunk that starts
            // inside a row is stored whole with 16-byte stores (the columns past N hold exact zeros from the TMA
            // fill).  With the natural stride an odd N (519) forced 4-byte stores: 6x write amplification in L2.
            float* pz = partial + (int64_t(z) * M + r) * ldp + n0 + c0;
            if (n0 + c0 + 32 <= ldp) {
#pragma unroll
              for (int j = 0; j < 32; j += 4)
                *reinterpret_cast<float4*>(pz + j) = make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]),
                                                                  __uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
            } else if (n0 + c0 < ldp) {
              for (int j = 0; j < 32; ++j)
                if (n0 + c0 + j < N) pz[j] = __uint_as_float(v[j]);
            }
          }
          continue;
        }
        if (rvalid) {
          const int nbase = n0 + c0;
          int64_t pr; int pc;
          if (!locate(c0, pr, pc)) continue;
          float o[32];
          const bool full_cols = nbase + 32 <= N;
          // EPI 2: the ReLU mask / residual rows are read as four 16-byte vectors per 32 columns when aligned
          // (32 scalar 2-byte loads per thread made fc_dgrad epilogue-bound)
          uint32_t m16[16], a16[16];
          bool vm = false, va = false;
          if constexpr (EPI >= 2) {
            if (full_cols && ep.mask16 && (ep.ldmask & 7) == 0) {
              const __nv_bfloat16* mp = ep.mask16 + pr * ep.ldmask + pc;
              if ((reinterpret_cast<uintptr_t>(mp) & 15) == 0) {
                vm = true;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const uint4 t = __ldg(reinterpret_cast<const uint4*>(mp) + q);
                  m16[4 * q] = t.x; m16[4 * q + 1] = t.y; m16[4 * q + 2] = t.z; m16[4 * q + 3] = t.w;
                }
              }
            }
            if (full_cols && ep.addend16 && (ep.ldadd & 7) == 0) {
              const __nv_bfloat16* ap = ep.addend16 + pr * ep.ldadd + pc;
              if ((reinterpret_cast<uintptr_t>(ap) & 15) == 0) {
                va = true;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const uint4 t = __ldg(reinterpret_cast<const uint4*>(ap) + q);
                  a16[4 * q] = t.x; a16[4 * q + 1] = t.y; a16[4 * q + 2] = t.z; a16[4 * q + 3] = t.w;
                }
              }
            }
          }
          // uniform branches around whole 32-element passes (per-element predication on the runtime flags cost ~15
          // instructions per output and made the short-K implicit convolutions issue-bound in this epilogue)
#pragma unroll
          for (int j = 0; j < 32; ++j) o[j] = __uint_as_float(v[j]);
          if constexpr (EPI >= 1) {
            if (ep.scale != 1.0f) {
#pragma unroll
              for (int j = 0; j < 32; ++j) o[j] *= ep.scale;
            }
            if (ep.bias) {
              const float* bp = ep.bias + nbase;
              if (full_cols && (reinterpret_cast<uintptr_t>(bp) & 15) == 0) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                  const float4 b4 = __ldg(reinterpret_cast<const float4*>(bp) + q);
                  o[4 * q] += b4.x; o[4 * q + 1] += b4.y; o[4 * q + 2] += b4.z; o[4 * q + 3] += b4.w;
                }
              } else {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  if (nbase + j < N) o[j] += __ldg(bp + j);
              }
            }
            if (ep.relu) {
#pragma unroll
              for (int j = 0; j < 32; ++j) o[j] = fmaxf(o[j], 0.0f);
            }
          }
          if constexpr (EPI >= 2) {
            if (ep.mask) {
              const float* mp = ep.mask + pr * ep.ldmask + pc;
              const bool mvec = (ep.ldmask & 3) == 0 && (reinterpret_cast<uintptr_t>(mp) & 15) == 0;
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                if (mvec && nbase + j + 4 <= N) {
                  const float4 m4 = __ldg(reinterpret_cast<const float4*>(mp + j));
                  o[j] = m4.x > 0.0f ? o[j] : 0.0f; o[j + 1] = m4.y > 0.0f ? o[j + 1] : 0.0f;
                  o[j + 2] = m4.z > 0.0f ? o[j + 2] : 0.0f; o[j + 3] = m4.w > 0.0f ? o[j + 3] : 0.0f;
                } else {
#pragma unroll
                  for (int jj = 0; jj < 4; ++jj)
                    if (nbase + j + jj < N) o[j + jj] = (mp[j + jj] > 0.0f) ? o[j + jj] : 0.0f;
                }
              }
            }
            if (vm) {  // a bf16 is positive iff its bit pattern, read as a signed 16-bit integer, is > 0
#pragma unroll
              for (int j = 0; j < 32; j += 2) {
                const uint32_t m = m16[j >> 1];
                o[j] = (int(m << 16) > 0) ? o[j] : 0.0f;
                o[j + 1] = (int(m & 0xffff0000u) > 0) ? o[j + 1] : 0.0f;
              }
            } else if (ep.mask16) {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (nbase + j < N) o[j] = (__bfloat162float(ep.mask16[pr * ep.ldmask + pc + j]) > 0.0f) ? o[j] : 0.0f;
            }
            if (va) {
#pragma unroll
              for (int j = 0; j < 32; j += 2) {
                const uint32_t m = a16[j >> 1];
                o[j] += __uint_as_float(m << 16);
                o[j + 1] += __uint_as_float(m & 0xffff0000u);
              }
            } else if (ep.addend16) {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (nbase + j < N) o[j] += __bfloat162float(ep.addend16[pr * ep.ldadd + pc + j]);
            }
            if (ep.addend32) {
              const float* ap = ep.addend32 + pr * ep.ldadd + pc;
              if (full_cols && (ep.ldadd & 3) == 0 && (reinterpret_cast<uintptr_t>(ap) & 15) == 0) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                  const float4 a4 = __ldg(reinterpret_cast<const float4*>(ap) + q);
                  o[4 * q] += a4.x; o[4 * q + 1] += a4.y; o[4 * q + 2] += a4.z; o[4 * q + 3] += a4.w;
                }
              } else {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                  if (nbase + j + 4 <= N && (ep.ldadd & 3) == 0 && (reinterpret_cast<uintptr_t>(ap) & 15) == 0) {
                    const float4 a4 = __ldg(reinterpret_cast<const float4*>(ap + j));
                    o[j] += a4.x; o[j + 1] += a4.y; o[j + 2] += a4.z; o[j + 3] += a4.w;
                  } else {
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj)
                      if (nbase + j + jj < N) o[j + jj] += __ldg(ap + j + jj);
                  }
                }
              }
            }
          }
          if (ep.C) {
            float* c = ep.C + pr * ep.ldc + pc;
            if (full_cols && (ep.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(c) & 15) == 0) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(c + j) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
            } else {
              const bool vec = (ep.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(c) & 15) == 0;
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                if (vec && nbase + j + 4 <= N) {
                  *reinterpret_cast<float4*>(c + j) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
                } else {
#pragma unroll
                  for (int jj = 0; jj < 4; ++jj)
                    if (nbase + j + jj < N) c[j + jj] = o[j + jj];
                }
              }
            }
          }
          if (ep.C16) {
            __nv_bfloat16* c = ep.C16 + pr * ep.ldc16 + pc;
            const bool wlo = SPLIT && ep.c16_lo != 0;  // also write the lo plane (c16_lo is a multiple of 8 elements)
            const bool vec = (ep.ldc16 & 7) == 0 && (reinterpret_cast<uintptr_t>(c) & 15) == 0;
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              // column tail (N = 144, 288, ...): still 16-byte stores for the complete groups of 8
              if (vec && (full_cols || nbase + j + 8 <= N)) {
                uint4 ph, pl;
                split_bf16x2(o[j], o[j + 1], ph.x, pl.x); split_bf16x2(o[j + 2], o[j + 3], ph.y, pl.y);
                split_bf16x2(o[j + 4], o[j + 5], ph.z, pl.z); split_bf16x2(o[j + 6], o[j + 7], ph.w, pl.w);
                *reinterpret_cast<uint4*>(c + j) = ph;
                if (wlo) *reinterpret_cast<uint4*>(c + ep.c16_lo + j) = pl;
              } else {
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
                  if (nbase + j + jj < N) {
                    const __nv_bfloat16 h = __float2bfloat16_rn(o[j + jj]);
                    c[j + jj] = h;
                    if (wlo) c[ep.c16_lo + j + jj] = bf16_lo_of(o[j + jj], h);
                  }
              }
            }
          }
        }
      }
    }
  }
}

struct TcMaps { CUtensorMap a, b, al, bl; };  // operand maps (+ lo planes in split mode; copies of a / b otherwise)

// cudaFuncSetAttribute is per device: remember which devices have had it applied for this instantiation
static inline bool attr_done(uint64_t* mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t bit = uint64_t(1) << (dev & 63);
  if (*mask & bit) return true;
  *mask |= bit;
  return false;
}

// dynamic shared memory of gemm_tc_kernel: 1 KB alignment slack, the stage ring, the barriers, the accumulator staging tile
constexpr size_t tc_smem(int block_n, int stages, bool split) {
  return 1024 + size_t(stages) * (split ? 2 : 1) * (kABytes + size_t(block_n) * kBlockK * 2) + 16 * stages +
         size_t(kBlockM) * (block_n + 4) * 4 + 16;
}
// the deepest ring of at most `want` stages that fits beside the staging tile
constexpr int tc_stages(int block_n, int want, bool split) {
  return (want <= 2 || tc_smem(block_n, want, split) <= 227 * 1024) ? want : tc_stages(block_n, want - 1, split);
}

// CTAs of `kernel` resident per SM with `smem` bytes of dynamic shared memory: registers, not shared memory, are the
// limit for most instantiations (a 128-column accumulator pair plus the epilogue needs > 204 registers per thread)
template <typename Kernel>
static int resident_per_sm(Kernel kernel, size_t smem) {
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kThreads, smem) != cudaSuccess || n < 1) n = 1;
  return n;
}

template <int BLOCK_N, bool A_MN, bool B_MN, int kStages, int EPI, bool SPLIT>
int launch_e(const TcMaps& mp, const TcEpilogue& ep, int64_t M, int64_t N, int64_t K, int splits,
             float* partial, cudaStream_t stream) {
  constexpr size_t smem = tc_smem(BLOCK_N, kStages, SPLIT);
  static_assert(smem <= 227 * 1024, "gemm_tc: stage ring exceeds shared memory");
  static uint64_t attr = 0;
  static int per_sm = 1;
  if (!attr_done(&attr)) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BLOCK_N, A_MN, B_MN, kStages, EPI, false, SPLIT>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "gemm_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    per_sm = resident_per_sm(gemm_tc_kernel<BLOCK_N, A_MN, B_MN, kStages, EPI, false, SPLIT>, smem);
  }
  const int64_t tiles_m = (M + kBlockM - 1) / kBlockM, tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int64_t total = tiles_m * tiles_n * splits;
  TB_REQUIRE(total < (int64_t(1) << 31), "gemm_tc: too many tiles");
  // persistent grid: as many CTAs as are resident at once
  int64_t grid = int64_t(kNumSMs) * per_sm;
  if (ep.max_ctas > 0 && grid > ep.max_ctas) grid = ep.max_ctas;
  if (grid > total) grid = total;
  gemm_tc_kernel<BLOCK_N, A_MN, B_MN, kStages, EPI, false, SPLIT><<<(unsigned)grid, kThreads, smem, stream>>>(
      mp.a, mp.b, mp.al, mp.bl, ep, int(M), int(N), int(K), partial, int(tiles_m), int(tiles_n), splits,
      int((N + 31) & ~int64_t(31)));
  return check_launch("gemm_tc_kernel");
}

template <int BLOCK_N, bool A_MN, bool B_MN, int kStages, bool SPLIT>
int launch_s(const TcMaps& mp, const TcEpilogue& ep, int64_t M, int64_t N, int64_t K, int splits,
             float* partial, cudaStream_t stream) {
  const bool loads = ep.mask || ep.mask16 || ep.addend16 || ep.addend32;
  const bool arith = ep.bias || ep.relu || ep.scale != 1.0f;
  if (loads) return launch_e<BLOCK_N, A_MN, B_MN, kStages, 2, SPLIT>(mp, ep, M, N, K, splits, partial, stream);
  if (arith && !partial) return launch_e<BLOCK_N, A_MN, B_MN, kStages, 1, SPLIT>(mp, ep, M, N, K, splits, partial, stream);
  return launch_e<BLOCK_N, A_MN, B_MN, kStages, 0, SPLIT>(mp, ep, M, N, K, splits, partial, stream);
}

// Few k-blocks per CTA (dgrad: K = 64 channels): a deeper ring than 2 stages would only hold the next tile's data, so
// the ring stays small.  Within a CTA the epilogue does not overlap the next tile's MMAs (the producer prefetches into
// the ring meanwhile); overlap across CTAs happens only where registers allow two per SM.
// Split mode doubles the stage (hi + lo planes); the ring is as deep as fits beside the accumulator staging tile.
template <int BLOCK_N, bool A_MN, bool B_MN>
int launch(const TcMaps& mp, const TcEpilogue& ep, int64_t M, int64_t N, int64_t K, int splits,
           float* partial, cudaStream_t stream) {
  const int64_t kb_per_cta = ((K + kBlockK - 1) / kBlockK + splits - 1) / splits;
  const bool split = ep.a_lo != 0;
  if (split) {
    if (kb_per_cta <= 2) return launch_s<BLOCK_N, A_MN, B_MN, 2, true>(mp, ep, M, N, K, splits, partial, stream);
    return launch_s<BLOCK_N, A_MN, B_MN, tc_stages(BLOCK_N, 4, true), true>(mp, ep, M, N, K, splits, partial, stream);
  }
  if (kb_per_cta <= 2) return launch_s<BLOCK_N, A_MN, B_MN, 2, false>(mp, ep, M, N, K, splits, partial, stream);
  return launch_s<BLOCK_N, A_MN, B_MN, tc_stages(BLOCK_N, 4, false), false>(mp, ep, M, N, K, splits, partial, stream);
}


// Implicit-GEMM convolution weight gradient: dW[o, k] = sum_patches dY[patch, o] * patch[patch, k] with the
// patches read straight from the NHWC activation (same overlapping-dimension tensor map as the forward).
// One stage = the `rows` patches of `fpt` whole frames: A = one 64(o) x rows box of dY (MN-major), B = two
// 64(k) x rows boxes of patches (MN-major: the k-th 64-wide group is k-block n0/64 + j of the kernel window).
// rows is padded to a multiple of 16 (the wgmma K step) with shared-memory rows that are zeroed once and
// never written by TMA, so the padding contributes exact zeros.  CTAs split the frames; raw fp32 partial
// tiles go to `partial` [z][O][K] and splitk_reduce_kernel folds them in a fixed order.
struct ImplicitWgrad {
  int rows = 0, rows_pad = 0, fpt = 1, kbw = 1, row_elems = 0;
  int stages_total = 0;  // ceil(frames / fpt)
  int per = 0;           // stages per split
};

// SPLIT (split-bf16): the stage also carries the lo planes, [dY hi][dY lo][patch0 hi][patch1 hi][patch0 lo][patch1 lo],
// and every k-step issues dYlo.Phi, dYhi.Plo, dYhi.Phi.
template <int kSt, bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_implicit_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                           const __grid_constant__ CUtensorMap tmAl, const __grid_constant__ CUtensorMap tmBl, int O, int Kdim,
                           float* __restrict__ partial, int tiles_n, ImplicitWgrad iw) {
  constexpr int BLOCK_N = 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
  const uint32_t group = uint32_t(iw.rows_pad) * 128u;  // one 64-wide group: rows_pad x 128 B (multiple of 1024)
  const uint32_t stage_bytes = (SPLIT ? 6u : 3u) * group;  // [dY group][patch group 0][patch group 1]
  const uint32_t offB = (SPLIT ? 2u : 1u) * group;         // first patch group
  const uint32_t bars = base + kSt * stage_bytes;       // full[kSt], empty[kSt]
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kSt + s); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x % tiles_n, z = blockIdx.x / tiles_n;
  const int n0 = nt * BLOCK_N;
  const int s0 = z * iw.per;
  const int s1 = (s0 + iw.per < iw.stages_total) ? s0 + iw.per : iw.stages_total;
  const int num = s1 > s0 ? s1 - s0 : 0;

  // zero the ring once: the padding rows [rows, rows_pad) of every group must read as exact zeros
  for (uint32_t off = threadIdx.x * 16u; off < kSt * stage_bytes; off += kThreads * 16u)
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(base + off), "r"(0u) : "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  if (warp == 4 && lane == 0) {
    for (int s = 0; s < kSt; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      const int kbA = n0 / kBlockK, kbB = kbA + 1;
      const int eA = (kbA / iw.kbw) * iw.row_elems + (kbA % iw.kbw) * kBlockK;
      const int eB = (kbB / iw.kbw) * iw.row_elems + (kbB % iw.kbw) * kBlockK;
      int stage = 0; uint32_t phase = 0;
      for (int i = 0; i < num; ++i) {
        const int f0 = (s0 + i) * iw.fpt;
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(full(stage), (SPLIT ? 6u : 3u) * uint32_t(iw.rows) * 128u);
        const uint32_t st = base + stage * stage_bytes;
        tma_load_2d(st, &tmA, full(stage), 0, f0 * (iw.rows / iw.fpt));
        tma_load_4d(st + offB, &tmB, full(stage), eA, 0, 0, f0);
        tma_load_4d(st + offB + group, &tmB, full(stage), eB, 0, 0, f0);
        if constexpr (SPLIT) {
          tma_load_2d(st + group, &tmAl, full(stage), 0, f0 * (iw.rows / iw.fpt));
          tma_load_4d(st + 4 * group, &tmBl, full(stage), eA, 0, 0, f0);
          tma_load_4d(st + 5 * group, &tmBl, full(stage), eB, 0, 0, f0);
        }
        if (++stage == kSt) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // M = 64 output channels (O <= 64): one m64n128 accumulator per warpgroup
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int j = 0; j < BLOCK_N / 2; ++j) acc[j] = 0.0f;
    const int ksteps = iw.rows_pad / 16;
    int stage = 0; uint32_t phase = 0;
    for (int i = 0; i < num; ++i) {
      mbar_wait(full(stage), phase);
      wgmma_fence();
      const uint32_t st = base + stage * stage_bytes;
      for (int k = 0; k < ksteps; ++k) {
        const uint64_t da = make_smem_desc_mn_lbo(st + k * 2048, group);
        const uint64_t db = make_smem_desc_mn_lbo(st + offB + k * 2048, group);
        if constexpr (SPLIT) {
          wgmma_bf16<BLOCK_N, 1, 1>(acc, make_smem_desc_mn_lbo(st + group + k * 2048, group), db, (i | k) != 0);
          wgmma_bf16<BLOCK_N, 1, 1>(acc, da, make_smem_desc_mn_lbo(st + 4 * group + k * 2048, group), 1);
          wgmma_bf16<BLOCK_N, 1, 1>(acc, da, db, 1);
        } else {
          wgmma_bf16<BLOCK_N, 1, 1>(acc, da, db, (i | k) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(stage));
      if (++stage == kSt) { stage = 0; phase ^= 1; }
    }
    // fragment rows r and r + 8 (output channels), column pairs 8j + fc
    const int r = warp * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int o = r + 8 * e;
      if (o >= O) continue;
      float* pz = partial + (int64_t(z) * O + o) * Kdim + n0;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int c = 8 * j + fc;
        if (n0 + c + 2 <= Kdim && (Kdim & 1) == 0) {
          *reinterpret_cast<float2*>(pz + c) = make_float2(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]);
        } else {
          if (n0 + c < Kdim) pz[c] = acc[4 * j + 2 * e];
          if (n0 + c + 1 < Kdim) pz[c + 1] = acc[4 * j + 2 * e + 1];
        }
      }
    }
  }
}

template <int BLOCK_N, int EPI, int kSt, bool SPLIT>
int launch_conv_fwd_s(const TcMaps& mp, const TcEpilogue& ep, int64_t M, int64_t N, int64_t K,
                      int64_t tiles_m, const ImplicitConv& ic, cudaStream_t stream) {
  constexpr size_t smem = tc_smem(BLOCK_N, kSt, SPLIT);
  static_assert(smem <= 227 * 1024, "gemm_tc: stage ring exceeds shared memory");
  static uint64_t attr = 0;
  static int per_sm = 1;
  if (!attr_done(&attr)) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BLOCK_N, false, false, kSt, EPI, true, SPLIT>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "gemm_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    per_sm = resident_per_sm(gemm_tc_kernel<BLOCK_N, false, false, kSt, EPI, true, SPLIT>, smem);
  }
  const int64_t tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int64_t total = tiles_m * tiles_n;
  int64_t grid = int64_t(kNumSMs) * per_sm;
  if (grid > total) grid = total;
  gemm_tc_kernel<BLOCK_N, false, false, kSt, EPI, true, SPLIT><<<(unsigned)grid, kThreads, smem, stream>>>(
      mp.a, mp.b, mp.al, mp.bl, ep, int(M), int(N), int(K), nullptr, int(tiles_m), int(tiles_n), 1, 0, ic);
  return check_launch("gemm_tc_kernel(implicit conv)");
}

template <int BLOCK_N, int EPI = 1, int kSt = 4>
int launch_conv_fwd(const TcMaps& mp, const TcEpilogue& ep, int64_t M, int64_t N, int64_t K, int64_t tiles_m,
                    const ImplicitConv& ic, cudaStream_t stream) {
  if (ep.a_lo != 0)  // split: stages of twice the size
    return launch_conv_fwd_s<BLOCK_N, EPI, tc_stages(BLOCK_N, kSt, true), true>(mp, ep, M, N, K, tiles_m, ic, stream);
  return launch_conv_fwd_s<BLOCK_N, EPI, tc_stages(BLOCK_N, kSt, false), false>(mp, ep, M, N, K, tiles_m, ic, stream);
}

}  // namespace

bool conv_tc_implicit_applicable(int H, int W, int C, int KH, int KW, int S, int O) {
  if (H < KH || W < KW || S < 1) return false;
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  return (KW * C) % kBlockK == 0 && (S * C * 2) % 16 == 0 && (C % 8) == 0 && OW * OH <= kBlockM && OW <= 256 && OH <= 256 &&
         (O == 32 || O == 64 || O % 128 == 0 || O <= 128);
}

int conv_tc_fwd_implicit(const void* act_nhwc_bf16, const void* w_packed_bf16, int64_t Nf, int H, int W, int C, int KH, int KW,
                         int S, int O, const TcEpilogue& ep, cudaStream_t stream) {
  TB_REQUIRE(act_nhwc_bf16 && w_packed_bf16 && (ep.C || ep.C16), "conv_tc_fwd_implicit: null pointer");
  TB_REQUIRE(conv_tc_implicit_applicable(H, W, C, KH, KW, S, O), "conv_tc_fwd_implicit: unsupported shape");
  if (Nf == 0) return 0;
  ProfScope prof(ep.tag, stream);
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  ImplicitConv ic;
  ic.fpt = kBlockM / (OW * OH);
  if (ic.fpt > 256) ic.fpt = 256;
  ic.rows = OW * OH * ic.fpt;
  ic.kbw = KW * C / kBlockK;
  ic.row_elems = W * C;
  const int64_t K = int64_t(KH) * KW * C, M = Nf * OH * OW;
  const int64_t tiles_m = (Nf + ic.fpt - 1) / ic.fpt;
  const uint64_t dims[4] = {uint64_t(H) * W * C, uint64_t(OW), uint64_t(OH), uint64_t(Nf)};
  const uint64_t strides[3] = {uint64_t(S) * C * 2, uint64_t(S) * W * C * 2, uint64_t(H) * W * C * 2};
  const uint32_t box[4] = {uint32_t(kBlockK), uint32_t(OW), uint32_t(OH), uint32_t(ic.fpt)};
  TB_REQUIRE((ep.a_lo != 0) == (ep.b_lo != 0), "conv_tc_fwd_implicit: split mode needs both lo planes");
  TcMaps mp;
  int rc = make_map_nd(&mp.a, act_nhwc_bf16, 4, dims, strides, box);
  if (rc) return rc;
  const int bn = (O <= 32) ? 32 : (O <= 64 ? 64 : 128);
  rc = make_map(&mp.b, w_packed_bf16, O, K, K, bn);
  if (rc) return rc;
  mp.al = mp.a; mp.bl = mp.b;
  if (ep.a_lo) {
    rc = make_map_nd(&mp.al, static_cast<const __nv_bfloat16*>(act_nhwc_bf16) + ep.a_lo, 4, dims, strides, box);
    if (rc) return rc;
    rc = make_map(&mp.bl, static_cast<const __nv_bfloat16*>(w_packed_bf16) + ep.b_lo, O, K, K, bn);
    if (rc) return rc;
  }
  if (bn == 32) return launch_conv_fwd<32>(mp, ep, M, O, K, tiles_m, ic, stream);
  if (bn == 64) return launch_conv_fwd<64>(mp, ep, M, O, K, tiles_m, ic, stream);
  return launch_conv_fwd<128>(mp, ep, M, O, K, tiles_m, ic, stream);
}

bool conv_tc_dgrad_implicit_applicable(int H, int W, int C, int KH, int KW, int S, int O) {
  if (O != 64 || H < KH || W < KW) return false;
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  if (S == 1) return H * W <= kBlockM && (C == 32 || C == 64 || C == 128) && (OH - 1) + KH == H && (OW - 1) + KW == W;
  if (S == 2)  // every input pixel is covered and the parity tiles are exact
    return KH == 4 && KW == 4 && C == 32 && (H % 2) == 0 && (W % 2) == 0 && (H / 2) * (W / 2) <= kBlockM &&
           2 * (OH - 1) + KH == H && 2 * (OW - 1) + KW == W;
  return false;
}

// dX (ep.C16, bf16 NHWC [Nf,H,W,C], multiplied by the ReLU mask ep.mask16 = forward activation) from dY [Nf,OH,OW,64];
// wt_bf16: stride 1: [C, (kh,kw,o)];  stride 2: [(py,px,c), (i,j,o)]   (net_kernels: pack_dgrad_weights_bf16)
int conv_tc_dgrad_implicit(const void* dy_nhwc_bf16, const void* wt_bf16, int64_t Nf, int H, int W, int C, int KH, int KW, int S,
                           int O, const TcEpilogue& ep, cudaStream_t stream) {
  TB_REQUIRE(dy_nhwc_bf16 && wt_bf16 && ep.C16 && ep.ldc16 == C && (!ep.mask16 || ep.ldmask == C),
             "conv_tc_dgrad_implicit: bad arguments");
  TB_REQUIRE(conv_tc_dgrad_implicit_applicable(H, W, C, KH, KW, S, O), "conv_tc_dgrad_implicit: unsupported shape");
  if (Nf == 0) return 0;
  ProfScope prof(ep.tag, stream);
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  ImplicitConv ic;
  ic.fpt = 1;
  TB_REQUIRE((ep.a_lo != 0) == (ep.b_lo != 0), "conv_tc_dgrad_implicit: split mode needs both lo planes");
  TcMaps mp;
  const __nv_bfloat16* dy_lo = static_cast<const __nv_bfloat16*>(dy_nhwc_bf16) + ep.a_lo;
  const __nv_bfloat16* wt_lo = static_cast<const __nv_bfloat16*>(wt_bf16) + ep.b_lo;
  const uint64_t dims[4] = {uint64_t(O), uint64_t(OW), uint64_t(OH), uint64_t(Nf)};
  const uint64_t strides[3] = {uint64_t(O) * 2, uint64_t(OW) * O * 2, uint64_t(OH) * OW * O * 2};
  int rc;
  if (S == 1) {
    ic.mode = 1; ic.rows = H * W; ic.kbw = KW;
    const uint32_t box[4] = {uint32_t(kBlockK), uint32_t(W), uint32_t(H), 1u};
    rc = make_map_nd(&mp.a, dy_nhwc_bf16, 4, dims, strides, box);
    if (rc) return rc;
    const int64_t K = int64_t(KH) * KW * O, M = Nf * ic.rows;
    const int bn = (C <= 32) ? 32 : (C <= 64 ? 64 : 128);
    rc = make_map(&mp.b, wt_bf16, C, K, K, bn);
    if (rc) return rc;
    mp.al = mp.a; mp.bl = mp.b;
    if (ep.a_lo) {
      rc = make_map_nd(&mp.al, dy_lo, 4, dims, strides, box);
      if (rc) return rc;
      rc = make_map(&mp.bl, wt_lo, C, K, K, bn);
      if (rc) return rc;
    }
    if (bn == 32) return launch_conv_fwd<32, 2>(mp, ep, M, C, K, Nf, ic, stream);
    if (bn == 64) return launch_conv_fwd<64, 2>(mp, ep, M, C, K, Nf, ic, stream);
    return launch_conv_fwd<128, 2>(mp, ep, M, C, K, Nf, ic, stream);
  }
  ic.mode = 2; ic.tw = W / 2; ic.rows = (H / 2) * (W / 2); ic.kbw = KW / 2; ic.outH = H; ic.outW = W;
  const uint32_t box[4] = {uint32_t(kBlockK), uint32_t(W / 2), uint32_t(H / 2), 1u};
  rc = make_map_nd(&mp.a, dy_nhwc_bf16, 4, dims, strides, box);
  if (rc) return rc;
  const int64_t K = int64_t(KH / 2) * (KW / 2) * O, M = Nf * ic.rows;
  rc = make_map(&mp.b, wt_bf16, 4 * C, K, K, 128);
  if (rc) return rc;
  mp.al = mp.a; mp.bl = mp.b;
  if (ep.a_lo) {
    rc = make_map_nd(&mp.al, dy_lo, 4, dims, strides, box);
    if (rc) return rc;
    rc = make_map(&mp.bl, wt_lo, 4 * C, K, K, 128);
    if (rc) return rc;
  }
  // 4 k-blocks per tile: a 2-stage ring holds the next tile's operands while the epilogue runs
  return launch_conv_fwd<128, 2, 2>(mp, ep, M, 4 * C, K, Nf, ic, stream);
}

template <int kSt, bool SPLIT>
static int launch_conv_wgrad(const TcMaps& mp, int O, int64_t K, float* partial, int tiles_n, int64_t splits,
                             const ImplicitWgrad& iw, cudaStream_t stream) {
  const size_t smem = 1024 + size_t(kSt) * (SPLIT ? 6 : 3) * iw.rows_pad * 128 + 8 * (2 * kSt + 1) + 16;
  TB_REQUIRE(smem <= 227 * 1024, "conv_tc_wgrad_implicit: stage too large");
  static size_t attr[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr[dev & 63] < smem) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_implicit_kernel<kSt, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "conv_tc_wgrad_implicit: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr[dev & 63] = smem;
  }
  conv_wgrad_implicit_kernel<kSt, SPLIT><<<(unsigned)(splits * tiles_n), kThreads, smem, stream>>>(mp.a, mp.b, mp.al, mp.bl, O, int(K),
                                                                                                 partial, tiles_n, iw);
  return check_launch("conv_wgrad_implicit_kernel");
}

int conv_tc_wgrad_implicit(const void* dy_bf16, const void* act_nhwc_bf16, int64_t Nf, int H, int W, int C, int KH, int KW, int S,
                           int O, float* dW, int permP, int permQ, float scale, float* partial, int64_t partial_floats,
                           const char* tag, cudaStream_t stream, int64_t dy_lo, int64_t act_lo) {
  TB_REQUIRE(dy_bf16 && act_nhwc_bf16 && dW && partial, "conv_tc_wgrad_implicit: null pointer");
  TB_REQUIRE(conv_tc_implicit_applicable(H, W, C, KH, KW, S, O) && O <= 64 && O % 8 == 0,
             "conv_tc_wgrad_implicit: unsupported shape");
  if (Nf == 0) return 0;
  ProfScope prof(tag, stream);
  const int OH = (H - KH) / S + 1, OW = (W - KW) / S + 1;
  const int64_t K = int64_t(KH) * KW * C;
  ImplicitWgrad iw;
  iw.fpt = kBlockM / (OW * OH);
  if (iw.fpt > 256) iw.fpt = 256;
  iw.rows = OW * OH * iw.fpt;
  iw.rows_pad = (iw.rows + 15) & ~15;
  if (iw.rows_pad % 8) iw.rows_pad = (iw.rows_pad + 7) & ~7;
  iw.kbw = KW * C / kBlockK;
  iw.row_elems = W * C;
  iw.stages_total = int((Nf + iw.fpt - 1) / iw.fpt);
  const int tiles_n = int((K + 127) / 128);
  // the second 64-wide group of the last n tile may start past K: its kernel-row offset must still be inside the frame
  {
    const int kb_last = tiles_n * 2 - 1;
    const int64_t e_last = int64_t(kb_last / iw.kbw) * iw.row_elems + int64_t(kb_last % iw.kbw) * kBlockK;
    TB_REQUIRE(e_last + kBlockK <= int64_t(H) * W * C, "conv_tc_wgrad_implicit: window tail outside the frame");
  }
  int64_t splits = kNumSMs / tiles_n;
  if (splits > iw.stages_total) splits = iw.stages_total;
  if (splits * O * K > partial_floats) splits = partial_floats / (int64_t(O) * K);
  TB_REQUIRE(splits >= 1, "conv_tc_wgrad_implicit: partial buffer too small");
  iw.per = int((iw.stages_total + splits - 1) / splits);
  splits = (iw.stages_total + iw.per - 1) / iw.per;
  TB_REQUIRE((dy_lo != 0) == (act_lo != 0), "conv_tc_wgrad_implicit: split mode needs both lo planes");
  TcMaps mp;
  // dY [patches, O]: MN-major box of 64 channels x `rows` patches
  int rc = make_map(&mp.a, dy_bf16, Nf * OH * OW, O, O, iw.rows, 64);
  if (rc) return rc;
  const uint64_t dims[4] = {uint64_t(H) * W * C, uint64_t(OW), uint64_t(OH), uint64_t(Nf)};
  const uint64_t strides[3] = {uint64_t(S) * C * 2, uint64_t(S) * W * C * 2, uint64_t(H) * W * C * 2};
  const uint32_t box[4] = {uint32_t(kBlockK), uint32_t(OW), uint32_t(OH), uint32_t(iw.fpt)};
  rc = make_map_nd(&mp.b, act_nhwc_bf16, 4, dims, strides, box);
  if (rc) return rc;
  mp.al = mp.a; mp.bl = mp.b;
  if (dy_lo) {
    rc = make_map(&mp.al, static_cast<const __nv_bfloat16*>(dy_bf16) + dy_lo, Nf * OH * OW, O, O, iw.rows, 64);
    if (rc) return rc;
    rc = make_map_nd(&mp.bl, static_cast<const __nv_bfloat16*>(act_nhwc_bf16) + act_lo, 4, dims, strides, box);
    if (rc) return rc;
    // 6 groups per stage: as many stages as fit (2 for the 98-patch conv3 tiles, 3 for the 81-patch conv2 tiles)
    if (size_t(3) * 6 * iw.rows_pad * 128 + 2048 <= 227 * 1024) rc = launch_conv_wgrad<3, true>(mp, O, K, partial, tiles_n, splits, iw, stream);
    else rc = launch_conv_wgrad<2, true>(mp, O, K, partial, tiles_n, splits, iw, stream);
  } else {
    rc = launch_conv_wgrad<4, false>(mp, O, K, partial, tiles_n, splits, iw, stream);
  }
  if (rc) return rc;
  GemmEpilogue rep;
  rep.permP = permP; rep.permQ = permQ; rep.scale = scale;
  return launch_splitk_reduce(partial, dW, O, K, K, int(splits), rep, K, stream);
}

int gemm_tc_bf16(const void* A, const void* B, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                 const TcEpilogue& ep, cudaStream_t stream) {
  return gemm_tc_bf16_ex(A, B, M, N, K, lda, ldb, false, false, ep, 1, nullptr, stream);
}

int gemm_tc_bf16_ex(const void* A, const void* B, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, bool a_mn,
                    bool b_mn, const TcEpilogue& ep, int splits, float* partial, cudaStream_t stream) {
  TB_REQUIRE(M >= 0 && N >= 0 && K >= 1, "gemm_tc: bad sizes M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
  if (M == 0 || N == 0) return 0;
  TB_REQUIRE(A && B && (ep.C || ep.C16 || partial), "gemm_tc: null pointer");
  TB_REQUIRE(M < (int64_t(1) << 31) && N < (int64_t(1) << 31) && K < (int64_t(1) << 31), "gemm_tc: size overflow");
  TB_REQUIRE(!a_mn || b_mn, "gemm_tc: A MN-major requires B MN-major (wgrad form)");
  if (splits < 1) splits = 1;
  TB_REQUIRE(splits == 1 || partial, "gemm_tc: split-K needs a partial buffer");
  ProfScope prof(ep.tag, stream);
  int bn = (N <= 32) ? 32 : (N <= 64 ? 64 : 128);
  if (b_mn && bn < 64) bn = 64;  // MN-major tiles are built from 64-wide boxes
  TB_REQUIRE((ep.a_lo != 0) == (ep.b_lo != 0), "gemm_tc: split mode needs the lo planes of both operands");
  TcMaps mp;
  // K-major operand [rows = mn, cols = k]: box {64 k, mn rows}.  MN-major operand [rows = k, cols = mn]: box {64 mn, 64 k}.
  int rc = a_mn ? make_map(&mp.a, A, K, M, lda, kBlockK, 64) : make_map(&mp.a, A, M, K, lda, kBlockM);
  if (rc) return rc;
  rc = b_mn ? make_map(&mp.b, B, K, N, ldb, kBlockK, 64) : make_map(&mp.b, B, N, K, ldb, bn);
  if (rc) return rc;
  mp.al = mp.a; mp.bl = mp.b;
  if (ep.a_lo) {
    const __nv_bfloat16* Al = static_cast<const __nv_bfloat16*>(A) + ep.a_lo;
    const __nv_bfloat16* Bl = static_cast<const __nv_bfloat16*>(B) + ep.b_lo;
    rc = a_mn ? make_map(&mp.al, Al, K, M, lda, kBlockK, 64) : make_map(&mp.al, Al, M, K, lda, kBlockM);
    if (rc) return rc;
    rc = b_mn ? make_map(&mp.bl, Bl, K, N, ldb, kBlockK, 64) : make_map(&mp.bl, Bl, N, K, ldb, bn);
    if (rc) return rc;
  }
  float* part = splits > 1 || partial ? partial : nullptr;
  if (splits == 1 && !(ep.permP > 1 || ep.permQ > 1)) part = nullptr;
#define TB_TC_LAUNCH(BN, AM, BM) rc = launch<BN, AM, BM>(mp, ep, M, N, K, splits, part, stream)
  if (!a_mn && !b_mn) {
    if (bn == 32) TB_TC_LAUNCH(32, false, false);
    else if (bn == 64) TB_TC_LAUNCH(64, false, false);
    else TB_TC_LAUNCH(128, false, false);
  } else if (!a_mn && b_mn) {
    if (bn == 64) TB_TC_LAUNCH(64, false, true);
    else TB_TC_LAUNCH(128, false, true);
  } else {
    if (bn == 64) TB_TC_LAUNCH(64, true, true);
    else TB_TC_LAUNCH(128, true, true);
  }
#undef TB_TC_LAUNCH
  if (rc || !part) return rc;
  TB_REQUIRE(ep.C, "gemm_tc: split-K reduce needs an fp32 output");
  GemmEpilogue rep;
  rep.bias = ep.bias; rep.relu = ep.relu; rep.permP = ep.permP; rep.permQ = ep.permQ; rep.scale = ep.scale;
  return launch_splitk_reduce(part, ep.C, M, N, ep.ldc, splits, rep, (N + 31) & ~int64_t(31), stream);
}

// fp32 [rows, cols] (ld) -> bf16 [rows, cols16] (ld16), optional ReLU-free straight convert
__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t rows,
                                   int64_t cols, int64_t ld, int64_t ld16, int64_t lo_off) {
  const int64_t total = rows * ld16;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t r = i / ld16, c = i % ld16;
    const float x = c < cols ? in[r * ld + c] : 0.0f;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    out[i] = h;
    if (lo_off) out[lo_off + i] = bf16_lo_of(x, h);
  }
}

int f32_to_bf16(const float* in, void* out, int64_t rows, int64_t cols, int64_t ld, int64_t ld16, cudaStream_t stream,
                int64_t lo_off) {
  const int64_t total = rows * ld16;
  if (total == 0) return 0;
  ProfScope prof("f32_to_bf16", stream);
  int64_t blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  f32_to_bf16_kernel<<<(unsigned)blocks, 256, 0, stream>>>(in, static_cast<__nv_bfloat16*>(out), rows, cols, ld, ld16, lo_off);
  return check_launch("f32_to_bf16_kernel");
}

}  // namespace tb

using namespace tb;

extern "C" {

int tb_gemm_bf16_tn(const void* A_bf16, const void* B_bf16, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                    float* C, int64_t ldc, void* C_bf16, int64_t ldc16, const float* bias, float scale, int relu,
                    void* stream) {
  TcEpilogue ep;
  ep.C = C; ep.ldc = ldc; ep.C16 = static_cast<__nv_bfloat16*>(C_bf16); ep.ldc16 = ldc16; ep.bias = bias;
  ep.scale = scale; ep.relu = relu; ep.tag = "gemm_bf16_tn";
  return gemm_tc_bf16(A_bf16, B_bf16, M, N, K, lda, ldb, ep, (cudaStream_t)stream);
}

int tb_gemm_bf16_ex(const void* A_bf16, const void* B_bf16, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                    int a_mn, int b_mn, float* C, int64_t ldc, int splits, float* partial, void* stream) {
  TcEpilogue ep;
  ep.C = C; ep.ldc = ldc; ep.tag = "gemm_bf16_ex";
  return gemm_tc_bf16_ex(A_bf16, B_bf16, M, N, K, lda, ldb, a_mn != 0, b_mn != 0, ep, splits, partial, (cudaStream_t)stream);
}

int tb_f32_to_bf16(const float* in, void* out_bf16, int64_t rows, int64_t cols, int64_t ld, int64_t ld16, void* stream) {
  TB_REQUIRE(in && out_bf16, "tb_f32_to_bf16: null pointer");
  return f32_to_bf16(in, out_bf16, rows, cols, ld, ld16, (cudaStream_t)stream, 0);
}

}  // extern "C"
