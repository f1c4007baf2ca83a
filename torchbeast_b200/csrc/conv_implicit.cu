// Implicit-GEMM first convolution on tensor cores: the uint8 NCHW frames ARE the operand.
//
// AtariNet's conv1 (monobeast.py:560, 8x8 stride 4 over [N,4,84,84] uint8) as a patch-matrix GEMM reads a
// [N*400, 256] bf16 matrix that is 7x larger than the frames it was gathered from; materialising it costs
// more HBM time than the product itself (im2col, GEMM and wgrad are all bound by the 531 MB patch matrix).  Here the
// frames are converted ONCE to bf16 (exact:
// pixel values are integers <= 2^8; the 1/255 stays in the epilogue; 146 MB instead of 531 MB) and producer
// warps gather each patch row straight from that image with per-thread async copies (cp.async 8 B, L1/L2
// resident: every pixel is reused by 4 patches) into shared memory in the SWIZZLE_128B layout the wgmma
// descriptors expect, so the patch matrix never exists in HBM.  (A first version converted u8 -> bf16 inside
// the gather: ncu showed it issue-bound on the 4x redundant conversion, 23 instructions per 16-byte chunk.)
//
//   forward : act[m, o] = relu(scale * sum_k patch[m, k] * W[o, k] + b[o])     A gathered (K-major), B = W resident
//   wgrad   : dW[o, k]  = scale * sum_m dY[m, o] * patch[m, k]                 A = dY^T via TMA (MN-major),
//                                                                             B gathered (MN-major), split over m
//
// One kernel-height row of a patch (KW = 8 pixels of one channel) is 16 bytes of the bf16 image (8-byte
// aligned: two cp.async) and becomes one 16-byte swizzle chunk; a (patch, channel) pair is one 128-byte swizzle row (KH*KW = 64 values).  The same
// physical rows serve as a K-major A tile (forward: 128 patches x 64 k) and as an MN-major B box (wgrad:
// 64 patches x 64 k-values) - only the descriptor differs.
// Requirements (checked by conv_u8_implicit_applicable): KH = KW = 8, C = 4, O = 32, W % 4 == 0, S % 4 == 0.
#include "conv_implicit.cuh"

#include "gemm_simt.cuh"  // splitk_reduce_kernel / GemmEpilogue
#include "restack.cuh"
#include "tc_common.cuh"

namespace tb {

using namespace tcd;

namespace {

constexpr int kProducers = 256;                         // 8 gather warps
constexpr int kGatherBase = 9 * 32;                     // warps 0-7: two wgmma + epilogue warpgroups, 8: TMA, 9-16: gather
constexpr int kConvThreads = kGatherBase + kProducers;
constexpr int kC = 4;                           // input channels = k-blocks of 64 (= KH*KW)
constexpr int kO = 32;                          // output channels
constexpr int kStagesF = 3;   // forward: a stage is a WHOLE 128-patch tile (4 k-blocks, 64 KB), so the consumers pay one
                              // mbarrier wait and one wgmma wait per tile instead of one per k-block
constexpr int kStagesW = 5;   // wgrad: 5 x (8 KB dY + 32 KB patches)

struct ConvGeom {
  int H, W, S, OH, OW;
  int per;        // patches per frame = OH*OW
  uint32_t magic; // ceil(2^20 / OW): (rem * magic) >> 20 == rem / OW for rem < per (checked on the host)
  int64_t M;      // patches = N*OH*OW
};

// Patch index as (frame, index within the frame), advanced by a constant stride: the gather threads walk
// patches in arithmetic progression, so the 64-bit division happens once per thread, not once per stage
// (the first version divided per stage and ncu showed the XU pipe 96 % busy with reciprocals).
struct PatchIter {
  int64_t n;
  int rem;
  __device__ __forceinline__ void init(const ConvGeom& g, int64_t m) {
    if (m >= g.M) m = g.M - 1;  // rows past the end: forward never stores them; their dY rows are TMA zero fill
    n = m / g.per;
    rem = int(m - n * g.per);
  }
  __device__ __forceinline__ void advance(const ConvGeom& g, int dn, int drem) {
    n += dn; rem += drem;
    if (rem >= g.per) { rem -= g.per; ++n; }
  }
  // element offset of the top-left pixel in channel 0; frames past the end clamp to the last patch
  __device__ __forceinline__ int64_t origin(const ConvGeom& g, int64_t nframes) const {
    int64_t nn = n; int r = rem;
    if (nn >= nframes) { nn = nframes - 1; r = g.per - 1; }
    const int oy = int((uint32_t(r) * g.magic) >> 20), ox = r - oy * g.OW;
    return (nn * kC * g.H + int64_t(oy) * g.S) * g.W + int64_t(ox) * g.S;
  }
};

// One 16-byte swizzle chunk = 8 bf16 pixels at an 8-byte aligned global address = two async 8-byte copies,
// issued by an even/odd lane PAIR: 16 rows x 2 halves per warp instruction cover all 32 banks exactly twice
// (2 shared-memory wavefronts per 256 B; one lane writing both halves of its own row cost 8, and ncu showed
// the L1/shared data pipe, not HBM or issue, bounding the kernel).
__device__ __forceinline__ void copy8(uint32_t saddr, const __nv_bfloat16* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(saddr), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- forward ---------------------------------------------------------------------------------------
// Persistent over 128-patch tiles.  Stage s of the A ring holds the tile's k-block of channel c (ring
// position runs on), filled by all 256 gather threads: thread p owns patch row p & 127 and kernel rows
// [4*(p>>7), +4).  The next tile's 32 words are loaded before the current tile is converted, so one
// global-load latency is exposed per tile, not per stage.
// SPLIT (split-bf16): the pixel operand is exact in bf16, so only the weights carry a lo plane (resident next to the
// hi plane, tmBl) - two MMAs per k-step, patch.Wlo then patch.Whi - and the output is written as hi / lo planes.
template <bool SPLIT>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_u8_fwd_implicit_kernel(const __nv_bfloat16* __restrict__ frame, const __grid_constant__ CUtensorMap tmB,
                            const __grid_constant__ CUtensorMap tmBl, TcEpilogue ep, ConvGeom g, int tiles_m) {
  constexpr uint32_t B_BYTES = kO * kBlockK * 2;  // 4 KB per k-block
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t kTileBytes = kC * kABytes;  // 64 KB
  const uint32_t sA = base, sB = base + kStagesF * kTileBytes;
  const uint32_t bars = sB + (SPLIT ? 2 : 1) * kC * B_BYTES;  // full[kStagesF], empty[kStagesF], wfull
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kStagesF + s); };
  const uint32_t wfull = bars + 8u * (2 * kStagesF);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < kStagesF; ++s) { mbar_init(full(s), kProducers / 32); mbar_init(empty(s), 8); }
    mbar_init(wfull, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {  // the whole weight matrix [32, 256] stays resident: one box per k-block
      mbar_expect_tx(wfull, (SPLIT ? 2 : 1) * kC * B_BYTES);
      for (int c = 0; c < kC; ++c) tma_load_2d(sB + c * B_BYTES, &tmB, wfull, c * kBlockK, 0);
      if constexpr (SPLIT)
        for (int c = 0; c < kC; ++c) tma_load_2d(sB + (kC + c) * B_BYTES, &tmBl, wfull, c * kBlockK, 0);
    }
  } else if (warp < 8) {
    // consumer warpgroup h: the 64-row half h of the tile, an m64n32 accumulator; the epilogue works on the fragments
    // (rows fr, fr + 8, column pairs 8j + fc)
    const int h = warp >> 2;
    const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);
    float bias_r[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { bias_r[2 * j] = __ldg(ep.bias + 8 * j + fc); bias_r[2 * j + 1] = __ldg(ep.bias + 8 * j + fc + 1); }
    mbar_wait(wfull, 0);
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < tiles_m; tile += gridDim.x) {
      float acc[kO / 2];
      mbar_wait(full(stage), phase);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < kC; ++c)
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          const uint64_t da = make_smem_desc(sA + stage * kTileBytes + c * kABytes + h * 8192 + k * 32);
          if constexpr (SPLIT) {
            wgmma_bf16<kO>(acc, da, make_smem_desc(sB + (kC + c) * B_BYTES + k * 32), (c | k) != 0);
            wgmma_bf16<kO>(acc, da, make_smem_desc(sB + c * B_BYTES + k * 32), 1);
          } else {
            wgmma_bf16<kO>(acc, da, make_smem_desc(sB + c * B_BYTES + k * 32), (c | k) != 0);
          }
        }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(stage));  // values are in registers: free the stage early
      if (++stage == kStagesF) { stage = 0; phase ^= 1; }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t r = int64_t(tile) * kBlockM + h * 64 + fr + 8 * e;
        if (r >= g.M) continue;
        __nv_bfloat16* c = ep.C16 + r * ep.ldc16;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float x0 = acc[4 * j + 2 * e] * ep.scale + bias_r[2 * j];
          float x1 = acc[4 * j + 2 * e + 1] * ep.scale + bias_r[2 * j + 1];
          if (ep.relu) { x0 = fmaxf(x0, 0.0f); x1 = fmaxf(x1, 0.0f); }
          uint32_t hi, lo;
          split_bf16x2(x0, x1, hi, lo);
          *reinterpret_cast<uint32_t*>(c + 8 * j + fc) = hi;
          if (SPLIT && ep.c16_lo) *reinterpret_cast<uint32_t*>(c + ep.c16_lo + 8 * j + fc) = lo;
        }
      }
    }
  } else {
    const int p = threadIdx.x - kGatherBase;
    const int half = lane & 1;                       // which 8 bytes of every chunk
    const int row = (p >> 5) * 16 + (lane >> 1);     // 16 patch rows per gather warp
    const uint32_t row_off = uint32_t(row >> 3) * 1024u + uint32_t(row & 7) * 128u + 8u * half;
    const int rr = row & 7;
    // async gather of a whole tile per stage, signalled one tile behind the issue point
    constexpr int kLag = 1;
    int stage = 0; uint32_t phase = 0;
    int sig = 0;       // next stage to signal
    int pending = 0;   // issued, not yet signalled
    const int64_t nframes = g.M / g.per;
    const int64_t stride = int64_t(kBlockM) * gridDim.x;
    const int dn = int(stride / g.per), drem = int(stride % g.per);
    PatchIter it;
    it.init(g, int64_t(blockIdx.x) * kBlockM + row);
    for (int tile = blockIdx.x; tile < tiles_m; tile += gridDim.x, it.advance(g, dn, drem)) {
      const __nv_bfloat16* src0 = frame + it.origin(g, nframes) + 4 * half;
      mbar_wait(empty(stage), phase ^ 1);
#pragma unroll
      for (int c = 0; c < kC; ++c) {
        const uint32_t dst = sA + stage * kTileBytes + c * kABytes + row_off;
        const __nv_bfloat16* src = src0 + int64_t(c) * g.H * g.W;
#pragma unroll
        for (int j = 0; j < 8; ++j) copy8(dst + (uint32_t(j ^ rr) << 4), src + j * g.W);
      }
      cp_commit();
      if (++stage == kStagesF) { stage = 0; phase ^= 1; }
      if (++pending > kLag) {
        cp_wait<kLag>();
        fence_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(full(sig));  // one arrival per gather warp
        if (++sig == kStagesF) sig = 0;
        --pending;
      }
    }
    cp_wait<0>();
    fence_async_smem();
    __syncwarp();
    for (; pending > 0; --pending) {
      if (lane == 0) mbar_arrive(full(sig));
      if (++sig == kStagesF) sig = 0;
    }
  }
}

// ---- weight gradient -------------------------------------------------------------------------------
// D[o (padded to 128), k = 256] accumulates over this CTA's slice of 64-patch blocks; stage = A: two
// 64(o) x 64(patch) TMA boxes of dY (columns >= 32 are out of bounds -> zero), B: four 64(patch) x 64(k)
// gathered boxes (one per channel).  Gather thread p owns patch row p & 63 of channel p >> 6.
// SPLIT (split-bf16): dY arrives as hi / lo planes (tmA / tmAl, two boxes per stage), the pixels are exact:
// two MMAs per k-step, dYlo.patch then dYhi.patch.
template <bool SPLIT>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_u8_wgrad_implicit_kernel(const __nv_bfloat16* __restrict__ frame, const __grid_constant__ CUtensorMap tmA,
                              const __grid_constant__ CUtensorMap tmAl, ConvGeom g, float* __restrict__ partial, int total_kb,
                              int per) {
  constexpr int kStW = SPLIT ? kStagesW - 1 : kStagesW;  // 4 x 48 KB (split) / 5 x 40 KB
  constexpr uint32_t B_BYTES = kC * 8192;  // 32 KB
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t A_BOX = 8192;   // one 64-wide box of dY^T: rows >= 32 of the m64 accumulator are zero fill
  constexpr uint32_t A_BYTES = (SPLIT ? 2u : 1u) * A_BOX;  // [hi][lo]
  const uint32_t sA = base, sB = base + kStW * A_BYTES;
  const uint32_t bars = sB + kStW * B_BYTES;  // full[kStW], empty[kStW]
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kStW + s); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb0 = blockIdx.x * per;
  const int kb1 = (kb0 + per < total_kb) ? kb0 + per : total_kb;
  const int num_kb = kb1 > kb0 ? kb1 - kb0 : 0;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < kStW; ++s) { mbar_init(full(s), kProducers / 32 + 1); mbar_init(empty(s), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int i = 0; i < num_kb; ++i) {
        const int kc = (kb0 + i) * kBlockK;  // first patch of the block
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(full(stage), A_BYTES);
        tma_load_2d(sA + stage * A_BYTES, &tmA, full(stage), 0, kc);
        if constexpr (SPLIT) tma_load_2d(sA + stage * A_BYTES + A_BOX, &tmAl, full(stage), 0, kc);
        if (++stage == kStW) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < 8) {
    // D[o, k]: warpgroup q owns columns [128q, 128q + 128) (two of the four gathered 64-wide k groups, 8192 B apart) as
    // an m64n128 accumulator, o < 32 real
    constexpr int NQ = kC * 64 / 2;
    const int q = warp >> 2;
    float acc[NQ / 2];
#pragma unroll
    for (int j = 0; j < NQ / 2; ++j) acc[j] = 0.0f;
    int stage = 0; uint32_t phase = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full(stage), phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
        const uint64_t db = make_smem_desc_mn(sB + stage * B_BYTES + q * 2 * 8192 + k * 2048);
        if constexpr (SPLIT) {
          wgmma_bf16<NQ, 1, 1>(acc, make_smem_desc_mn(sA + stage * A_BYTES + A_BOX + k * 2048), db, (kb | k) != 0);
          wgmma_bf16<NQ, 1, 1>(acc, make_smem_desc_mn(sA + stage * A_BYTES + k * 2048), db, 1);
        } else {
          wgmma_bf16<NQ, 1, 1>(acc, make_smem_desc_mn(sA + stage * A_BYTES + k * 2048), db, (kb | k) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(stage));
      if (++stage == kStW) { stage = 0; phase ^= 1; }
    }
    if ((warp & 3) < 2) {  // fragment rows 0..31 = the 32 real output channels
      const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float* pz = partial + (int64_t(blockIdx.x) * kO + fr + 8 * e) * (kC * 64) + q * NQ;
#pragma unroll
        for (int j = 0; j < NQ / 8; ++j)
          *reinterpret_cast<float2*>(pz + 8 * j + fc) = make_float2(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]);
      }
    }
  } else {
    const int p = threadIdx.x - kGatherBase;
    const int half = lane & 1;
    const int c = p >> 6;                                      // two gather warps per channel
    const int row = ((p >> 5) & 1) * 32 + (lane >> 1);         // this thread's rows: row and row + 16
    const uint32_t row_off = uint32_t(c) * 8192u + uint32_t(row >> 3) * 1024u + uint32_t(row & 7) * 128u + 8u * half;
    const int rr = row & 7;                                    // (row + 16) & 7 is the same
    constexpr int kLag = 2;  // ring 5: three stages of slack between the signalled and the freed position
    int stage = 0; uint32_t phase = 0;
    int sig = 0, pending = 0;
    const int64_t nframes = g.M / g.per;
    const int dn = kBlockK / g.per, drem = kBlockK % g.per;
    PatchIter itA, itB;
    itA.init(g, int64_t(kb0) * kBlockK + row);
    itB.init(g, int64_t(kb0) * kBlockK + row + 16);
    // init() clamps to the last patch; past-the-end blocks only occur in this CTA's final stage
    const int64_t chan = int64_t(c) * g.H * g.W + 4 * half;
    for (int i = 0; i < num_kb; ++i, itA.advance(g, dn, drem), itB.advance(g, dn, drem)) {
      const __nv_bfloat16* srcA = frame + itA.origin(g, nframes) + chan;
      const __nv_bfloat16* srcB = frame + itB.origin(g, nframes) + chan;
      mbar_wait(empty(stage), phase ^ 1);
      const uint32_t dst = sB + stage * B_BYTES + row_off;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        copy8(dst + (uint32_t(j ^ rr) << 4), srcA + j * g.W);
        copy8(dst + 2048u + (uint32_t(j ^ rr) << 4), srcB + j * g.W);  // row + 16: two 8-row groups further
      }
      cp_commit();
      if (++stage == kStW) { stage = 0; phase ^= 1; }
      if (++pending > kLag) {
        cp_wait<kLag>();
        fence_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(full(sig));
        if (++sig == kStW) sig = 0;
        --pending;
      }
    }
    cp_wait<0>();
    fence_async_smem();
    __syncwarp();
    for (; pending > 0; --pending) {
      if (lane == 0) mbar_arrive(full(sig));
      if (++sig == kStW) sig = 0;
    }
  }
}

// 16 pixels per thread: one 16-byte load, two 16-byte stores; u8 -> bf16 via the exact 2^23 + v float trick
__device__ __forceinline__ uint32_t u8pair_to_bf16x2(uint32_t w, uint32_t sel0, uint32_t sel1) {
  const float f0 = __uint_as_float(__byte_perm(w, 0x4B000000u, sel0)) - 8388608.0f;
  const float f1 = __uint_as_float(__byte_perm(w, 0x4B000000u, sel1)) - 8388608.0f;
  return __byte_perm(__float_as_uint(f0), __float_as_uint(f1), 0x7632);
}
__global__ void frames_u8_to_bf16_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t count) {
  const int64_t nvec = count >> 4;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(in) + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o[2 * j] = u8pair_to_bf16x2(w[j], 0x7650, 0x7651);
      o[2 * j + 1] = u8pair_to_bf16x2(w[j], 0x7652, 0x7653);
    }
    uint4* dst = reinterpret_cast<uint4*>(out) + 2 * i;
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (int64_t i = nvec << 4; i < count; ++i) out[i] = __float2bfloat16_rn(float(in[i]));
}

// the same image from an unstacked rollout: vector i of plane (n, c) is read from the row unstacked_row() names
__global__ void frames_u8_unstacked_to_bf16_kernel(const uint8_t* __restrict__ frames, const uint8_t* __restrict__ done,
                                                   int64_t T1, int64_t B, int64_t vpp, __nv_bfloat16* __restrict__ out) {
  const int64_t nvec = T1 * B * 4 * vpp;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const int64_t plane = i / vpp;
    const int c = int(plane & 3);
    const int64_t n = plane >> 2, t = n / B, b = n - t * B;
    const int64_t row = unstacked_row(done, t, b, B, c);
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(frames) + (row * B + b) * vpp + (i - plane * vpp));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o[2 * j] = u8pair_to_bf16x2(w[j], 0x7650, 0x7651);
      o[2 * j + 1] = u8pair_to_bf16x2(w[j], 0x7652, 0x7653);
    }
    uint4* dst = reinterpret_cast<uint4*>(out) + 2 * i;
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

ConvGeom make_geom(int64_t N, int H, int W, int S) {
  ConvGeom g;
  g.H = H; g.W = W; g.S = S; g.OH = (H - 8) / S + 1; g.OW = (W - 8) / S + 1;
  g.per = g.OH * g.OW;
  g.magic = uint32_t(((1u << 20) + g.OW - 1) / g.OW);
  g.M = N * g.per;
  return g;
}

}  // namespace

int frames_u8_to_bf16(const uint8_t* frame, void* frame_bf16, int64_t count, cudaStream_t stream) {
  TB_REQUIRE(frame && frame_bf16 && (reinterpret_cast<uintptr_t>(frame) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(frame_bf16) & 15) == 0,
             "frames_u8_to_bf16: null or unaligned pointer");
  if (count == 0) return 0;
  ProfScope prof("frames_to_bf16", stream);
  int64_t blocks = ((count >> 4) + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  if (blocks < 1) blocks = 1;
  frames_u8_to_bf16_kernel<<<(unsigned)blocks, 256, 0, stream>>>(frame, static_cast<__nv_bfloat16*>(frame_bf16), count);
  return check_launch("frames_u8_to_bf16_kernel");
}

int frames_u8_unstacked_to_bf16(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW,
                                void* frame_bf16, cudaStream_t stream) {
  TB_REQUIRE(frames && done && frame_bf16 && (reinterpret_cast<uintptr_t>(frames) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(frame_bf16) & 15) == 0,
             "frames_u8_unstacked_to_bf16: null or unaligned pointer");
  TB_REQUIRE(HW % 16 == 0, "frames_u8_unstacked_to_bf16: HW must be a multiple of 16");
  ProfScope prof("frames_to_bf16", stream);
  const int64_t vpp = HW / 16;
  int64_t blocks = (T1 * B * 4 * vpp + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  if (blocks < 1) blocks = 1;
  frames_u8_unstacked_to_bf16_kernel<<<(unsigned)blocks, 256, 0, stream>>>(frames, done, T1, B, vpp,
                                                                           static_cast<__nv_bfloat16*>(frame_bf16));
  return check_launch("frames_u8_unstacked_to_bf16_kernel");
}

bool conv_u8_implicit_applicable(int C, int H, int W, int KH, int KW, int S, int O) {
  if (!(C == kC && KH == 8 && KW == 8 && O == kO && (W % 4) == 0 && (S % 4) == 0 && H >= 8 && W >= 8)) return false;
  const ConvGeom g = make_geom(1, H, W, S);
  if (g.per > 4096) return false;
  for (int r = 0; r < g.per; ++r)  // the multiply-shift division the gather threads use must be exact
    if (int((uint32_t(r) * g.magic) >> 20) != r / g.OW) return false;
  return true;
}

int conv_u8_fwd_implicit(const void* frame_bf16, const void* w_bf16, int64_t N, int H, int W, int S, const TcEpilogue& ep,
                         cudaStream_t stream) {
  const __nv_bfloat16* frame = static_cast<const __nv_bfloat16*>(frame_bf16);
  TB_REQUIRE(frame && w_bf16 && ep.C16 && ep.bias && ep.ldc16 == kO, "conv_u8_fwd_implicit: bad arguments");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(frame) & 7) == 0 && (reinterpret_cast<uintptr_t>(ep.C16) & 15) == 0,
             "conv_u8_fwd_implicit: unaligned pointer");
  if (N == 0) return 0;
  ProfScope prof(ep.tag, stream);
  const ConvGeom g = make_geom(N, H, W, S);
  CUtensorMap mb, mbl;
  int rc = make_map(&mb, w_bf16, kO, kC * 64, kC * 64, kO);
  if (rc) return rc;
  mbl = mb;
  const bool split = ep.b_lo != 0;
  if (split) {
    rc = make_map(&mbl, static_cast<const __nv_bfloat16*>(w_bf16) + ep.b_lo, kO, kC * 64, kC * 64, kO);
    if (rc) return rc;
  }
  constexpr size_t smem = 1024 + kStagesF * size_t(kC) * kABytes + 2 * kC * (kO * kBlockK * 2) + 8 * (2 * kStagesF + 5) + 16;
  static uint64_t attr = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  if (!((attr >> (dev & 63)) & 1)) {
    cudaError_t e = cudaFuncSetAttribute(conv_u8_fwd_implicit_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(conv_u8_fwd_implicit_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "conv_u8_fwd_implicit: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr |= uint64_t(1) << (dev & 63);
  }
  const int64_t tiles = (g.M + kBlockM - 1) / kBlockM;
  TB_REQUIRE(tiles < (int64_t(1) << 31), "conv_u8_fwd_implicit: too many tiles");
  const int64_t grid = tiles < kNumSMs ? tiles : kNumSMs;
  if (split) conv_u8_fwd_implicit_kernel<true><<<(unsigned)grid, kConvThreads, smem, stream>>>(frame, mb, mbl, ep, g, int(tiles));
  else conv_u8_fwd_implicit_kernel<false><<<(unsigned)grid, kConvThreads, smem, stream>>>(frame, mb, mbl, ep, g, int(tiles));
  return check_launch("conv_u8_fwd_implicit_kernel");
}

int conv_u8_wgrad_implicit(const void* dy_bf16, const void* frame_bf16, int64_t N, int H, int W, int S, float* dW, float scale,
                           float* partial, int64_t partial_floats, const char* tag, cudaStream_t stream, int64_t dy_lo) {
  const __nv_bfloat16* frame = static_cast<const __nv_bfloat16*>(frame_bf16);
  TB_REQUIRE(frame && dy_bf16 && dW && partial, "conv_u8_wgrad_implicit: null pointer");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(frame) & 7) == 0, "conv_u8_wgrad_implicit: unaligned frame pointer");
  ProfScope prof(tag, stream);
  const ConvGeom g = make_geom(N, H, W, S);
  const int64_t total_kb = (g.M + kBlockK - 1) / kBlockK;
  TB_REQUIRE(total_kb >= 1 && total_kb < (int64_t(1) << 31), "conv_u8_wgrad_implicit: bad size");
  int64_t grid = total_kb < kNumSMs ? total_kb : kNumSMs;
  const int64_t per = (total_kb + grid - 1) / grid;
  grid = (total_kb + per - 1) / per;
  TB_REQUIRE(grid * kO * kC * 64 <= partial_floats, "conv_u8_wgrad_implicit: partial buffer too small");
  CUtensorMap ma, mal;  // dY [M, 32] with the patch index as the reduction (row) index: MN-major boxes of 64 x 64
  int rc = make_map(&ma, dy_bf16, g.M, kO, kO, kBlockK, 64);
  if (rc) return rc;
  mal = ma;
  if (dy_lo) {
    rc = make_map(&mal, static_cast<const __nv_bfloat16*>(dy_bf16) + dy_lo, g.M, kO, kO, kBlockK, 64);
    if (rc) return rc;
  }
  constexpr size_t smem = 1024 + kStagesW * (8192 + size_t(kC) * 8192) + 8 * (2 * kStagesW + 1) + 16;  // >= the split ring (4 x 48 KB)
  static_assert(smem <= 227 * 1024 && smem >= 1024 + (kStagesW - 1) * (2 * 8192 + size_t(kC) * 8192) + 8 * (2 * kStagesW + 1) + 16,
                "conv_u8_wgrad_implicit: ring size");
  static uint64_t attr = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  if (!((attr >> (dev & 63)) & 1)) {
    cudaError_t e = cudaFuncSetAttribute(conv_u8_wgrad_implicit_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(conv_u8_wgrad_implicit_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "conv_u8_wgrad_implicit: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr |= uint64_t(1) << (dev & 63);
  }
  if (dy_lo)
    conv_u8_wgrad_implicit_kernel<true><<<(unsigned)grid, kConvThreads, smem, stream>>>(frame, ma, mal, g, partial, int(total_kb), int(per));
  else
    conv_u8_wgrad_implicit_kernel<false><<<(unsigned)grid, kConvThreads, smem, stream>>>(frame, ma, mal, g, partial, int(total_kb), int(per));
  rc = check_launch("conv_u8_wgrad_implicit_kernel");
  if (rc) return rc;
  GemmEpilogue rep;
  rep.scale = scale;
  return launch_splitk_reduce(partial, dW, kO, kC * 64, kC * 64, int(grid), rep, kC * 64, stream);
}

}  // namespace tb
