// Shifted-window implicit-GEMM 3x3 convolutions (stride 1, pad 1) of the IMPALA ResNet trunk on wgmma
// (reference: torchbeast/polybeast_learner.py:141-199, nn.Conv2d(kernel_size=3, stride=1, padding=1)).
//
// These convolutions have 16 / 32 channels: as GEMMs they are [pixels, 9*C] x [9*C, 16..32] - the A stream is everything.
// A patch matrix (or a per-tap TMA box) moves every input element 9-12 times through the TMA -> shared-memory path, and
// that path, not HBM and not the tensor pipe, bounds patch-matrix kernels.  Here the image is stored as zero-padded CHANNEL-CHUNK PLANES [frame][C/8][(H+2)*(W+2)][8] (split-bf16: hi
// and lo planes).  A tile = 128 consecutive flattened padded pixels of one frame; its input window (128 + 2*(W+2) + 2
// pixels of every chunk plane) is ONE contiguous 1-D bulk copy per plane.  In shared memory a chunk plane is a K-major
// no-swizzle wgmma operand as it stands - row = pixel, 16 bytes = 8 channels, rows 16 bytes apart (canonical layout
// ((8,n),2):((1,SBO),LBO) in 16-byte units with SBO = 8 and LBO = the chunk-plane pitch) - and the operand of tap (kh, kw)
// is the same rows shifted by (kh*(W+2) + kw)*16 bytes: 9 descriptors over one copy of the data.  Output rows that fall on
// padding columns / rows are computed and dropped by the epilogue (2/(W+2) of the tile).
//
// Split-bf16 (see gemm_tc.cuh): x = hi + lo per operand, products x_hi.w_hi + x_hi.w_lo + x_lo.w_hi in fp32.  The
// weight rows are stored [w_hi | w_lo] so that x_hi.[w_hi | w_lo] is ONE MMA with N = 2*NO (the A operand is read from
// shared memory once for both products); x_lo.w_hi accumulates onto the first half and the epilogue adds the halves.
// The epilogue can also write the NEXT conv's padded image (and per-tile column sums = its bias gradient in the backward
// pass), so most fp32 -> image passes do not exist.  Weight gradients (M = 16..32 output channels: a shape the 64-row wgmma
// atom cannot fill) run on mma.sync.m16n8k16 from the same planar tiles (sw_conv_wgrad_kernel).
#include "conv3x3_sw.cuh"

#include "tc_common.cuh"
#include "restack.cuh"

namespace tb {

using namespace tcd;

namespace {

constexpr int kTile = 128;
constexpr int kSwStages = 4;

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// K-major, no swizzle: rows 16 B apart inside an 8-row core matrix, 8-row groups `sbo` bytes apart, the second 8-element
// k-chunk `lbo` bytes away
__device__ __forceinline__ uint64_t desc_k_noswz(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return uint64_t((saddr & 0x3FFFF) >> 4) | (uint64_t(lbo >> 4) << 16) | (uint64_t(sbo >> 4) << 32);  // layout 0: no swizzle
}
struct SwGeom {
  int H, W, Wp, Hp;
  int pin;        // pixels of the input window of one tile, multiple of 8
  int tpf;        // tiles per frame
  int vend;       // flattened padded pixels that can hold an output: (H-1)*Wp + W
  int64_t plane;  // elements of one chunk plane: Hp*Wp*8
};

inline SwGeom sw_geom(int H, int W) {
  SwGeom g;
  g.H = H; g.W = W; g.Wp = W + 2; g.Hp = H + 2;
  g.pin = (kTile + 2 * g.Wp + 2 + 7) & ~7;
  g.vend = (H - 1) * g.Wp + W;
  g.tpf = (g.vend + kTile - 1) / kTile;
  g.plane = int64_t(g.Hp) * g.Wp * 8;
  return g;
}

struct SwFwdArgs {
  const __nv_bfloat16* img; int64_t img_lo;
  const __nv_bfloat16* wk;
  float* out; const float* bias; const float* mask; const float* addend; float scale;
  // optional second output: the result (through ReLU if emit_relu) as the padded planar hi / lo image of the NEXT conv (same
  // spatial size, NO channels), borders and slack included; and per (tile, epilogue warp) column sums of the result
  // (csum[(tile*4 + warp)*NO + c]: the bias gradient when the result is a dY)
  __nv_bfloat16* emit; int64_t emit_lo; int emit_relu; float* csum;
  int Nf; SwGeom g;
};

// persistent: CTA walks (frame, tile) work items; warp 8 = bulk-copy producer, warps 0..7 = two consumer warpgroups, group g
// owning the CTA's even / odd tiles: each issues the wgmma of its tile and runs its epilogue, so one group's epilogue (global
// loads of mask / residual, ~10 16-byte stores per row) overlaps the other group's MMAs.  The accumulator fragments go
// through a per-group shared-memory staging tile so that each thread of the group owns one row in the epilogue.
constexpr int kSwThreads = 9 * 32;
template <int CK, int NO>
__global__ void __launch_bounds__(kSwThreads, 1) sw_conv_fwd_kernel(SwFwdArgs a) {
  constexpr int CH = CK / 8;                   // chunk planes per frame
  constexpr int KP = CK / 16;                  // k16 steps per tap
  constexpr uint32_t W_PLANE = 9u * CK * NO * 2u;   // bytes of one weight plane (the image interleaves hi and lo rows)
  constexpr int LDS = NO + 4;                  // staging row pitch in floats
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 127u) & ~127u;
  const uint32_t chb = uint32_t(a.g.pin) * 16u;     // bytes of one chunk plane window
  const uint32_t stage_bytes = 2u * CH * chb;       // [plane hi / lo][chunk][pixel][16 B]
  const uint32_t sW = base;                         // [tap][kp][j][hi rows | lo rows][16 B]
  const uint32_t sX = sW + 2u * W_PLANE;
  const uint32_t bars = sX + kSwStages * stage_bytes;  // full[kSt], empty[kSt], wbar, then the two staging tiles
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kSwStages + s); };
  const uint32_t wbar = bars + 8u * (2 * kSwStages);
  __shared__ float csum_s[8][32][NO + 1];   // column-sum staging of the eight epilogue warps

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_work = a.Nf * a.g.tpf;
  if (warp == 8 && lane == 0) {
    for (int s = 0; s < kSwStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 4); }
    mbar_init(wbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(wbar, 2u * W_PLANE);
      bulk_g2s(sW, a.wk, 2u * W_PLANE, wbar);
      int stage = 0; uint32_t phase = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int n = w / a.g.tpf, p0 = (w - n * a.g.tpf) * kTile;
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(full(stage), stage_bytes);
        const uint32_t st = sX + stage * stage_bytes;
#pragma unroll
        for (int pl = 0; pl < 2; ++pl)
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const __nv_bfloat16* src = a.img + (pl ? a.img_lo : 0) + (int64_t(n) * CH + c) * a.g.plane + int64_t(p0) * 8;
            bulk_g2s(st + (pl * CH + c) * chb, src, chb, full(stage));
          }
        if (++stage == kSwStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int quarter = warp & 3, ew = warp, grp = ew >> 2;
    const int rl = quarter * 32 + lane;
    float* stg = reinterpret_cast<float*>(smem_raw + (wbar + 16u - smem_addr(smem_raw))) + grp * kTile * LDS;
    mbar_wait(wbar, 0);
    for (int w = blockIdx.x + grp * gridDim.x, it = grp; w < total_work; w += 2 * gridDim.x, it += 2) {
      const int stage = it % kSwStages;
      const uint32_t phase = uint32_t(it / kSwStages) & 1u;
      const int n = w / a.g.tpf, p = (w - n * a.g.tpf) * kTile + rl;
      const int y = p / a.g.Wp, x = p - y * a.g.Wp;
      const bool valid = x < a.g.W && y < a.g.H;
      const int64_t r = (int64_t(n) * a.g.H + y) * a.g.W + x;
      if (valid) {  // pull the mask / residual rows towards L2 while the MMAs run
        if (a.mask) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.mask + r * NO));
        if (a.addend) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.addend + r * NO));
      }
      // The split product as TWO wgmmas per k-step: x_hi . [w_hi | w_lo] (N = 2*NO, the lo half lands in columns [NO, 2*NO))
      // and x_lo . w_hi accumulated onto columns [0, NO) - the first NO/2 registers of the 2*NO-wide accumulator.
      float acc[2][NO];  // rows [0, 64) and [64, 128) of the tile
      mbar_wait(full(stage), phase);
      wgmma_fence();
      const uint32_t st = sX + stage * stage_bytes;
      // fully unrolled: the first product's scale-d flag is then a constant - with a runtime flag in a rolled loop ptxas
      // serialises the whole wgmma chain
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const uint32_t shift = uint32_t((tap / 3) * a.g.Wp + (tap % 3)) * 16u;
#pragma unroll
        for (int kp = 0; kp < KP; ++kp) {
          const uint32_t wa = sW + uint32_t((tap * KP + kp) * 2 * 2 * NO) * 16u;
          const uint64_t dbw = desc_k_noswz(wa, 2u * NO * 16u, 128u);   // rows [0, NO) = hi, [NO, 2*NO) = lo
#pragma unroll
          for (int h = 0; h < 2; ++h) {  // 64 pixel rows = 1024 B further
            const uint32_t xa = st + uint32_t(2 * kp) * chb + shift + h * 1024u;
            const uint64_t dah = desc_k_noswz(xa, chb, 128u), dal = desc_k_noswz(xa + CH * chb, chb, 128u);
            wgmma_bf16<2 * NO>(acc[h], dah, dbw, (tap | kp) != 0);
            wgmma_bf16<NO>(acc[h], dal, dbw, 1);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(stage));   // the values are in registers: the stage can be refilled
      named_sync(1 + grp, 128);  // this group's previous epilogue has read the staging tile
      {
        // lo.hi + hi.hi (columns [0, NO)) + hi.lo (columns [NO, 2*NO)): registers i and i + NO/2
        const int fr = quarter * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < NO / 8; ++j) {
            float* sp = stg + (h * 64 + fr) * LDS + 8 * j + fc;
            *reinterpret_cast<float2*>(sp) = make_float2(acc[h][4 * j] + acc[h][4 * j + NO / 2], acc[h][4 * j + 1] + acc[h][4 * j + 1 + NO / 2]);
            *reinterpret_cast<float2*>(sp + 8 * LDS) =
                make_float2(acc[h][4 * j + 2] + acc[h][4 * j + 2 + NO / 2], acc[h][4 * j + 3] + acc[h][4 * j + 3 + NO / 2]);
          }
      }
      named_sync(1 + grp, 128);
      float o[NO];
#pragma unroll
      for (int j = 0; j < NO; ++j) o[j] = 0.f;
      if (valid) {
#pragma unroll
        for (int j = 0; j < NO; j += 4) {
          const float4 t = *reinterpret_cast<const float4*>(stg + rl * LDS + j);
          o[j] = t.x * a.scale; o[j + 1] = t.y * a.scale; o[j + 2] = t.z * a.scale; o[j + 3] = t.w * a.scale;
        }
        if (a.bias) {
#pragma unroll
          for (int q = 0; q < NO / 4; ++q) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.bias) + q);
            o[4 * q] += b4.x; o[4 * q + 1] += b4.y; o[4 * q + 2] += b4.z; o[4 * q + 3] += b4.w;
          }
        }
        if (a.mask) {
          const float4* mp = reinterpret_cast<const float4*>(a.mask + r * NO);
#pragma unroll
          for (int q = 0; q < NO / 4; ++q) {
            const float4 m4 = __ldg(mp + q);
            o[4 * q] = m4.x > 0.f ? o[4 * q] : 0.f; o[4 * q + 1] = m4.y > 0.f ? o[4 * q + 1] : 0.f;
            o[4 * q + 2] = m4.z > 0.f ? o[4 * q + 2] : 0.f; o[4 * q + 3] = m4.w > 0.f ? o[4 * q + 3] : 0.f;
          }
        }
        if (a.addend) {
          const float4* ap = reinterpret_cast<const float4*>(a.addend + r * NO);
#pragma unroll
          for (int q = 0; q < NO / 4; ++q) {
            const float4 a4 = __ldg(ap + q);
            o[4 * q] += a4.x; o[4 * q + 1] += a4.y; o[4 * q + 2] += a4.z; o[4 * q + 3] += a4.w;
          }
        }
        float4* op = reinterpret_cast<float4*>(a.out + r * NO);
#pragma unroll
        for (int q = 0; q < NO / 4; ++q) op[q] = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
      }
      if (a.emit) {
        // Tile row p (an output pixel or a padding position of the flattened grid) is pixel p + Wp + 1 of the next image:
        // valid rows carry the result, the others are exactly that image's side borders; the top border, what the last
        // tile does not reach of the bottom border, and the slack behind the image are zeroed by the first / last tile.
        const int hpwp = a.g.Hp * a.g.Wp, t = w - n * a.g.tpf;
        const int64_t fbase = int64_t(n) * (NO / 8) * hpwp;
        auto put = [&](int q, int c, uint4 ph, uint4 pl) {
          __nv_bfloat16* dst = a.emit + (fbase + int64_t(c) * hpwp + q) * 8;
          *reinterpret_cast<uint4*>(dst) = ph;
          *reinterpret_cast<uint4*>(dst + a.emit_lo) = pl;
        };
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        const int q = p + a.g.Wp + 1;
        if (q < hpwp) {
#pragma unroll
          for (int c = 0; c < NO / 8; ++c) {
            uint4 ph, pl;
            float e[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) e[j] = a.emit_relu ? fmaxf(o[8 * c + j], 0.f) : o[8 * c + j];
            split_bf16x2(e[0], e[1], ph.x, pl.x); split_bf16x2(e[2], e[3], ph.y, pl.y);
            split_bf16x2(e[4], e[5], ph.z, pl.z); split_bf16x2(e[6], e[7], ph.w, pl.w);
            put(q, c, ph, pl);
          }
        }
        // pixels [0, Wp + 1): the top border and the first left border - 129 of them at W = 126, one more than a tile
        // has rows
        for (int u = rl; t == 0 && u < a.g.Wp + 1; u += kTile) {
#pragma unroll
          for (int c = 0; c < NO / 8; ++c) put(u, c, z, z);
        }
        if (t == a.g.tpf - 1) {
          const int q2 = a.g.tpf * kTile + a.g.Wp + 1 + rl;
          if (q2 < hpwp) {
#pragma unroll
            for (int c = 0; c < NO / 8; ++c) put(q2, c, z, z);
          }
        }
        if (w == 0) {   // slack behind the last frame (see zero_slack_units)
          const int64_t body = int64_t(a.Nf) * (NO / 8) * hpwp * 8;
          for (int u = rl; u < a.g.pin + 8; u += 128) {
            *reinterpret_cast<uint4*>(a.emit + body + int64_t(u) * 8) = z;
            *reinterpret_cast<uint4*>(a.emit + a.emit_lo + body + int64_t(u) * 8) = z;
          }
        }
      }
      if (a.csum) {   // per (tile, warp) column sums in a fixed order: rows of padding positions hold zeros
#pragma unroll
        for (int j = 0; j < NO; ++j) csum_s[ew][lane][j] = o[j];
        __syncwarp();
        if (lane < NO) {
          float sum = 0.f;
#pragma unroll 8
          for (int rr = 0; rr < 32; ++rr) sum += csum_s[ew][rr][lane];
          a.csum[(int64_t(w) * 4 + quarter) * NO + lane] = sum;
        }
        __syncwarp();
      }
    }
  }
}

// dynamic shared memory of the forward kernel: weights, kSwStages input windows of `pin` pixels, barriers, staging tiles
inline size_t sw_fwd_smem(int pin, int CK, int NO) {
  return 128 + 2 * size_t(9) * CK * NO * 2 + size_t(kSwStages) * 2 * (CK / 8) * pin * 16 + 8 * (2 * kSwStages + 2) +
         2 * size_t(kTile) * (NO + 4) * sizeof(float) + 16;
}

template <int CK, int NO>
int launch_sw_fwd(const SwFwdArgs& a, cudaStream_t stream) {
  const size_t smem = sw_fwd_smem(a.g.pin, CK, NO);
  TB_REQUIRE(smem <= 227 * 1024, "sw_conv_fwd: shared memory");
  static size_t attr[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr[dev & 63] < smem) {
    cudaError_t e = cudaFuncSetAttribute(sw_conv_fwd_kernel<CK, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "sw_conv_fwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr[dev & 63] = smem;
  }
  int per_sm = int((224 * 1024) / (smem + sizeof(float) * 8 * 32 * (NO + 1) + 1024));   // + the static column-sum staging
  if (per_sm > 4) per_sm = 4;
  if (per_sm < 1) per_sm = 1;
  int64_t grid = int64_t(kNumSMs) * per_sm;
  const int64_t total = int64_t(a.Nf) * a.g.tpf;
  if (grid > total) grid = total;
  sw_conv_fwd_kernel<CK, NO><<<(unsigned)grid, kSwThreads, smem, stream>>>(a);
  return check_launch("sw_conv_fwd_kernel");
}

// ---- forward with a 64-channel side (or a 32 -> 32 row too wide for the kernel above) -------------------------------
// The kernel above keeps all weights resident and a whole tile's window (every chunk plane) per ring stage: at 64 -> 64
// and W = 63 that is 144 KiB of weights + 4 x 66 KiB of windows.  This one (any pair with CK or NO = 64, and the 16 / 32
// pairs the kernel above does not fit, e.g. 32 -> 32 at W = 63 in a 32-wide first section) changes two things and keeps
// the image format, the tile, the split product and the epilogue:
//   - output columns in blocks of NT = min(NO, 32): a CTA owns ONE block (blockIdx.x % NCB, the grid is a multiple of
//     NCB) and keeps only that block's weights (<= 72 KiB); the CTAs of the NCB blocks of a tile read its window from L2;
//   - the window is streamed one k16 step (2 chunk planes, hi + lo) per ring stage, KP = CK/16 stages per tile, accumulating
//     into the same registers.  Each consumer group has its own 2-stage ring: a group then waits only on stages it released
//     itself, so a parity wait cannot match a phase two rounds old however many stages a tile takes.
// Shared memory at the widest rows the nets use: 64 -> 64 at W = 63: 72 KiB weights + 4 x 16.5 KiB stages + 2 x 18 KiB
// staging + 33 KiB column-sum staging = 207 KiB; 16 -> 64 at W = 126: 18 + 4 x 24.5 + 36 + 33 = 185 KiB.
constexpr int kWideGroupStages = 2;
constexpr int kWideStages = 2 * kWideGroupStages;

template <int CK, int NO>
__global__ void __launch_bounds__(kSwThreads, 1) sw_conv_fwd_wide_kernel(SwFwdArgs a) {
  constexpr int CH = CK / 8, KP = CK / 16;
  constexpr int NT = NO < 32 ? NO : 32, NCB = NO / NT;
  constexpr uint32_t W_BLOCK = 36u * CK * NT;       // bytes of one column block's [w_hi | w_lo] operand
  constexpr int LDS = NT + 4;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 127u) & ~127u;
  const uint32_t chb = uint32_t(a.g.pin) * 16u;
  const uint32_t stage_bytes = 4u * chb;            // [plane hi / lo][chunk 2*ks / 2*ks + 1][pixel][16 B]
  const uint32_t sW = base;
  const uint32_t sX = sW + W_BLOCK;
  const uint32_t bars = sX + kWideStages * stage_bytes;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kWideStages + s); };
  const uint32_t wbar = bars + 8u * (2 * kWideStages);
  __shared__ float csum_s[8][32][NT + 1];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cb = blockIdx.x % NCB, G = gridDim.x / NCB, wb = blockIdx.x / NCB;
  const int total_work = a.Nf * a.g.tpf;
  if (warp == 8 && lane == 0) {
    for (int s = 0; s < kWideStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 4); }
    mbar_init(wbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(wbar, W_BLOCK);
      bulk_g2s(sW, a.wk + int64_t(cb) * (W_BLOCK / 2), W_BLOCK, wbar);
      int cnt0 = 0, cnt1 = 0;   // ring items issued per consumer group
      for (int w = wb, it = 0; w < total_work; w += G, ++it) {
        const int grp = it & 1;
        const int n = w / a.g.tpf, p0 = (w - n * a.g.tpf) * kTile;
#pragma unroll
        for (int ks = 0; ks < KP; ++ks) {
          const int item = grp ? cnt1++ : cnt0++;
          const int stage = grp * kWideGroupStages + item % kWideGroupStages;
          mbar_wait(empty(stage), (uint32_t(item / kWideGroupStages) & 1u) ^ 1u);
          mbar_expect_tx(full(stage), stage_bytes);
          const uint32_t st = sX + stage * stage_bytes;
#pragma unroll
          for (int pl = 0; pl < 2; ++pl)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const __nv_bfloat16* src =
                  a.img + (pl ? a.img_lo : 0) + (int64_t(n) * CH + 2 * ks + j) * a.g.plane + int64_t(p0) * 8;
              bulk_g2s(st + (pl * 2 + j) * chb, src, chb, full(stage));
            }
        }
      }
    }
  } else {
    const int quarter = warp & 3, ew = warp, grp = ew >> 2;
    const int rl = quarter * 32 + lane;
    float* stg = reinterpret_cast<float*>(smem_raw + (wbar + 16u - smem_addr(smem_raw))) + grp * kTile * LDS;
    const int c0 = cb * NT;   // first output column of this CTA
    mbar_wait(wbar, 0);
    int item = 0;
    for (int w = wb + grp * G; w < total_work; w += 2 * G) {
      const int n = w / a.g.tpf, p = (w - n * a.g.tpf) * kTile + rl;
      const int y = p / a.g.Wp, x = p - y * a.g.Wp;
      const bool valid = x < a.g.W && y < a.g.H;
      const int64_t r = (int64_t(n) * a.g.H + y) * a.g.W + x;
      if (valid) {
        if (a.mask) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.mask + r * NO + c0));
        if (a.addend) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.addend + r * NO + c0));
      }
      float acc[2][NT];
#pragma unroll
      for (int ks = 0; ks < KP; ++ks, ++item) {
        const int stage = grp * kWideGroupStages + item % kWideGroupStages;
        mbar_wait(full(stage), uint32_t(item / kWideGroupStages) & 1u);
        wgmma_fence();
        const uint32_t st = sX + stage * stage_bytes;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t shift = uint32_t((tap / 3) * a.g.Wp + (tap % 3)) * 16u;
          const uint32_t wa = sW + uint32_t((tap * KP + ks) * 2 * 2 * NT) * 16u;
          const uint64_t dbw = desc_k_noswz(wa, 2u * NT * 16u, 128u);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t xa = st + shift + h * 1024u;
            const uint64_t dah = desc_k_noswz(xa, chb, 128u), dal = desc_k_noswz(xa + 2u * chb, chb, 128u);
            wgmma_bf16<2 * NT>(acc[h], dah, dbw, (ks | tap) != 0);
            wgmma_bf16<NT>(acc[h], dal, dbw, 1);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(stage));
      }
      named_sync(1 + grp, 128);
      {
        const int fr = quarter * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) {
            float* sp = stg + (h * 64 + fr) * LDS + 8 * j + fc;
            *reinterpret_cast<float2*>(sp) = make_float2(acc[h][4 * j] + acc[h][4 * j + NT / 2], acc[h][4 * j + 1] + acc[h][4 * j + 1 + NT / 2]);
            *reinterpret_cast<float2*>(sp + 8 * LDS) =
                make_float2(acc[h][4 * j + 2] + acc[h][4 * j + 2 + NT / 2], acc[h][4 * j + 3] + acc[h][4 * j + 3 + NT / 2]);
          }
      }
      named_sync(1 + grp, 128);
      float o[NT];
#pragma unroll
      for (int j = 0; j < NT; ++j) o[j] = 0.f;
      if (valid) {
#pragma unroll
        for (int j = 0; j < NT; j += 4) {
          const float4 t = *reinterpret_cast<const float4*>(stg + rl * LDS + j);
          o[j] = t.x * a.scale; o[j + 1] = t.y * a.scale; o[j + 2] = t.z * a.scale; o[j + 3] = t.w * a.scale;
        }
        if (a.bias) {
#pragma unroll
          for (int q = 0; q < NT / 4; ++q) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.bias + c0) + q);
            o[4 * q] += b4.x; o[4 * q + 1] += b4.y; o[4 * q + 2] += b4.z; o[4 * q + 3] += b4.w;
          }
        }
        if (a.mask) {
          const float4* mp = reinterpret_cast<const float4*>(a.mask + r * NO + c0);
#pragma unroll
          for (int q = 0; q < NT / 4; ++q) {
            const float4 m4 = __ldg(mp + q);
            o[4 * q] = m4.x > 0.f ? o[4 * q] : 0.f; o[4 * q + 1] = m4.y > 0.f ? o[4 * q + 1] : 0.f;
            o[4 * q + 2] = m4.z > 0.f ? o[4 * q + 2] : 0.f; o[4 * q + 3] = m4.w > 0.f ? o[4 * q + 3] : 0.f;
          }
        }
        if (a.addend) {
          const float4* ap = reinterpret_cast<const float4*>(a.addend + r * NO + c0);
#pragma unroll
          for (int q = 0; q < NT / 4; ++q) {
            const float4 a4 = __ldg(ap + q);
            o[4 * q] += a4.x; o[4 * q + 1] += a4.y; o[4 * q + 2] += a4.z; o[4 * q + 3] += a4.w;
          }
        }
        float4* op = reinterpret_cast<float4*>(a.out + r * NO + c0);
#pragma unroll
        for (int q = 0; q < NT / 4; ++q) op[q] = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
      }
      if (a.emit) {   // as in sw_conv_fwd_kernel, for this CTA's chunk planes c0/8 .. (c0 + NT)/8 - 1
        const int hpwp = a.g.Hp * a.g.Wp, t = w - n * a.g.tpf;
        const int64_t fbase = (int64_t(n) * (NO / 8) + c0 / 8) * hpwp;
        auto put = [&](int q, int c, uint4 ph, uint4 pl) {
          __nv_bfloat16* dst = a.emit + (fbase + int64_t(c) * hpwp + q) * 8;
          *reinterpret_cast<uint4*>(dst) = ph;
          *reinterpret_cast<uint4*>(dst + a.emit_lo) = pl;
        };
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        const int q = p + a.g.Wp + 1;
        if (q < hpwp) {
#pragma unroll
          for (int c = 0; c < NT / 8; ++c) {
            uint4 ph, pl;
            float e[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) e[j] = a.emit_relu ? fmaxf(o[8 * c + j], 0.f) : o[8 * c + j];
            split_bf16x2(e[0], e[1], ph.x, pl.x); split_bf16x2(e[2], e[3], ph.y, pl.y);
            split_bf16x2(e[4], e[5], ph.z, pl.z); split_bf16x2(e[6], e[7], ph.w, pl.w);
            put(q, c, ph, pl);
          }
        }
        for (int u = rl; t == 0 && u < a.g.Wp + 1; u += kTile) {   // as in sw_conv_fwd_kernel
#pragma unroll
          for (int c = 0; c < NT / 8; ++c) put(u, c, z, z);
        }
        if (t == a.g.tpf - 1) {
          const int q2 = a.g.tpf * kTile + a.g.Wp + 1 + rl;
          if (q2 < hpwp) {
#pragma unroll
            for (int c = 0; c < NT / 8; ++c) put(q2, c, z, z);
          }
        }
        if (w == 0 && cb == 0) {
          const int64_t body = int64_t(a.Nf) * (NO / 8) * hpwp * 8;
          for (int u = rl; u < a.g.pin + 8; u += 128) {
            *reinterpret_cast<uint4*>(a.emit + body + int64_t(u) * 8) = z;
            *reinterpret_cast<uint4*>(a.emit + a.emit_lo + body + int64_t(u) * 8) = z;
          }
        }
      }
      if (a.csum) {
#pragma unroll
        for (int j = 0; j < NT; ++j) csum_s[ew][lane][j] = o[j];
        __syncwarp();
        if (lane < NT) {
          float sum = 0.f;
#pragma unroll 8
          for (int rr = 0; rr < 32; ++rr) sum += csum_s[ew][rr][lane];
          a.csum[(int64_t(w) * 4 + quarter) * NO + c0 + lane] = sum;
        }
        __syncwarp();
      }
    }
  }
}

// dynamic shared memory of the wide forward kernel (+ its static column-sum staging, which counts against the same 227 KiB)
inline size_t sw_fwd_wide_smem(int pin, int CK, int NO) {
  const int NT = NO < 32 ? NO : 32;
  return 128 + size_t(36) * CK * NT + size_t(kWideStages) * 4 * pin * 16 + 8 * (2 * kWideStages + 2) +
         2 * size_t(kTile) * (NT + 4) * sizeof(float) + 16;
}
inline size_t sw_fwd_wide_static(int NO) { return sizeof(float) * 8 * 32 * ((NO < 32 ? NO : 32) + 1); }

template <int CK, int NO>
int launch_sw_fwd_wide(const SwFwdArgs& a, cudaStream_t stream) {
  constexpr int NCB = NO < 32 ? 1 : NO / 32;
  const size_t smem = sw_fwd_wide_smem(a.g.pin, CK, NO);
  TB_REQUIRE(smem + sw_fwd_wide_static(NO) <= 227 * 1024, "sw_conv_fwd: shared memory");
  static size_t attr[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr[dev & 63] < smem) {
    cudaError_t e = cudaFuncSetAttribute(sw_conv_fwd_wide_kernel<CK, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "sw_conv_fwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr[dev & 63] = smem;
  }
  int per_sm = int((224 * 1024) / (smem + sw_fwd_wide_static(NO) + 1024));
  if (per_sm > 4) per_sm = 4;
  if (per_sm < 1) per_sm = 1;
  int64_t groups = int64_t(kNumSMs) * per_sm / NCB;   // CTAs per column block
  const int64_t total = int64_t(a.Nf) * a.g.tpf;
  if (groups > total) groups = total;
  if (groups < 1) groups = 1;
  sw_conv_fwd_wide_kernel<CK, NO><<<(unsigned)(groups * NCB), kSwThreads, smem, stream>>>(a);
  return check_launch("sw_conv_fwd_wide_kernel");
}

// ---- weight gradient ------------------------------------------------------------------------------------------
// dW[o, tap, c] = sum over pixels p of dY[p, o] * x[p + shift(tap), c]: M = O and N = C are 16..32 and the reduction runs
// over pixels.  A wgmma atom is 64 rows, so three quarters of every MMA would be padding.  The
// warp-level mma.sync.m16n8k16 atom fits exactly (M = 16 channels of dY, N = 8 channels of x, K = 16 pixels): A = dY^T and B = the x window both come straight out of the planar tiles with ldmatrix.trans (a
// row of either tile is one pixel's 8 channels = 16 bytes, 8 consecutive pixels are one 8x8 matrix), the tap shift is a
// 16-byte multiple in the row address, and the products are split-bf16 (lo.hi + hi.lo + hi.hi).
// CTA = 9 MMA warps = 3 tap groups (one kernel row each) x 3 pixel groups (k16 steps kg, kg+3, kg+6 of a tile) + 1 producer
// warp issuing the same bulk copies as the forward kernel; accumulators stay in registers over all of the CTA's tiles, are
// folded over the pixel groups through shared memory and written to partial[cta][o][tap*C + c] (folded in CTA order by
// sw_wgrad_reduce_kernel: deterministic).
constexpr int kWgStages = 3;
constexpr int kWgMinW = 5;   // 2*(W + 2) + 2 >= 15: the zero run behind a frame's last pixel covers the last k16 step
constexpr int kWgWarps = 9;
constexpr int kWgThreads = (kWgWarps + 1) * 32;

struct SwWgradArgs {
  const __nv_bfloat16* dy; int64_t dy_lo;
  const __nv_bfloat16* x; int64_t x_lo;
  float* partial;
  int Nf; SwGeom g;
};

__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 64-channel sides: a CTA computes one (OT x CT) block of dW (OT, CT <= 32, block blockIdx.y of the O/OT x C/CT blocks),
// loading only that block's dY and input chunk planes - the accumulators and the fold buffer are those of a 32 x 32 conv.
// The blocks of a tile re-read its planes from L2 (each chunk plane is loaded by C/CT or O/OT blocks).
template <int CF, int OF, int C = CF, int O = OF>
__global__ void __launch_bounds__(kWgThreads, 1) sw_conv_wgrad_kernel(SwWgradArgs a) {
  constexpr int CC = C / 8, CO = O / 8, MT = O / 16, NP = C / 16;   // chunk planes; m16 tiles; pairs of n8 tiles
  constexpr int CCF = CF / 8, COF = OF / 8, NBC = CF / C;           // chunk planes of the whole images; C blocks
  const int blk = (NBC * (OF / O) > 1) ? int(blockIdx.y) : 0;
  const int cc0 = (blk % NBC) * CC, co0 = (blk / NBC) * CO;         // first chunk plane of this block's x / dY
  constexpr uint32_t DY_CH = kTile * 16u;            // bytes of one dY chunk plane tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_addr(smem_raw) + 127u) & ~127u;
  const uint32_t chb = uint32_t(a.g.pin) * 16u;
  const uint32_t dy_bytes = 2u * CO * DY_CH, x_bytes = 2u * CC * chb;
  const uint32_t stage_bytes = dy_bytes + x_bytes;   // [dY hi chunks][dY lo chunks][x hi chunks][x lo chunks]
  const uint32_t bars = base;                        // full[kSt], empty[kSt]
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (kWgStages + s); };
  const uint32_t sS = base + 128u;
  float* red = reinterpret_cast<float*>(smem_raw + ((sS - smem_addr(smem_raw)) + kWgStages * stage_bytes));   // [9*C][O + 1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_work = a.Nf * a.g.tpf;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kWgStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), kWgWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kWgWarps) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int n = w / a.g.tpf, p0 = (w - n * a.g.tpf) * kTile;
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(full(stage), stage_bytes);
        const uint32_t st = sS + stage * stage_bytes;
#pragma unroll
        for (int pl = 0; pl < 2; ++pl) {
#pragma unroll
          for (int c = 0; c < CO; ++c) {   // output pixel p is padded pixel p + Wp + 1 of the dY image
            const __nv_bfloat16* src =
                a.dy + (pl ? a.dy_lo : 0) + (int64_t(n) * COF + co0 + c) * a.g.plane + int64_t(p0 + a.g.Wp + 1) * 8;
            bulk_g2s(st + (pl * CO + c) * DY_CH, src, DY_CH, full(stage));
          }
#pragma unroll
          for (int c = 0; c < CC; ++c) {
            const __nv_bfloat16* src = a.x + (pl ? a.x_lo : 0) + (int64_t(n) * CCF + cc0 + c) * a.g.plane + int64_t(p0) * 8;
            bulk_g2s(st + dy_bytes + (pl * CC + c) * chb, src, chb, full(stage));
          }
        }
        if (++stage == kWgStages) { stage = 0; phase ^= 1; }
      }
    }
    // falls through to the fold below (takes no part in it)
  }
  const int tg = warp % 3, kg = warp / 3;      // kernel row of this warp's 3 taps; pixel group (MMA warps only)
  float acc[3][MT][2 * NP][4];
#pragma unroll
  for (int t = 0; t < 3; ++t)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < 2 * NP; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[t][mt][nt][e] = 0.f;
  if (warp < kWgWarps) {
    int stage = 0; uint32_t phase = 0;
    // ldmatrix row addresses: lane -> (matrix = lane / 8, row = lane % 8)
    //   A (dY^T, m16 x k16): matrices (m half, k half) = (0,0), (1,0), (0,1), (1,1): chunk plane = 2*mt + (mat & 1), pixel = 8*(mat >> 1) + row
    //   B (x, k16 x 2 n8 tiles): matrices (n tile, k half) = (0,0), (0,1), (1,0), (1,1): chunk plane = 2*np + (mat >> 1), pixel = 8*(mat & 1) + row
    const int mat = lane >> 3, row = lane & 7;
    const uint32_t a_off = uint32_t(mat & 1) * DY_CH + uint32_t(8 * (mat >> 1) + row) * 16u;
    const uint32_t b_off = uint32_t(mat >> 1) * chb + uint32_t(8 * (mat & 1) + row) * 16u;
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
      const int n = w / a.g.tpf, p0 = (w - n * a.g.tpf) * kTile;
      // pixels past the frame's last output row alias the next chunk plane: stop at the 16-pixel step that covers the last
      // valid pixel (the rest of that step, up to 15 pixels, falls into the 2*Wp + 2 zero pixels that follow in the dY image:
      // the last row's right border, the bottom border, the next plane's top border and first left border - 15 or more
      // only for W >= kWgMinW, which sw_conv_wgrad requires)
      int ksteps = (a.g.vend - p0 + 15) / 16;
      if (ksteps > kTile / 16) ksteps = kTile / 16;
      mbar_wait(full(stage), phase);
      const uint32_t st = sS + stage * stage_bytes;
      const uint32_t dyh = st, dyl = st + CO * DY_CH, xh = st + dy_bytes, xl = xh + CC * chb;
      for (int ks = kg; ks < ksteps; ks += 3) {
        uint32_t ah[MT][4], al[MT][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          ldsm_x4_t(ah[mt], dyh + uint32_t(2 * mt) * DY_CH + uint32_t(ks) * 256u + a_off);
          ldsm_x4_t(al[mt], dyl + uint32_t(2 * mt) * DY_CH + uint32_t(ks) * 256u + a_off);
        }
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const uint32_t shift = uint32_t(tg * a.g.Wp + t) * 16u + uint32_t(ks) * 256u;
#pragma unroll
          for (int np = 0; np < NP; ++np) {
            uint32_t bh[4], bl[4];
            ldsm_x4_t(bh, xh + uint32_t(2 * np) * chb + shift + b_off);
            ldsm_x4_t(bl, xl + uint32_t(2 * np) * chb + shift + b_off);
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
              mma16816(acc[t][mt][2 * np], al[mt], bh[0], bh[1]);
              mma16816(acc[t][mt][2 * np], ah[mt], bl[0], bl[1]);
              mma16816(acc[t][mt][2 * np], ah[mt], bh[0], bh[1]);
              mma16816(acc[t][mt][2 * np + 1], al[mt], bh[2], bh[3]);
              mma16816(acc[t][mt][2 * np + 1], ah[mt], bl[2], bl[3]);
              mma16816(acc[t][mt][2 * np + 1], ah[mt], bh[2], bh[3]);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(stage));
      if (++stage == kWgStages) { stage = 0; phase ^= 1; }
    }
  }
  // fold the three pixel groups (fixed order kg = 0, 1, 2) into red[col = tap*C + c][o], then one coalesced store
  constexpr int LDR = O + 1;
  for (int g = 0; g < 3; ++g) {
    if (warp < kWgWarps && kg == g) {
#pragma unroll
      for (int t = 0; t < 3; ++t)
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int nt = 0; nt < 2 * NP; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int o = mt * 16 + (lane >> 2) + (e >> 1) * 8;
              const int col = (tg * 3 + t) * C + nt * 8 + (lane & 3) * 2 + (e & 1);
              float* d = red + col * LDR + o;
              *d = (g == 0) ? acc[t][mt][nt][e] : *d + acc[t][mt][nt][e];
            }
    }
    __syncthreads();
  }
  float* dst = a.partial + (int64_t(blk) * gridDim.x + blockIdx.x) * O * (9 * C);
  for (int i = threadIdx.x; i < O * 9 * C; i += kWgThreads) {
    const int o = i / (9 * C), col = i - o * (9 * C);
    dst[i] = red[col * LDR + o];
  }
}

// dW[o, c, kh, kw] = scale * sum over CTAs of partial[cta][o][(kh*3 + kw)*C + c].  Block = 32 consecutive partial columns x 8
// CTA groups (coalesced 128-byte reads; a per-thread loop over every CTA's partial with strided reads took longer than
// a third of the weight-gradient kernels themselves); the 8 group sums are folded in a fixed order (deterministic).
__global__ void __launch_bounds__(256) sw_wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dW, int ctas,
                                                              int O, int C, int c_real, float scale) {
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int q = blockIdx.x * 32 + lane;          // column of the [O][9*C] partial matrix
  const int total = O * 9 * C;
  float s = 0.f;
  if (q < total)
    for (int b = g; b < ctas; b += 8) s += partial[int64_t(b) * total + q];
  red[g][lane] = s;
  __syncthreads();
  if (g == 0 && q < total) {
    float t = red[0][lane];
#pragma unroll
    for (int k = 1; k < 8; ++k) t += red[k][lane];
    const int o = q / (9 * C), col = q - o * (9 * C);
    const int tap = col / C, c = col - tap * C;
    if (c < c_real) dW[(int64_t(o) * c_real + c) * 9 + tap] = t * scale;
  }
}

// dynamic shared memory of the weight-gradient kernel: kWgStages (dY tile + input window) stages and the fold buffer
inline size_t sw_wgrad_smem(int pin, int C, int O) {
  return 384 + size_t(kWgStages) * (2 * size_t(O / 8) * kTile * 16 + 2 * size_t(C / 8) * pin * 16) + sizeof(float) * 9 * C * (O + 1);
}

// the (C, O) block a CTA of the weight gradient computes: the whole conv when both sides are 16 or 32, else 32-channel
// blocks of the 64-channel sides
inline int sw_wgrad_block(int n) { return n < 32 ? n : 32; }

template <int C, int O, int CT = C, int OT = O>
int launch_sw_wgrad(const SwWgradArgs& a, int grid, cudaStream_t stream) {
  const size_t smem = sw_wgrad_smem(a.g.pin, CT, OT);
  TB_REQUIRE(smem <= 227 * 1024, "sw_conv_wgrad: shared memory");
  static size_t attr[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (attr[dev & 63] < smem) {
    cudaError_t e = cudaFuncSetAttribute(sw_conv_wgrad_kernel<C, O, CT, OT>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    TB_REQUIRE(e == cudaSuccess, "sw_conv_wgrad: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr[dev & 63] = smem;
  }
  sw_conv_wgrad_kernel<C, O, CT, OT><<<dim3(grid, (C / CT) * (O / OT)), kWgThreads, smem, stream>>>(a);
  return check_launch("sw_conv_wgrad_kernel");
}

static inline unsigned sgrid(int64_t work, int threads) {
  int64_t blocks = (work + threads - 1) / threads;
  const int64_t cap = int64_t(kNumSMs) * 16;
  if (blocks > cap) blocks = cap;
  return (unsigned)(blocks < 1 ? 1 : blocks);
}

// The weight-gradient kernel's last k16 step of a frame reads up to 15 pixels past the frame's last chunk plane (multiplied by
// the zeros of the dY image's padding): for the last frame that is the slack behind the image, which must hold finite
// values - stale memory can be a NaN pattern and 0 * NaN poisons the accumulator.  The first block of an image producer
// zeroes the slack of both planes (`units` 16-byte units starting `body` elements into a plane).
__device__ __forceinline__ void zero_slack_units(__nv_bfloat16* out, int64_t lo_off, int64_t body, int units) {
  for (int u = threadIdx.x; u < units; u += blockDim.x) {
    *reinterpret_cast<uint4*>(out + body + int64_t(u) * 8) = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(out + lo_off + body + int64_t(u) * 8) = make_uint4(0u, 0u, 0u, 0u);
  }
}

// q / d for 0 <= q < 2^22 and d < 2^10 without the integer-division sequence (ncu: these index kernels were instruction-issue
// bound with the XU pipe saturated by 32-bit divisions): one float multiply + a fix-up
__device__ __forceinline__ int fast_div(int q, int d, float inv_d) {
  int r = __float2int_rd((float(q) + 0.5f) * inv_d);
  r -= (r * d > q);
  r += ((r + 1) * d <= q);
  return r;
}

// one thread = 8 channels of one padded pixel (borders written as zeros every time: the buffers are shared between images);
// block = 256 / C8 consecutive padded pixels of frame blockIdx.y x all chunk planes (32-bit index arithmetic: one division).
// COLSUM: block partial sums of the C channels -> partial[(frame * gridDim.x + blockIdx.x) * C + c]
template <bool COLSUM>
__global__ void __launch_bounds__(256) sw_pad_split_kernel(const float4* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                                           int64_t lo_off, int H, int W, int C8, int relu_in,
                                                           float* __restrict__ partial, int slack_units) {
  const int Hp = H + 2, Wp = W + 2;
  if (blockIdx.x == 0 && blockIdx.y == 0) zero_slack_units(out, lo_off, int64_t(gridDim.y) * C8 * Hp * Wp * 8, slack_units);
  const int lc = (C8 == 8) ? 3 : (C8 == 4) ? 2 : (C8 == 2 ? 1 : 0);   // C8 is 1, 2, 4 or 8
  const int cv = threadIdx.x & (C8 - 1);
  const int p = blockIdx.x * (256 >> lc) + (threadIdx.x >> lc);
  const int64_t n = blockIdx.y;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (p < Hp * Wp) {
    const int py = fast_div(p, Wp, 1.0f / float(Wp)), px = p - py * Wp;
    uint4 ph = make_uint4(0u, 0u, 0u, 0u), pl = ph;
    if (py >= 1 && py <= H && px >= 1 && px <= W) {
      const float4* src = x + (((n * H + (py - 1)) * W + (px - 1)) * C8 + cv) * 2;
      float4 a = __ldg(src), b = __ldg(src + 1);
      if (relu_in) {
        a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
        b.x = fmaxf(b.x, 0.f); b.y = fmaxf(b.y, 0.f); b.z = fmaxf(b.z, 0.f); b.w = fmaxf(b.w, 0.f);
      }
      if (COLSUM) { acc[0] = a.x; acc[1] = a.y; acc[2] = a.z; acc[3] = a.w; acc[4] = b.x; acc[5] = b.y; acc[6] = b.z; acc[7] = b.w; }
      split_bf16x2(a.x, a.y, ph.x, pl.x); split_bf16x2(a.z, a.w, ph.y, pl.y);
      split_bf16x2(b.x, b.y, ph.z, pl.z); split_bf16x2(b.z, b.w, ph.w, pl.w);
    }
    __nv_bfloat16* dst = out + ((n * C8 + cv) * int64_t(Hp) * Wp + p) * 8;
    *reinterpret_cast<uint4*>(dst) = ph;
    *reinterpret_cast<uint4*>(dst + lo_off) = pl;
  }
  if (COLSUM) {
    __shared__ float red[256][9];
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x][j] = acc[j];
    __syncthreads();
    if (int(threadIdx.x) < C8 * 8) {   // thread t holds chunk t % C8: channel c = 8*(t % C8) + j
      const int c8 = threadIdx.x / 8, j = threadIdx.x % 8;
      float s = 0.f;
      for (int t = c8; t < 256; t += C8) s += red[t][j];   // fixed order
      partial[(n * gridDim.x + blockIdx.x) * (C8 * 8) + c8 * 8 + j] = s;
    }
  }
}

// Max-pool backward fused with the image producer: the gradient of the feat conv's output (dL/dP, [N, H, W, C]) is only ever
// consumed as the dY image of that conv's backward (and its column sums = the bias gradient), so it is gathered from the
// pooled gradient dyp [N, OH, OW, C] through the recorded argmax taps (gather form of nn.MaxPool2d(3, 2, 1) backward: pixel
// (iy, ix) sums the <= 4 windows whose first maximum it was) straight into the padded planar hi / lo image - no fp32
// [N, H, W, C] round trip.  Same grid / column-sum scheme as sw_pad_split_kernel<true>.
__global__ void __launch_bounds__(256) sw_pool_bwd_image_kernel(const uint8_t* __restrict__ arg, const float4* __restrict__ dyp,
                                                                __nv_bfloat16* __restrict__ out, int64_t lo_off, int H, int W, int OH,
                                                                int OW, int C8, float* __restrict__ partial, int slack_units) {
  const int Hp = H + 2, Wp = W + 2;
  if (blockIdx.x == 0 && blockIdx.y == 0) zero_slack_units(out, lo_off, int64_t(gridDim.y) * C8 * Hp * Wp * 8, slack_units);
  const int lc = (C8 == 8) ? 3 : (C8 == 4) ? 2 : (C8 == 2 ? 1 : 0);
  const int cv = threadIdx.x & (C8 - 1);
  const int p = blockIdx.x * (256 >> lc) + (threadIdx.x >> lc);
  const int64_t n = blockIdx.y;
  float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (p < Hp * Wp) {
    const int py = fast_div(p, Wp, 1.0f / float(Wp)), px = p - py * Wp;
    uint4 ph = make_uint4(0u, 0u, 0u, 0u), pl = ph;
    if (py >= 1 && py <= H && px >= 1 && px <= W) {
      const int iy = py - 1, ix = px - 1;
      // the <= 4 windows (oy, ox) in {iy/2, (iy+1)/2} x {ix/2, (ix+1)/2} (same order as maxpool_bwd_kernel: bit-identical sums);
      // all loads first, then byte-wise compares of the 8 recorded taps against this pixel's tap
      const int oy0 = iy >> 1, ox0 = ix >> 1;
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int oy = oy0 + a;
        if ((a == 1 && (iy & 1) == 0) || oy >= OH) continue;     // even iy: (iy+1)/2 == iy/2
        const int kh = iy - (oy * 2 - 1);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int ox = ox0 + b;
          if ((b == 1 && (ix & 1) == 0) || ox >= OW) continue;
          const uint32_t tapv = uint32_t(kh * 3 + (ix - (ox * 2 - 1))) * 0x01010101u;
          const int64_t o = ((n * OH + oy) * OW + ox) * C8 + cv;            // 8-channel group of the pooled pixel
          const float4 d0 = __ldg(dyp + o * 2), d1 = __ldg(dyp + o * 2 + 1);
          const uint2 am = __ldg(reinterpret_cast<const uint2*>(arg) + o);  // 8 argmax bytes
          const uint32_t m0 = __vcmpeq4(am.x, tapv), m1 = __vcmpeq4(am.y, tapv);
          g[0] += (m0 & 0x000000ffu) ? d0.x : 0.f; g[1] += (m0 & 0x0000ff00u) ? d0.y : 0.f;
          g[2] += (m0 & 0x00ff0000u) ? d0.z : 0.f; g[3] += (m0 & 0xff000000u) ? d0.w : 0.f;
          g[4] += (m1 & 0x000000ffu) ? d1.x : 0.f; g[5] += (m1 & 0x0000ff00u) ? d1.y : 0.f;
          g[6] += (m1 & 0x00ff0000u) ? d1.z : 0.f; g[7] += (m1 & 0xff000000u) ? d1.w : 0.f;
        }
      }
      split_bf16x2(g[0], g[1], ph.x, pl.x); split_bf16x2(g[2], g[3], ph.y, pl.y);
      split_bf16x2(g[4], g[5], ph.z, pl.z); split_bf16x2(g[6], g[7], ph.w, pl.w);
    }
    __nv_bfloat16* dst = out + ((n * C8 + cv) * int64_t(Hp) * Wp + p) * 8;
    *reinterpret_cast<uint4*>(dst) = ph;
    *reinterpret_cast<uint4*>(dst + lo_off) = pl;
  }
  __shared__ float red[256][9];
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.x][j] = g[j];
  __syncthreads();
  if (int(threadIdx.x) < C8 * 8) {
    const int c8 = threadIdx.x / 8, j = threadIdx.x % 8;
    float t = 0.f;
    for (int k = c8; k < 256; k += C8) t += red[k][j];   // fixed order
    partial[(n * gridDim.x + blockIdx.x) * (C8 * 8) + c8 * 8 + j] = t;
  }
}

// uint8 NCHW frames -> 16-channel padded planar image: chunk cv = frame channels 8*cv .. 8*cv + 7 (zeros from Cf on),
// lo = zeros
__global__ void sw_frames_u8_kernel(const uint8_t* __restrict__ frame, __nv_bfloat16* __restrict__ out, int64_t lo_off, int64_t Nf,
                                    int Cf, int H, int W, int slack_units) {
  const int Hp = H + 2, Wp = W + 2;
  const int64_t total = Nf * 2 * Hp * Wp;
  if (blockIdx.x == 0) zero_slack_units(out, lo_off, total * 8, slack_units);
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int px = int(i % Wp);
    int64_t t = i / Wp;
    const int py = int(t % Hp); t /= Hp;
    const int cv = int(t & 1);
    const int64_t n = t >> 1;
    uint4 ph = make_uint4(0u, 0u, 0u, 0u);
    const int c0 = 8 * cv;
    if (c0 < Cf && py >= 1 && py <= H && px >= 1 && px <= W) {
      float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int c = c0; c < Cf && c < c0 + 8; ++c) f[c - c0] = float(__ldg(frame + ((n * Cf + c) * H + (py - 1)) * W + (px - 1)));
      __nv_bfloat162 p0 = __floats2bfloat162_rn(f[0], f[1]), p1 = __floats2bfloat162_rn(f[2], f[3]);
      __nv_bfloat162 p2 = __floats2bfloat162_rn(f[4], f[5]), p3 = __floats2bfloat162_rn(f[6], f[7]);
      ph.x = *reinterpret_cast<uint32_t*>(&p0); ph.y = *reinterpret_cast<uint32_t*>(&p1);
      ph.z = *reinterpret_cast<uint32_t*>(&p2); ph.w = *reinterpret_cast<uint32_t*>(&p3);
    }
    __nv_bfloat16* dst = out + i * 8;   // i already walks [n][chunk][py][px]
    *reinterpret_cast<uint4*>(dst) = ph;
    *reinterpret_cast<uint4*>(dst + lo_off) = make_uint4(0u, 0u, 0u, 0u);
  }
}

// the same image (Cf = 4) from an unstacked rollout: channel c of frame n = (t, b) is row unstacked_row(t, b, c)
__global__ void sw_frames_u8_unstacked_kernel(const uint8_t* __restrict__ frames, const uint8_t* __restrict__ done,
                                              __nv_bfloat16* __restrict__ out, int64_t lo_off, int64_t T1, int64_t B, int H,
                                              int W, int slack_units) {
  const int Hp = H + 2, Wp = W + 2;
  const int64_t total = T1 * B * 2 * Hp * Wp;
  if (blockIdx.x == 0) zero_slack_units(out, lo_off, total * 8, slack_units);
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int px = int(i % Wp);
    int64_t t = i / Wp;
    const int py = int(t % Hp); t /= Hp;
    const int cv = int(t & 1);
    const int64_t n = t >> 1;
    uint4 ph = make_uint4(0u, 0u, 0u, 0u);
    if (cv == 0 && py >= 1 && py <= H && px >= 1 && px <= W) {
      const int64_t ts = n / B, b = n - ts * B;
      float f[4];
#pragma unroll
      for (int c = 0; c < 4; ++c)
        f[c] = float(__ldg(frames + ((unstacked_row(done, ts, b, B, c) * B + b) * H + (py - 1)) * W + (px - 1)));
      __nv_bfloat162 p0 = __floats2bfloat162_rn(f[0], f[1]), p1 = __floats2bfloat162_rn(f[2], f[3]);
      ph.x = *reinterpret_cast<uint32_t*>(&p0); ph.y = *reinterpret_cast<uint32_t*>(&p1);
    }
    __nv_bfloat16* dst = out + i * 8;
    *reinterpret_cast<uint4*>(dst) = ph;
    *reinterpret_cast<uint4*>(dst + lo_off) = make_uint4(0u, 0u, 0u, 0u);
  }
}

// column sums of the block partials [blocks][C] in two levels (fixed association: deterministic): level 1 = kColsumSlices
// blocks, each folding a contiguous slice of rows with coalesced reads (thread = (row group, channel)); level 2 = one block
constexpr int kColsumSlices = 128;
__global__ void __launch_bounds__(256) sw_colsum_l1_kernel(const float* __restrict__ partial, float* __restrict__ part2, int64_t blocks,
                                                           int C) {
  __shared__ float red[256];
  const int c = threadIdx.x % C, rg = threadIdx.x / C, RG = 256 / C;
  const int64_t per = (blocks + gridDim.x - 1) / gridDim.x;
  const int64_t b0 = int64_t(blockIdx.x) * per, b1 = (b0 + per < blocks) ? b0 + per : blocks;
  float s = 0.f;
  for (int64_t b = b0 + rg; b < b1; b += RG) s += partial[b * C + c];
  red[threadIdx.x] = s;
  __syncthreads();
  if (rg == 0) {
    float t = red[c];
    for (int k = 1; k < RG; ++k) t += red[k * C + c];
    part2[int64_t(blockIdx.x) * C + c] = t;
  }
}
__global__ void __launch_bounds__(256) sw_colsum_l2_kernel(const float* __restrict__ part2, float* __restrict__ out, int slices, int C) {
  __shared__ float red[256];
  const int c = threadIdx.x % C, rg = threadIdx.x / C, RG = 256 / C;
  float s = 0.f;
  for (int b = rg; b < slices; b += RG) s += part2[int64_t(b) * C + c];
  red[threadIdx.x] = s;
  __syncthreads();
  if (rg == 0) {
    float t = red[c];
    for (int k = 1; k < RG; ++k) t += red[k * C + c];
    out[c] = t;
  }
}

__global__ void sw_pack_weights_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int O, int C, int transpose,
                                       int c_real, int RB) {
  const int R = transpose ? C : O, K = transpose ? O : C;   // operand rows, reduction channels
  const int KP = K / 16, NB = 9 * KP * 2;
  const int64_t total = int64_t(9) * K * R;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    // hi element index i = (((rb*9 + tap)*KP + kp)*2 + j)*RB + r_in)*8 + e for row r = rb*RB + r_in; stored at row r_in
    // (hi) and row RB + r_in (lo) of a 2RB-row block: one complete operand per block of RB rows
    const int e = int(i & 7);
    int64_t t = i >> 3;
    const int r_in = int(t % RB); t /= RB;
    const int64_t blk = t % NB;                    // ((tap*KP + kp)*2 + j)
    const int rb = int(t / NB);
    const int r = rb * RB + r_in;
    const int j = int(blk & 1);
    const int kp = int((blk >> 1) % KP);
    const int tap = int((blk >> 1) / KP);
    const int k = kp * 16 + j * 8 + e;
    const int a = tap / 3, b = tap % 3;
    float v;
    if (transpose) v = w[((int64_t(k) * C + r) * 3 + (2 - a)) * 3 + (2 - b)];
    else v = k < c_real ? w[((int64_t(r) * c_real + k) * 3 + a) * 3 + b] : 0.0f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const int64_t ob = (int64_t(rb) * NB + blk) * 2 * RB;
    out[(ob + r_in) * 8 + e] = h;
    out[(ob + RB + r_in) * 8 + e] = bf16_lo_of(v, h);
  }
}

}  // namespace

int64_t sw_image_elems(int64_t Nf, int H, int W, int C) {
  const SwGeom g = sw_geom(H, W);
  return Nf * (C / 8) * g.plane + int64_t(g.pin + 8) * 8;   // + the window overhang of the last frame's last tile
}

int sw_pad_split(const float* x, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int H, int W, int C, int relu_in,
                 cudaStream_t stream) {
  ProfScope prof("pad_split", stream);
  TB_REQUIRE(C % 8 == 0 && 256 % (C / 8) == 0 && lo_off % 8 == 0 && Nf < 65536, "sw_pad_split: unsupported channel / frame count");
  if (Nf == 0) return 0;
  const int ppb = 256 / (C / 8);
  dim3 grid(unsigned(((H + 2) * (W + 2) + ppb - 1) / ppb), unsigned(Nf));
  sw_pad_split_kernel<false><<<grid, 256, 0, stream>>>(reinterpret_cast<const float4*>(x), out, lo_off, H, W, C / 8, relu_in, nullptr,
                                                       sw_geom(H, W).pin + 8);
  return check_launch("sw_pad_split_kernel");
}

int sw_pad_split_colsum(const float* x, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int H, int W, int C, float* db,
                        float* scratch, int64_t scratch_floats, cudaStream_t stream) {
  ProfScope prof("bias_grad_colsum", stream);
  TB_REQUIRE(C % 8 == 0 && 256 % C == 0 && lo_off % 8 == 0 && Nf < 65536, "sw_pad_split_colsum: unsupported channel / frame count");
  if (Nf == 0) return 0;
  const int ppb = 256 / (C / 8);
  dim3 grid(unsigned(((H + 2) * (W + 2) + ppb - 1) / ppb), unsigned(Nf));
  const int64_t blocks = int64_t(grid.x) * grid.y;
  TB_REQUIRE((blocks + kColsumSlices) * C <= scratch_floats, "sw_pad_split_colsum: scratch too small");
  sw_pad_split_kernel<true><<<grid, 256, 0, stream>>>(reinterpret_cast<const float4*>(x), out, lo_off, H, W, C / 8, 0, scratch,
                                                      sw_geom(H, W).pin + 8);
  int rc = check_launch("sw_pad_split_kernel");
  if (rc) return rc;
  float* part2 = scratch + blocks * C;
  sw_colsum_l1_kernel<<<kColsumSlices, 256, 0, stream>>>(scratch, part2, blocks, C);
  rc = check_launch("sw_colsum_l1_kernel");
  if (rc) return rc;
  sw_colsum_l2_kernel<<<1, 256, 0, stream>>>(part2, db, kColsumSlices, C);
  return check_launch("sw_colsum_l2_kernel");
}

int sw_pool_bwd_image_colsum(const uint8_t* argmax, const float* dy_pooled, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int H, int W,
                             int C, float* db, float* scratch, int64_t scratch_floats, cudaStream_t stream) {
  ProfScope prof("maxpool_bwd", stream);
  TB_REQUIRE(C % 8 == 0 && 256 % C == 0 && lo_off % 8 == 0 && Nf < 65536, "sw_pool_bwd_image_colsum: unsupported channel / frame count");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(argmax) & 7) == 0, "sw_pool_bwd_image_colsum: argmax must be 8-byte aligned");
  if (Nf == 0) return 0;
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  const int ppb = 256 / (C / 8);
  dim3 grid(unsigned(((H + 2) * (W + 2) + ppb - 1) / ppb), unsigned(Nf));
  const int64_t blocks = int64_t(grid.x) * grid.y;
  TB_REQUIRE((blocks + kColsumSlices) * C <= scratch_floats, "sw_pool_bwd_image_colsum: scratch too small");
  sw_pool_bwd_image_kernel<<<grid, 256, 0, stream>>>(argmax, reinterpret_cast<const float4*>(dy_pooled), out, lo_off, H, W, OH, OW,
                                                     C / 8, scratch, sw_geom(H, W).pin + 8);
  int rc = check_launch("sw_pool_bwd_image_kernel");
  if (rc) return rc;
  float* part2 = scratch + blocks * C;
  sw_colsum_l1_kernel<<<kColsumSlices, 256, 0, stream>>>(scratch, part2, blocks, C);
  rc = check_launch("sw_colsum_l1_kernel");
  if (rc) return rc;
  sw_colsum_l2_kernel<<<1, 256, 0, stream>>>(part2, db, kColsumSlices, C);
  return check_launch("sw_colsum_l2_kernel");
}

int64_t sw_csum_rows(int64_t Nf, int H, int W) { return Nf * sw_geom(H, W).tpf * 4; }

int sw_csum_reduce(float* csum, int64_t rows, int C, float* db, cudaStream_t stream) {
  ProfScope prof("bias_grad_colsum", stream);
  TB_REQUIRE(256 % C == 0, "sw_csum_reduce: unsupported channel count");
  float* part2 = csum + rows * C;
  sw_colsum_l1_kernel<<<kColsumSlices, 256, 0, stream>>>(csum, part2, rows, C);
  int rc = check_launch("sw_colsum_l1_kernel");
  if (rc) return rc;
  sw_colsum_l2_kernel<<<1, 256, 0, stream>>>(part2, db, kColsumSlices, C);
  return check_launch("sw_colsum_l2_kernel");
}

int sw_frames_u8(const uint8_t* frame, __nv_bfloat16* out, int64_t lo_off, int64_t Nf, int Cf, int H, int W, cudaStream_t stream) {
  ProfScope prof("frames_to_image", stream);
  TB_REQUIRE(Cf >= 1 && Cf <= 16 && lo_off % 8 == 0, "sw_frames_u8: 1 to 16 frame channels");
  const int64_t total = Nf * 2 * (H + 2) * (W + 2);
  if (total == 0) return 0;
  sw_frames_u8_kernel<<<sgrid(total, 256), 256, 0, stream>>>(frame, out, lo_off, Nf, Cf, H, W, sw_geom(H, W).pin + 8);
  return check_launch("sw_frames_u8_kernel");
}

int sw_frames_u8_unstacked(const uint8_t* frames, const uint8_t* done, __nv_bfloat16* out, int64_t lo_off, int64_t T1, int64_t B,
                           int H, int W, cudaStream_t stream) {
  ProfScope prof("frames_to_image", stream);
  TB_REQUIRE(frames && done && lo_off % 8 == 0, "sw_frames_u8_unstacked: null pointer or misaligned lo plane");
  const int64_t total = T1 * B * 2 * (H + 2) * (W + 2);
  if (total == 0) return 0;
  sw_frames_u8_unstacked_kernel<<<sgrid(total, 256), 256, 0, stream>>>(frames, done, out, lo_off, T1, B, H, W,
                                                                       sw_geom(H, W).pin + 8);
  return check_launch("sw_frames_u8_unstacked_kernel");
}

int64_t sw_weight_elems(int O, int C) { return int64_t(2) * 9 * O * C; }

int sw_pack_weights(const float* w, __nv_bfloat16* out, int O, int C, int transpose, cudaStream_t stream, int c_real) {
  TB_REQUIRE(O % 16 == 0 && C % 16 == 0, "sw_pack_weights: channel counts must be multiples of 16");
  TB_REQUIRE(c_real == 0 || (!transpose && c_real <= C), "sw_pack_weights: c_real only for the forward operand");
  const int64_t total = int64_t(9) * O * C;
  const int R = transpose ? C : O;   // blocks of 32 operand rows: the wide forward kernel loads one block per CTA
  sw_pack_weights_kernel<<<sgrid(total, 256), 256, 0, stream>>>(w, out, O, C, transpose, c_real > 0 ? c_real : C, R < 32 ? R : 32);
  return check_launch("sw_pack_weights_kernel");
}

namespace {
bool sw_channels_ok(int c) { return c == 16 || c == 32 || c == 64; }
// sw_conv_fwd_kernel (all weights and a whole window per stage) takes a 16 / 32-channel pair when it fits, static
// column-sum staging included (32 -> 32 does not from W = 54 on); everything else runs on sw_conv_fwd_wide_kernel
bool sw_fwd_resident(int pin, int CK, int NO) {
  return CK <= 32 && NO <= 32 && sw_fwd_smem(pin, CK, NO) + sizeof(float) * 8 * 32 * (NO + 1) <= 227 * 1024;
}
// shared memory (dynamic + static) of the forward kernel that runs a CK -> NO conv at this window
size_t sw_fwd_smem_any(int pin, int CK, int NO) {
  return sw_fwd_resident(pin, CK, NO) ? sw_fwd_smem(pin, CK, NO) + sizeof(float) * 8 * 32 * (NO + 1)
                                      : sw_fwd_wide_smem(pin, CK, NO) + sw_fwd_wide_static(NO);
}
}  // namespace

bool sw_conv_applicable(int H, int W, int CK, int NO) {
  if (!(sw_channels_ok(CK) && sw_channels_ok(NO) && H >= 3 && W >= 3 && W <= 126)) return false;
  // a 64 -> 32 / 64 window fits up to W = 101
  return sw_fwd_smem_any(sw_geom(H, W).pin, CK, NO) <= 227 * 1024;
}

bool sw_conv_trainable(int H, int W, int CK, int NO, bool input_grad) {
  if (!sw_conv_applicable(H, W, CK, NO) || (input_grad && !sw_conv_applicable(H, W, NO, CK)) || W < kWgMinW) return false;
  const int pin = sw_geom(H, W).pin;
  const size_t limit = 227 * 1024;
  return sw_fwd_smem_any(pin, CK, NO) <= limit && (!input_grad || sw_fwd_smem_any(pin, NO, CK) <= limit) &&
         sw_wgrad_smem(pin, sw_wgrad_block(CK), sw_wgrad_block(NO)) <= limit;
}

int64_t sw_colsum_scratch_floats(int64_t Nf, int H, int W, int C) {
  const int ppb = 256 / (C / 8);
  return (int64_t(((H + 2) * (W + 2) + ppb - 1) / ppb) * Nf + kColsumSlices) * C;
}

int sw_conv_fwd(const __nv_bfloat16* img, int64_t img_lo, const __nv_bfloat16* wk, float* out, int64_t Nf, int H, int W, int CK, int NO,
                const SwEpilogue& ep, cudaStream_t stream) {
  TB_REQUIRE(img && wk && out && img_lo > 0, "sw_conv_fwd: null pointer");
  TB_REQUIRE(sw_conv_applicable(H, W, CK, NO), "sw_conv_fwd: unsupported shape");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(img) & 15) == 0 && (reinterpret_cast<uintptr_t>(wk) & 15) == 0 && img_lo % 8 == 0 &&
                 (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "sw_conv_fwd: operands must be 16-byte aligned");
  if (Nf == 0) return 0;
  TB_REQUIRE(Nf * sw_geom(H, W).tpf < (int64_t(1) << 31), "sw_conv_fwd: too many tiles");
  ProfScope prof(ep.tag, stream);
  SwFwdArgs a;
  a.img = img; a.img_lo = img_lo; a.wk = wk; a.out = out; a.bias = ep.bias; a.mask = ep.mask; a.addend = ep.addend;
  a.scale = ep.scale; a.Nf = int(Nf); a.g = sw_geom(H, W);
  a.emit = ep.emit; a.emit_lo = ep.emit_lo; a.emit_relu = ep.emit_relu; a.csum = ep.csum;
  TB_REQUIRE(!ep.emit || (ep.emit_lo > 0 && ep.emit_lo % 8 == 0 && (reinterpret_cast<uintptr_t>(ep.emit) & 15) == 0),
             "sw_conv_fwd: the emitted image needs a 16-byte aligned base and a lo plane");
  if (sw_fwd_resident(a.g.pin, CK, NO)) {
    if (CK == 16 && NO == 16) return launch_sw_fwd<16, 16>(a, stream);
    if (CK == 16 && NO == 32) return launch_sw_fwd<16, 32>(a, stream);
    if (CK == 32 && NO == 16) return launch_sw_fwd<32, 16>(a, stream);
    return launch_sw_fwd<32, 32>(a, stream);
  }
  if (CK == 16 && NO == 16) return launch_sw_fwd_wide<16, 16>(a, stream);
  if (CK == 16 && NO == 32) return launch_sw_fwd_wide<16, 32>(a, stream);
  if (CK == 32 && NO == 16) return launch_sw_fwd_wide<32, 16>(a, stream);
  if (CK == 32 && NO == 32) return launch_sw_fwd_wide<32, 32>(a, stream);
  if (CK == 16) return launch_sw_fwd_wide<16, 64>(a, stream);
  if (CK == 32) return launch_sw_fwd_wide<32, 64>(a, stream);
  if (NO == 16) return launch_sw_fwd_wide<64, 16>(a, stream);
  if (NO == 32) return launch_sw_fwd_wide<64, 32>(a, stream);
  return launch_sw_fwd_wide<64, 64>(a, stream);
}

int sw_conv_wgrad(const __nv_bfloat16* dyimg, int64_t dy_lo, const __nv_bfloat16* ximg, int64_t x_lo, float* dW, int64_t Nf, int H,
                  int W, int C, int O, float* partial, int64_t partial_floats, const char* tag, cudaStream_t stream, float scale,
                  int c_real) {
  TB_REQUIRE(dyimg && ximg && dW && partial && dy_lo > 0 && x_lo > 0, "sw_conv_wgrad: null pointer");
  TB_REQUIRE(sw_conv_applicable(H, W, C, O), "sw_conv_wgrad: unsupported shape");
  TB_REQUIRE(W >= kWgMinW, "sw_conv_wgrad: W = %d < %d: the last pixel step of a frame would read the next plane", W, kWgMinW);
  if (Nf == 0) return 0;
  ProfScope prof(tag, stream);
  SwWgradArgs a;
  a.dy = dyimg; a.dy_lo = dy_lo; a.x = ximg; a.x_lo = x_lo; a.partial = partial; a.Nf = int(Nf); a.g = sw_geom(H, W);
  // 64-channel sides run as NB blocks of CT x OT channels, kNumSMs / NB CTAs each (sw_conv_wgrad_kernel)
  const int CT = sw_wgrad_block(C), OT = sw_wgrad_block(O), NBC = C / CT, NB = NBC * (O / OT);
  int64_t grid = kNumSMs / NB;
  const int64_t total = Nf * a.g.tpf;
  if (grid > total) grid = total;
  TB_REQUIRE(grid * O * 9 * C <= partial_floats, "sw_conv_wgrad: partial buffer too small");
  int rc;
  if (C == 16 && O == 16) rc = launch_sw_wgrad<16, 16>(a, int(grid), stream);
  else if (C == 16 && O == 32) rc = launch_sw_wgrad<16, 32>(a, int(grid), stream);
  else if (C == 32 && O == 16) rc = launch_sw_wgrad<32, 16>(a, int(grid), stream);
  else if (C == 32 && O == 32) rc = launch_sw_wgrad<32, 32>(a, int(grid), stream);
  else if (C == 16) rc = launch_sw_wgrad<16, 64, 16, 32>(a, int(grid), stream);
  else if (C == 32) rc = launch_sw_wgrad<32, 64, 32, 32>(a, int(grid), stream);
  else if (O == 16) rc = launch_sw_wgrad<64, 16, 32, 16>(a, int(grid), stream);
  else if (O == 32) rc = launch_sw_wgrad<64, 32, 32, 32>(a, int(grid), stream);
  else rc = launch_sw_wgrad<64, 64, 32, 32>(a, int(grid), stream);
  if (rc) return rc;
  if (c_real <= 0 || c_real > C) c_real = C;
  // one fixed-order reduce per block: block (ob, cb) holds rows ob*OT.. of dW and its columns cb*CT.. (c_real == C
  // whenever C is split, so the row pitch c_real and the column bound hold for every block)
  for (int b = 0; b < NB; ++b) {
    const int ob = b / NBC, cb = b % NBC;
    sw_wgrad_reduce_kernel<<<(OT * 9 * CT + 31) / 32, 256, 0, stream>>>(partial + int64_t(b) * grid * OT * 9 * CT,
                                                                       dW + (int64_t(ob) * OT * c_real + cb * CT) * 9, int(grid),
                                                                       OT, CT, c_real, scale);
    rc = check_launch("sw_wgrad_reduce_kernel");
    if (rc) return rc;
  }
  return 0;
}

}  // namespace tb
