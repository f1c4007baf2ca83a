// Four-frame stacks rebuilt on the GPU from unstacked rollouts (restack.cuh, include/torchbeast_b200.h).
// The default backends fuse the restack into their frame-image pass (frames_u8_unstacked_to_bf16 in conv_implicit.cu,
// sw_frames_u8_unstacked in conv3x3_sw.cu); the backends that read stacked frames directly (AtariNet fp32, ResNet
// fp32 / bf16) restack into a caller-owned scratch with the kernel below and then run their stacked path unchanged.
#include "restack.cuh"

namespace tb {

// one 16-byte vector per iteration; a plane (HW bytes, HW % 16 == 0) never straddles a vector
__global__ void restack_frames_u8_kernel(const uint8_t* __restrict__ frames, const uint8_t* __restrict__ done, int64_t T1,
                                         int64_t B, int64_t vpp, uint4* __restrict__ stacked) {
  const int64_t total = T1 * B * 4 * vpp;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t plane = i / vpp;
    const int c = int(plane & 3);
    const int64_t n = plane >> 2, t = n / B, b = n - t * B;
    const int64_t row = unstacked_row(done, t, b, B, c);
    stacked[i] = __ldg(reinterpret_cast<const uint4*>(frames) + (row * B + b) * vpp + (i - plane * vpp));
  }
}

int restack_frames_u8(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW, uint8_t* stacked,
                      cudaStream_t stream) {
  TB_REQUIRE(T1 >= 1 && B >= 1 && HW >= 16 && HW % 16 == 0, "restack_frames_u8: bad sizes T1=%lld B=%lld HW=%lld",
             (long long)T1, (long long)B, (long long)HW);
  TB_REQUIRE(frames && done && stacked, "restack_frames_u8: null pointer");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(frames) & 15) == 0 && (reinterpret_cast<uintptr_t>(stacked) & 15) == 0,
             "restack_frames_u8: frames and stacked_out must be 16-byte aligned");
  ProfScope prof("restack_frames", stream);
  const int64_t vpp = HW / 16, total = T1 * B * 4 * vpp;
  int64_t blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  restack_frames_u8_kernel<<<(unsigned)blocks, 256, 0, stream>>>(frames, done, T1, B, vpp, reinterpret_cast<uint4*>(stacked));
  return check_launch("restack_frames_u8_kernel");
}

// One thread per (column, 16-byte vector).  The thread loads its stream's three history vectors into registers before
// it stores anything, and it is the only thread that touches those history bytes or rows 0..2 of its column at that
// vector, so distinct ids cannot race.  The rows unstacked_row picks for step T-1 are either rows 0..2, which are
// exactly the loaded vectors, or newest-frame rows the caller wrote, which nothing here stores to.
__global__ void frame_history_fill_u8_kernel(uint4* __restrict__ frames, const uint8_t* __restrict__ done,
                                             const int64_t* __restrict__ stream_ids, int64_t T, int64_t B, int64_t vpp,
                                             uint4* __restrict__ history, int64_t S) {
  const int64_t total = B * vpp;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t b = i / vpp, v = i - b * vpp;
    const int64_t s = __ldg(stream_ids + b);
    uint4 h[3];
    if (s >= 0 && s < S) {
#pragma unroll
      for (int c = 0; c < 3; ++c) h[c] = history[(s * 3 + c) * vpp + v];
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) h[c] = make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) frames[(c * B + b) * vpp + v] = h[c];
    if (s < 0 || s >= S) continue;
#pragma unroll
    for (int c = 1; c < 4; ++c) {
      const int64_t row = unstacked_row(done, T - 1, b, B, c);
      // selects rather than h[row]: a register array indexed at run time would live in local memory
      history[(s * 3 + c - 1) * vpp + v] = row == 0 ? h[0] : row == 1 ? h[1] : row == 2 ? h[2]
                                                                                          : frames[(row * B + b) * vpp + v];
    }
  }
}

int frame_history_fill_u8(uint8_t* frames, const uint8_t* done, const int64_t* stream_ids, int64_t T, int64_t B,
                          int64_t HW, uint8_t* history, int64_t S, cudaStream_t stream) {
  TB_REQUIRE(T >= 1 && B >= 1 && S >= 1 && HW >= 16 && HW % 16 == 0,
             "frame_history_fill_u8: bad sizes T=%lld B=%lld HW=%lld S=%lld", (long long)T, (long long)B, (long long)HW,
             (long long)S);
  TB_REQUIRE(frames && done && stream_ids && history, "frame_history_fill_u8: null pointer");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(frames) & 15) == 0 && (reinterpret_cast<uintptr_t>(history) & 15) == 0,
             "frame_history_fill_u8: frames and history must be 16-byte aligned");
  ProfScope prof("frame_history_fill", stream);
  const int64_t vpp = HW / 16, total = B * vpp;
  int64_t blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  frame_history_fill_u8_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<uint4*>(frames), done, stream_ids, T,
                                                                      B, vpp, reinterpret_cast<uint4*>(history), S);
  return check_launch("frame_history_fill_u8_kernel");
}

}  // namespace tb

using namespace tb;

extern "C" {

int tb_restack_frames_u8(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW, uint8_t* stacked_out,
                         void* stream) {
  return restack_frames_u8(frames, done, T1, B, HW, stacked_out, (cudaStream_t)stream);
}

int tb_frame_history_fill_u8(uint8_t* frames, const uint8_t* done, const int64_t* stream_ids, int64_t T, int64_t B,
                             int64_t HW, uint8_t* history, int64_t S, void* stream) {
  return frame_history_fill_u8(frames, done, stream_ids, T, B, HW, history, S, (cudaStream_t)stream);
}

size_t tb_unstacked_scratch_bytes(int net, int64_t T1, int64_t B, int precision) {
  if (net < 0 || net > 1 || precision < 0 || precision > 2 || T1 < 1 || B < 1) {
    set_error("tb_unstacked_scratch_bytes: unknown net %d / precision %d or bad sizes", net, precision);
    return SIZE_MAX;
  }
  // fused: AtariNet bf16 / bf16x3 (frame image of conv1), ResNet bf16x3 (padded image of the first conv)
  const bool fused = net == 0 ? precision != 0 : precision == 2;
  return fused ? 0 : size_t(T1) * size_t(B) * 4 * 84 * 84;
}

}  // extern "C"
