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

}  // namespace tb

using namespace tb;

extern "C" {

int tb_restack_frames_u8(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW, uint8_t* stacked_out,
                         void* stream) {
  return restack_frames_u8(frames, done, T1, B, HW, stacked_out, (cudaStream_t)stream);
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
