// Unstacked rollouts (include/torchbeast_b200.h, "unstacked rollouts"): frame u8 [T1+3, B, HW] holds rows 0..2 =
// channels 0..2 of step 0's four-frame stack, row 3+t = the newest channel of step t's stack; done [T1, B] (non-zero =
// the step starts an episode, so FrameStack.reset filled every channel with that frame).
#pragma once
#include "common.cuh"

namespace tb {

// Row of the unstacked frame array that holds channel c (0..3) of step t's stack in column b:
//   3 + max(t - 3 + c, last_done(t, b)),  last_done = the largest s <= t with done[s, b] != 0, else -3.
// Only a done in (t - 3 + c, t] can win the max, so at most three entries of `done` are read.
__device__ __forceinline__ int64_t unstacked_row(const uint8_t* __restrict__ done, int64_t t, int64_t b, int64_t B, int c) {
  for (int64_t s = t; s > t - 3 + c && s >= 0; --s)
    if (__ldg(done + s * B + b)) return 3 + s;
  return t + c;
}

// stacked[T1, B, 4, HW] = the stacks rebuilt from frames [T1+3, B, HW]; HW % 16 == 0, both pointers 16-byte aligned
int restack_frames_u8(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW, uint8_t* stacked,
                      cudaStream_t stream);

// rows 0..2 of frames [T+3, B, HW] from history [S, 3, HW] at stream_ids[b], then each history := channels 1..3 of
// step T-1's stack; ids outside [0, S) get zero rows and leave the history alone (tb_frame_history_fill_u8)
int frame_history_fill_u8(uint8_t* frames, const uint8_t* done, const int64_t* stream_ids, int64_t T, int64_t B,
                          int64_t HW, uint8_t* history, int64_t S, cudaStream_t stream);

}  // namespace tb
