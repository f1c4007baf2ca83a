// Seeded categorical action sampling for sm_90a (H100): the acting forward's
//   action = torch.multinomial(F.softmax(policy_logits, dim=1), num_samples=1)
// (reference monobeast.py:618-619, polybeast_learner.py:256-257) as a stateless, counter-based kernel.
//
// The sampling contract (include/torchbeast_b200.h, tb_sample_actions_f32) fixes every step, so a CPU restatement
// (oracle/sampling_np.py) gives the same action on every row that is not within rounding of a cumulative boundary:
// Philox4x32-10 keyed by the seed, counter (step + t, stream id) -> 24-bit uniform u; precise expf of the
// max-shifted logits summed in index order; the first index whose fp32 running sum exceeds u*S.
//
// One thread per row, three passes over the row in global memory (max, sum, running sum); no shared memory, no
// atomics.  At acting sizes (B <= 512, A <= 18) the launch is latency-bound, not bandwidth-bound.
#include <math.h>

#include "common.cuh"

namespace tb {

// Steps 2-5 of the sampling contract on one segment of A logits, as sample_actions_kernel runs them on a whole row
// (that kernel keeps its own copy, so its code is what it was before factored spaces existed); `draw()` gives the
// segment's Philox word and is called only when the segment has a distribution to sample.
template <typename Draw>
__device__ __forceinline__ int64_t sample_row(const float* __restrict__ row, int64_t A, Draw draw) {
  // pass 1: maximum; NaN is tracked apart because fmaxf ignores it
  float m = -INFINITY;
  bool nan = false;
  for (int64_t a = 0; a < A; ++a) {
    const float l = row[a];
    nan |= isnan(l);
    m = fmaxf(m, l);
  }
  if (nan || !isfinite(m)) return -1;  // NaN anywhere, every logit -inf, or a +inf logit: no distribution to sample
  // pass 2: S = sum of expf(l - m) in index order
  float S = 0.0f;
  for (int64_t a = 0; a < A; ++a) S += expf(row[a] - m);
  const uint32_t x = draw();
  const float u = float(x >> 8) * 0x1p-24f;
  const float target = u * S;
  // pass 3: first a whose running sum exceeds u*S; if rounding leaves none, the last a with e_a > 0
  float c = 0.0f;
  int64_t pick = -1, last_pos = -1;
  for (int64_t a = 0; a < A; ++a) {
    const float e = expf(row[a] - m);
    c += e;
    if (e > 0.0f) last_pos = a;
    if (c > target) {
      pick = a;
      break;
    }
  }
  return pick >= 0 ? pick : last_pos;
}

// kSeedStepOnDevice: seed and step are read from seed_step[0..1] when the kernel runs instead of the by-value
// arguments, so a launch captured in a CUDA graph picks up whatever (seed, step) was written there before each replay.
template <bool kSeedStepOnDevice>
__global__ void __launch_bounds__(256) sample_actions_kernel(const float* __restrict__ logits, int64_t N, int64_t B,
                                                             int64_t A, uint64_t seed, uint64_t step,
                                                             const uint64_t* __restrict__ seed_step,
                                                             const int64_t* __restrict__ stream_ids,
                                                             int64_t* __restrict__ actions) {
  if (kSeedStepOnDevice) {
    seed = seed_step[0];
    step = seed_step[1];
  }
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const int64_t t = i / B, b = i - t * B;
    const float* row = logits + i * A;
    // pass 1: maximum; NaN is tracked apart because fmaxf ignores it
    float m = -INFINITY;
    bool nan = false;
    for (int64_t a = 0; a < A; ++a) {
      const float l = row[a];
      nan |= isnan(l);
      m = fmaxf(m, l);
    }
    if (nan || !isfinite(m)) {  // NaN anywhere, every logit -inf, or a +inf logit: no distribution to sample
      actions[i] = -1;
      continue;
    }
    // pass 2: S = sum of expf(l - m) in index order
    float S = 0.0f;
    for (int64_t a = 0; a < A; ++a) S += expf(row[a] - m);
    // the row's uniform: counter (step + t, stream id), key = seed
    const uint64_t ctr = step + uint64_t(t);
    const uint64_t sid = stream_ids ? uint64_t(stream_ids[b]) : uint64_t(b);
    const uint32_t x = philox4x32_10_w0(uint32_t(ctr), uint32_t(ctr >> 32), uint32_t(sid), uint32_t(sid >> 32),
                                        uint32_t(seed), uint32_t(seed >> 32));
    const float u = float(x >> 8) * 0x1p-24f;
    const float target = u * S;
    // pass 3: first a whose running sum exceeds u*S; if rounding leaves none, the last a with e_a > 0
    float c = 0.0f;
    int64_t pick = -1, last_pos = -1;
    for (int64_t a = 0; a < A; ++a) {
      const float e = expf(row[a] - m);
      c += e;
      if (e > 0.0f) last_pos = a;
      if (c > target) {
        pick = a;
        break;
      }
    }
    actions[i] = pick >= 0 ? pick : last_pos;
  }
}

// The factored form: component k of row i samples its segment with word k % 4 of the Philox block keyed
// (lo32(seed), hi32(seed) + k / 4), under the flat sampler's counter.  seed_step non-NULL: read when the kernel runs.
__global__ void __launch_bounds__(256) sample_actions_factored_kernel(const float* __restrict__ logits, int64_t N,
                                                                      int64_t B, int64_t A, uint64_t seed,
                                                                      uint64_t step,
                                                                      const uint64_t* __restrict__ seed_step,
                                                                      const int64_t* __restrict__ stream_ids,
                                                                      ActionSegments seg,
                                                                      int64_t* __restrict__ actions) {
  if (seed_step) {
    seed = seed_step[0];
    step = seed_step[1];
  }
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const int64_t t = i / B, b = i - t * B;
    const uint64_t ctr = step + uint64_t(t);
    const uint64_t sid = stream_ids ? uint64_t(stream_ids[b]) : uint64_t(b);
    const float* row = logits + i * A;
    for (int k = 0; k < seg.D; ++k) {
      actions[i * seg.D + k] = sample_row(row + seg.off[k], seg.off[k + 1] - seg.off[k], [&] {
        const uint4 w = philox4x32_10(uint32_t(ctr), uint32_t(ctr >> 32), uint32_t(sid), uint32_t(sid >> 32),
                                      uint32_t(seed), uint32_t(seed >> 32) + uint32_t(k / 4));
        const int j = k % 4;
        return j == 0 ? w.x : j == 1 ? w.y : j == 2 ? w.z : w.w;
      });
    }
  }
}

// Host validation and launch shared by both entries; seed_step is non-null exactly for the device-memory entry.
// seg non-NULL: the factored kernel (seed_step then nullable).
static int sample_actions(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                          const uint64_t* seed_step, const int64_t* stream_ids, int64_t* actions, void* stream,
                          const ActionSegments* seg = nullptr) {
  TB_REQUIRE(T >= 0 && B >= 0, "sample_actions: negative size T=%lld B=%lld", (long long)T, (long long)B);
  TB_REQUIRE(A >= 1, "sample_actions: A must be at least 1, got %lld", (long long)A);
  if (T == 0 || B == 0) return 0;
  TB_REQUIRE(T <= INT64_MAX / B && T * B <= INT64_MAX / A, "sample_actions: size overflow T=%lld B=%lld A=%lld",
             (long long)T, (long long)B, (long long)A);
  TB_REQUIRE(logits && actions, "sample_actions: null pointer");
  const int64_t N = T * B;
  const int threads = 256;
  int64_t blocks = (N + threads - 1) / threads;
  if (blocks > int64_t(kNumSMs) * 16) blocks = int64_t(kNumSMs) * 16;
  if (seg) {
    ProfScope prof("sample_actions_factored", (cudaStream_t)stream);
    sample_actions_factored_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(logits, N, B, A, seed, step,
                                                                                          seed_step, stream_ids, *seg,
                                                                                          actions);
    return check_launch("sample_actions_factored_kernel");
  }
  ProfScope prof("sample_actions", (cudaStream_t)stream);
  if (seed_step)
    sample_actions_kernel<true><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(logits, N, B, A, 0, 0, seed_step,
                                                                                        stream_ids, actions);
  else
    sample_actions_kernel<false><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(logits, N, B, A, seed, step,
                                                                                         nullptr, stream_ids, actions);
  return check_launch("sample_actions_kernel");
}

// The Gaussian form (include/torchbeast_b200.h, tb_sample_gaussian_f32): a row is (mu, log sigma) of width 2D, and the
// components 2j and 2j + 1 share the Philox block keyed (lo32(seed), hi32(seed) + j), words (0, 1) and (2, 3), each pair
// turned into one standard normal by Box-Muller.  seed_step non-NULL: read when the kernel runs.
__global__ void __launch_bounds__(256) sample_gaussian_kernel(const float* __restrict__ logits, int64_t N, int64_t B,
                                                              int D, uint64_t seed, uint64_t step,
                                                              const uint64_t* __restrict__ seed_step,
                                                              const int64_t* __restrict__ stream_ids,
                                                              float* __restrict__ actions) {
  if (seed_step) {
    seed = seed_step[0];
    step = seed_step[1];
  }
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) {
    const int64_t t = i / B, b = i - t * B;
    const uint64_t ctr = step + uint64_t(t);
    const uint64_t sid = stream_ids ? uint64_t(stream_ids[b]) : uint64_t(b);
    const float* row = logits + i * 2 * D;
    float* out = actions + i * D;
    for (int k = 0; k < D; k += 2) {
      const uint4 w = philox4x32_10(uint32_t(ctr), uint32_t(ctr >> 32), uint32_t(sid), uint32_t(sid >> 32),
                                    uint32_t(seed), uint32_t(seed >> 32) + uint32_t(k / 2));
      for (int h = 0; h < 2 && k + h < D; ++h) {
        const uint32_t x0 = h ? w.z : w.x, x1 = h ? w.w : w.y;
        const float u1 = float((x0 >> 8) + 1u) * 0x1p-24f, u2 = float(x1 >> 8) * 0x1p-24f;
        const float z = sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
        const float mu = row[k + h], l = row[D + k + h];
        out[k + h] = (isfinite(mu) && isfinite(l)) ? mu + expf(l) * z : __int_as_float(0x7fffffff);
      }
    }
  }
}

}  // namespace tb

using namespace tb;

extern "C" int tb_sample_gaussian_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed,
                                      uint64_t step, const uint64_t* seed_step, const int64_t* stream_ids,
                                      float* actions, void* stream) {
  TB_REQUIRE(T >= 0 && B >= 0, "sample_gaussian: negative size T=%lld B=%lld", (long long)T, (long long)B);
  TB_REQUIRE(A >= 2 && A % 2 == 0 && A / 2 <= TB_MAX_CONTINUOUS_DIM,
             "sample_gaussian: A = %lld must be 2D with 1 <= D <= %d", (long long)A, TB_MAX_CONTINUOUS_DIM);
  if (T == 0 || B == 0) return 0;
  TB_REQUIRE(T <= INT64_MAX / B && T * B <= INT64_MAX / A, "sample_gaussian: size overflow T=%lld B=%lld A=%lld",
             (long long)T, (long long)B, (long long)A);
  TB_REQUIRE(logits && actions, "sample_gaussian: null pointer");
  const int64_t N = T * B;
  const int threads = 256;
  int64_t blocks = (N + threads - 1) / threads;
  if (blocks > int64_t(kNumSMs) * 16) blocks = int64_t(kNumSMs) * 16;
  ProfScope prof("sample_gaussian", (cudaStream_t)stream);
  sample_gaussian_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(logits, N, B, int(A / 2), seed, step,
                                                                                 seed_step, stream_ids, actions);
  return check_launch("sample_gaussian_kernel");
}

extern "C" int tb_sample_actions_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                                     const int64_t* stream_ids, int64_t* actions, void* stream) {
  return sample_actions(logits, T, B, A, seed, step, nullptr, stream_ids, actions, stream);
}

extern "C" int tb_sample_actions_dev_f32(const float* logits, int64_t T, int64_t B, int64_t A, const uint64_t* seed_step,
                                         const int64_t* stream_ids, int64_t* actions, void* stream) {
  TB_REQUIRE(seed_step, "sample_actions_dev: null seed_step");
  return sample_actions(logits, T, B, A, 0, 0, seed_step, stream_ids, actions, stream);
}

extern "C" int tb_sample_actions_factored_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed,
                                              uint64_t step, const uint64_t* seed_step, const int64_t* stream_ids,
                                              const tb_action_space* space, int64_t* actions, void* stream) {
  ActionSegments seg;
  TB_TRY(action_segments(space, A, "sample_actions_factored", &seg));
  return sample_actions(logits, T, B, A, seed, step, seed_step, stream_ids, actions, stream, &seg);
}
