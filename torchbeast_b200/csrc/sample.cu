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

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011); only word 0 is used.
__device__ __forceinline__ uint32_t philox4x32_10_w0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                     uint32_t k1) {
  constexpr uint32_t kM0 = 0xD2511F53u, kM1 = 0xCD9E8D57u, kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(kM0, c0), lo0 = kM0 * c0;
    const uint32_t hi1 = __umulhi(kM1, c2), lo1 = kM1 * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += kW0;
    k1 += kW1;
  }
  return c0;
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

// Host validation and launch shared by both entries; seed_step is non-null exactly for the device-memory entry.
static int sample_actions(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                          const uint64_t* seed_step, const int64_t* stream_ids, int64_t* actions, void* stream) {
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
  ProfScope prof("sample_actions", (cudaStream_t)stream);
  if (seed_step)
    sample_actions_kernel<true><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(logits, N, B, A, 0, 0, seed_step,
                                                                                        stream_ids, actions);
  else
    sample_actions_kernel<false><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(logits, N, B, A, seed, step,
                                                                                         nullptr, stream_ids, actions);
  return check_launch("sample_actions_kernel");
}

}  // namespace tb

using namespace tb;

extern "C" int tb_sample_actions_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                                     const int64_t* stream_ids, int64_t* actions, void* stream) {
  return sample_actions(logits, T, B, A, seed, step, nullptr, stream_ids, actions, stream);
}

extern "C" int tb_sample_actions_dev_f32(const float* logits, int64_t T, int64_t B, int64_t A, const uint64_t* seed_step,
                                         const int64_t* stream_ids, int64_t* actions, void* stream) {
  TB_REQUIRE(seed_step, "sample_actions_dev: null seed_step");
  return sample_actions(logits, T, B, A, 0, 0, seed_step, stream_ids, actions, stream);
}
