// Legal-action masks for sm_90a (H100): the policy over each step's legal actions ("invalid action masking", Huang &
// Ontañón 2022), formed by replacing every illegal logit of a row with a finite sentinel before any softmax reads it.
//
// The contract is stated with tb_mask_logits_f32 in include/torchbeast_b200.h.  The sentinel TB_MASKED_LOGIT =
// -FLT_MAX is finite: expf(-FLT_MAX - m) is exactly 0 for any realistic row maximum m, so the loss, UPGO,
// kickstarting, trust-region and sampling kernels see p = 0, p * log p = -0 and a logit gradient of +-0 at an illegal
// entry, and their legal sums keep their bits, without a mask flag of their own.
//
// Layout: a group of G lanes (G = the power of two >= min(A, 32)) owns one row and strides over it, so a row of a few
// actions does not leave most of a warp idle and a row of hundreds is not walked by one thread.  The group's "any legal
// entry" is one warp ballot.  No shared memory, no atomics, no host sync: graph-capturable.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace tb {

template <int G>
__global__ void __launch_bounds__(256) mask_logits_kernel(const float* in, float* out, const uint8_t* __restrict__ legal,
                                                          const int64_t* __restrict__ actions, int64_t N, int64_t A,
                                                          float fill) {
  constexpr int kRowsPerWarp = kWarp / G;
  const int lane = threadIdx.x & (kWarp - 1);
  const int sub = lane & (G - 1);                  // lane within the row's group
  const int shift = lane & ~(G - 1);               // the group's first lane
  const unsigned gmask = G == kWarp ? 0xffffffffu : ((1u << G) - 1u);
  const int64_t warps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  // every lane of a warp runs the same iterations, so the ballot below always has the full warp
  for (int64_t w = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; w * kRowsPerWarp < N; w += warps) {
    const int64_t i = w * kRowsPerWarp + (lane / G);
    const bool row_ok = i < N;
    const uint8_t* lrow = legal + i * A;
    bool any = false;
    if (row_ok)
      for (int64_t a = sub; a < A; a += G) any |= lrow[a] != 0;
    any = ((__ballot_sync(0xffffffffu, any) >> shift) & gmask) != 0u;
    if (!row_ok) continue;
    const float* irow = in + i * A;
    float* orow = out + i * A;
    if (!any) {  // no legal action: the row stays as it is
      if (irow != orow)
        for (int64_t a = sub; a < A; a += G) orow[a] = irow[a];
      continue;
    }
    bool bad = false;
    if (actions) {  // an illegal taken action in a row that has a legal one: a caller bug, made a NaN row
      const int64_t act = actions[i];
      bad = act >= 0 && act < A && lrow[act] == 0;
    }
    for (int64_t a = sub; a < A; a += G) orow[a] = bad ? NAN : (lrow[a] ? irow[a] : fill);
  }
}

static int mask_logits(const float* in, float* out, const uint8_t* legal, const int64_t* actions, int64_t N, int64_t A,
                       float fill, void* stream) {
  TB_REQUIRE(N >= 0, "mask_logits: negative size N=%lld", (long long)N);
  TB_REQUIRE(A >= 1, "mask_logits: A must be at least 1, got %lld", (long long)A);
  if (N == 0) return 0;
  TB_REQUIRE(N <= INT64_MAX / A, "mask_logits: size overflow N=%lld A=%lld", (long long)N, (long long)A);
  TB_REQUIRE(in && out && legal, "mask_logits: null pointer");
  const int G = A > 16 ? 32 : A > 8 ? 16 : A > 4 ? 8 : A > 2 ? 4 : A > 1 ? 2 : 1;
  const int threads = 256;
  const int64_t rows_per_block = threads / G;
  int64_t blocks = (N + rows_per_block - 1) / rows_per_block;
  if (blocks > int64_t(kNumSMs) * 16) blocks = int64_t(kNumSMs) * 16;
  const cudaStream_t st = (cudaStream_t)stream;
  ProfScope prof("mask_logits", st);
  switch (G) {
    case 1: mask_logits_kernel<1><<<(unsigned)blocks, threads, 0, st>>>(in, out, legal, actions, N, A, fill); break;
    case 2: mask_logits_kernel<2><<<(unsigned)blocks, threads, 0, st>>>(in, out, legal, actions, N, A, fill); break;
    case 4: mask_logits_kernel<4><<<(unsigned)blocks, threads, 0, st>>>(in, out, legal, actions, N, A, fill); break;
    case 8: mask_logits_kernel<8><<<(unsigned)blocks, threads, 0, st>>>(in, out, legal, actions, N, A, fill); break;
    case 16: mask_logits_kernel<16><<<(unsigned)blocks, threads, 0, st>>>(in, out, legal, actions, N, A, fill); break;
    default: mask_logits_kernel<32><<<(unsigned)blocks, threads, 0, st>>>(in, out, legal, actions, N, A, fill); break;
  }
  return check_launch("mask_logits_kernel");
}

}  // namespace tb

using namespace tb;

static_assert(TB_MASKED_LOGIT == -FLT_MAX, "TB_MASKED_LOGIT is -FLT_MAX, torch.finfo(torch.float32).min");

extern "C" int tb_mask_logits_f32(const float* in, float* out, const uint8_t* legal, const int64_t* actions, int64_t N,
                                  int64_t A, float fill, void* stream) {
  return mask_logits(in, out, legal, actions, N, A, fill, stream);
}
