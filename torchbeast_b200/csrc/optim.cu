// Flat-buffer optimizer step for the learner: global-norm gradient clip + RMSprop, two launches
// over ONE contiguous parameter/gradient buffer (instead of ~100 foreach launches).
//
// Replaces, per learn() step (paths under /root/reference/torchbeast/):
//   nn.utils.clip_grad_norm_(model.parameters(), flags.grad_norm_clipping)   monobeast.py:291
//   optimizer.step()  (torch.optim.RMSprop, centered=False, weight_decay=0)  monobeast.py:292,388-394
// In multi-GPU runs the NCCL all-reduce of the flat gradient sits between backward and
// tb_grad_sumsq_f32, so every rank clips and steps on the reduced gradient (SURVEY.md 8(e)).
// Pure HBM-bound streaming: 128-bit accesses, grid = multiple of the SM count.
#include "common.cuh"

namespace tb {

__global__ void grad_sumsq_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ out, void* ws) {
  double s = 0.0;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t n4 = n / 4;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  // squares of one 16-byte vector are summed in fp32 (4 terms), the running sum in fp64; 4 loads in flight
#pragma unroll 4
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = __ldg(g4 + i);
    s += double(fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w))));
  }
  for (int64_t i = n4 * 4 + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    s += double(g[i]) * g[i];
  double tot[3];
  if (grid_sum3(s, 0.0, 0.0, ws, tot)) out[0] = float(tot[0]);
}

// coef = min(1, max_norm / (norm + 1e-6)); g *= coef; sq = alpha*sq + (1-alpha) g^2;
// avg = sqrt(sq) + eps; momentum==0: p -= lr * g/avg; else buf = momentum*buf + g/avg; p -= lr*buf
__global__ void clip_rmsprop_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ sq,
                                    float* __restrict__ mom, int64_t n, const float* __restrict__ sumsq,
                                    float max_norm, const float* __restrict__ lr_dev, float lr_host, float alpha,
                                    float eps, float momentum, float* __restrict__ norm_out) {
  const float norm = sqrtf(sumsq[0]);
  float coef = 1.0f;
  if (max_norm >= 0.0f) coef = fminf(max_norm / (norm + 1e-6f), 1.0f);
  const float lr = lr_dev ? lr_dev[0] : lr_host;
  if (norm_out && blockIdx.x == 0 && threadIdx.x == 0) norm_out[0] = norm;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  int64_t done = 0;
  if (!mom && ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(sq)) & 15) == 0) {
    // 128-bit path (no momentum buffer: the learner's configuration)
    const int64_t n4 = n / 4;
    float4* p4 = reinterpret_cast<float4*>(p); float4* g4 = reinterpret_cast<float4*>(g); float4* s4 = reinterpret_cast<float4*>(sq);
#pragma unroll 2
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
      float4 gv = g4[i], sv = s4[i], pv = p4[i];
      gv.x *= coef; gv.y *= coef; gv.z *= coef; gv.w *= coef;
      sv.x = alpha * sv.x + (1.0f - alpha) * gv.x * gv.x; sv.y = alpha * sv.y + (1.0f - alpha) * gv.y * gv.y;
      sv.z = alpha * sv.z + (1.0f - alpha) * gv.z * gv.z; sv.w = alpha * sv.w + (1.0f - alpha) * gv.w * gv.w;
      pv.x -= lr * (gv.x / (sqrtf(sv.x) + eps)); pv.y -= lr * (gv.y / (sqrtf(sv.y) + eps));
      pv.z -= lr * (gv.z / (sqrtf(sv.z) + eps)); pv.w -= lr * (gv.w / (sqrtf(sv.w) + eps));
      g4[i] = gv; s4[i] = sv; p4[i] = pv;
    }
    done = n4 * 4;
  }
  for (int64_t i = done + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = g[i] * coef;
    g[i] = gi;
    const float s = alpha * sq[i] + (1.0f - alpha) * gi * gi;
    sq[i] = s;
    const float avg = sqrtf(s) + eps;
    if (mom) {
      const float b = momentum * mom[i] + gi / avg;
      mom[i] = b;
      p[i] -= lr * b;
    } else {
      p[i] -= lr * (gi / avg);
    }
  }
}

}  // namespace tb

using namespace tb;

extern "C" {

int tb_grad_sumsq_f32(const float* grads, int64_t n, float* out_sumsq, void* workspace, void* stream) {
  TB_REQUIRE(n >= 0 && out_sumsq && workspace, "tb_grad_sumsq_f32: bad arguments");
  TB_REQUIRE(n == 0 || grads, "tb_grad_sumsq_f32: null gradient buffer");
  TB_REQUIRE((reinterpret_cast<uintptr_t>(grads) & 15) == 0, "tb_grad_sumsq_f32: gradient buffer must be 16-byte aligned");
  int64_t blocks = (n / 4 + 255) / 256;
  if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
  if (blocks < 1) blocks = 1;
  ProfScope prof("grad_sumsq", (cudaStream_t)stream);
  grad_sumsq_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(grads, n, out_sumsq, workspace);
  return check_launch("grad_sumsq_kernel");
}

int tb_clip_rmsprop_step_f32(float* params, float* grads, float* square_avg, float* momentum_buf, int64_t n,
                             const float* sumsq, float max_norm, const float* lr_device, float lr, float alpha,
                             float eps, float momentum, float* grad_norm_out, void* stream) {
  TB_REQUIRE(n >= 0 && sumsq, "tb_clip_rmsprop_step_f32: bad arguments");
  if (n == 0) return 0;
  TB_REQUIRE(params && grads && square_avg, "tb_clip_rmsprop_step_f32: null buffer");
  TB_REQUIRE(momentum == 0.0f || momentum_buf, "tb_clip_rmsprop_step_f32: momentum needs a buffer");
  int64_t blocks = (n + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  ProfScope prof("clip_rmsprop", (cudaStream_t)stream);
  clip_rmsprop_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      params, grads, square_avg, momentum != 0.0f ? momentum_buf : nullptr, n, sumsq, max_norm, lr_device, lr, alpha,
      eps, momentum, grad_norm_out);
  return check_launch("clip_rmsprop_kernel");
}

}  // extern "C"
