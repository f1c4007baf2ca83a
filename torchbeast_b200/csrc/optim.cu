// Flat-buffer optimizer step for the learner: global-norm gradient clip + RMSprop, two launches
// over ONE contiguous parameter/gradient buffer (instead of ~100 foreach launches).  The same clip is
// also fused with Adam / AdamW (tb_clip_adam_step_f32) and with RMSprop's centered / weight_decay
// options (tb_clip_rmsprop_ex_step_f32); the default RMSprop keeps its own kernel below.
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

// clip_grad_norm_'s coefficient: min(max_norm / (norm + 1e-6), 1), NaN when the norm is NaN (torch clamps with
// torch.clamp, which propagates NaN, so one NaN gradient element turns the whole step into NaN); max_norm < 0: 1, no
// clipping.  Thread 0 of block 0 reports the pre-clip norm.
__device__ __forceinline__ float clip_coef(const float* sumsq, float max_norm, float* norm_out) {
  const float norm = sqrtf(sumsq[0]);
  if (norm_out && blockIdx.x == 0 && threadIdx.x == 0) norm_out[0] = norm;
  const float coef = max_norm / (norm + 1e-6f);
  return max_norm >= 0.0f ? (coef > 1.0f ? 1.0f : coef) : 1.0f;  // not fminf: fminf(NaN, 1) is 1
}

// coef = clip_coef(...); g *= coef; sq = alpha*sq + (1-alpha) g^2;
// avg = sqrt(sq) + eps; momentum==0: p -= lr * g/avg; else buf = momentum*buf + g/avg; p -= lr*buf
// hp (nullable) overrides max_norm, alpha, eps and momentum, as lr_dev overrides lr_host.
__global__ void clip_rmsprop_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ sq,
                                    float* __restrict__ mom, int64_t n, const float* __restrict__ sumsq,
                                    float max_norm, const float* __restrict__ lr_dev, float lr_host, float alpha,
                                    float eps, float momentum, const tb_hparams* __restrict__ hp,
                                    float* __restrict__ norm_out) {
  if (hp) { max_norm = hp->max_norm; alpha = hp->alpha; eps = hp->eps; momentum = hp->momentum; }
  const float coef = clip_coef(sumsq, max_norm, norm_out);
  const float lr = lr_dev ? lr_dev[0] : lr_host;
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

__device__ __forceinline__ bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

// One element of torch.optim.Adam / AdamW (non-amsgrad), in the op order of torch's single-tensor implementation.
// g is clipped and written back; the L2 term is added to a copy, as torch adds it to a temporary.
struct AdamArgs {
  float coef, lr, beta1, beta2, one_minus_beta1, one_minus_beta2, eps, wd, step_size, bc2_sqrt;
  int decoupled;
};

__device__ __forceinline__ void adam_elem(float& p, float& g, float& m, float& v, const AdamArgs& a) {
  g *= a.coef;
  float gi = g;
  if (a.wd != 0.0f) {
    if (a.decoupled) p *= 1.0f - a.lr * a.wd;
    else gi += a.wd * p;
  }
  m = a.beta1 * m + a.one_minus_beta1 * gi;
  v = a.beta2 * v + a.one_minus_beta2 * gi * gi;
  p -= a.step_size * (m / (sqrtf(v) / a.bc2_sqrt + a.eps));
}

// step[0] holds the number of completed steps; this call is step t = step[0] + 1.  Every block reads the counter;
// adam_step_advance_kernel, the next launch on the stream, increments it.
__global__ void clip_adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                 float* __restrict__ v, int64_t n, const float* __restrict__ sumsq, float max_norm,
                                 const float* __restrict__ lr_dev, float lr_host, double beta1, double beta2, float eps,
                                 float wd, int decoupled, const int64_t* __restrict__ step,
                                 const tb_hparams* __restrict__ hp, float* __restrict__ norm_out) {
  if (hp) { max_norm = hp->max_norm; beta1 = hp->beta1; beta2 = hp->beta2; eps = hp->eps; wd = hp->weight_decay; }
  AdamArgs a;
  a.coef = clip_coef(sumsq, max_norm, norm_out);
  a.lr = lr_dev ? lr_dev[0] : lr_host;
  // 1 - beta rounded from double, as torch passes it: 1 - float(0.999) would be off by 1.3e-5 relative
  a.beta1 = float(beta1); a.beta2 = float(beta2);
  a.one_minus_beta1 = float(1.0 - beta1); a.one_minus_beta2 = float(1.0 - beta2);
  a.eps = eps; a.wd = wd; a.decoupled = decoupled;
  // bias corrections in double from the double betas, as torch computes them on the host
  const double t = double(step[0] + 1);
  a.step_size = float(double(a.lr) / (1.0 - pow(beta1, t)));
  a.bc2_sqrt = float(sqrt(1.0 - pow(beta2, t)));
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  int64_t done = 0;
  if (aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v)) {
    const int64_t n4 = n / 4;
    float4* p4 = reinterpret_cast<float4*>(p); float4* g4 = reinterpret_cast<float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m); float4* v4 = reinterpret_cast<float4*>(v);
#pragma unroll 2
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
      float4 pv = p4[i], gv = g4[i], mv = m4[i], vv = v4[i];
      adam_elem(pv.x, gv.x, mv.x, vv.x, a); adam_elem(pv.y, gv.y, mv.y, vv.y, a);
      adam_elem(pv.z, gv.z, mv.z, vv.z, a); adam_elem(pv.w, gv.w, mv.w, vv.w, a);
      p4[i] = pv; g4[i] = gv; m4[i] = mv; v4[i] = vv;
    }
    done = n4 * 4;
  }
  for (int64_t i = done + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    adam_elem(p[i], g[i], m[i], v[i], a);
}

__global__ void adam_step_advance_kernel(int64_t* step) { step[0] += 1; }

// torch.optim.RMSprop with weight_decay and/or centered (grad_avg != nullptr), combined with momentum as torch does:
//   g += wd*p; sq = alpha*sq + (1-alpha) g^2; centered: ga = alpha*ga + (1-alpha) g, avg = sqrt(sq - ga^2) + eps,
//   else avg = sqrt(sq) + eps; momentum: buf = momentum*buf + g/avg, p -= lr*buf; else p -= lr * g/avg
struct RmsExArgs {
  float coef, lr, alpha, eps, wd, momentum;
};

__device__ __forceinline__ void rmsprop_ex_elem(float& p, float& g, float& sq, float* ga, float* buf,
                                                const RmsExArgs& a) {
  g *= a.coef;
  const float gi = g + a.wd * p;
  sq = a.alpha * sq + (1.0f - a.alpha) * gi * gi;
  float avg;
  if (ga) {
    *ga = a.alpha * *ga + (1.0f - a.alpha) * gi;
    avg = sqrtf(sq - *ga * *ga) + a.eps;
  } else {
    avg = sqrtf(sq) + a.eps;
  }
  if (buf) {
    *buf = a.momentum * *buf + gi / avg;
    p -= a.lr * *buf;
  } else {
    p -= a.lr * (gi / avg);
  }
}

__global__ void clip_rmsprop_ex_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ sq,
                                       float* __restrict__ ga, float* __restrict__ mom, int64_t n,
                                       const float* __restrict__ sumsq, float max_norm,
                                       const float* __restrict__ lr_dev, float lr_host, float alpha, float eps,
                                       float wd, float momentum, const tb_hparams* __restrict__ hp,
                                       float* __restrict__ norm_out) {
  if (hp) { max_norm = hp->max_norm; alpha = hp->alpha; eps = hp->eps; wd = hp->weight_decay; momentum = hp->momentum; }
  RmsExArgs a;
  a.coef = clip_coef(sumsq, max_norm, norm_out);
  a.lr = lr_dev ? lr_dev[0] : lr_host;
  a.alpha = alpha; a.eps = eps; a.wd = wd; a.momentum = momentum;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  int64_t done = 0;
  if (aligned16(p) && aligned16(g) && aligned16(sq) && aligned16(ga) && aligned16(mom)) {
    const int64_t n4 = n / 4;
    float4* p4 = reinterpret_cast<float4*>(p); float4* g4 = reinterpret_cast<float4*>(g);
    float4* s4 = reinterpret_cast<float4*>(sq); float4* a4 = reinterpret_cast<float4*>(ga);
    float4* b4 = reinterpret_cast<float4*>(mom);
#pragma unroll 2
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
      float4 pv = p4[i], gv = g4[i], sv = s4[i];
      float4 av = ga ? a4[i] : make_float4(0.f, 0.f, 0.f, 0.f), bv = mom ? b4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      rmsprop_ex_elem(pv.x, gv.x, sv.x, ga ? &av.x : nullptr, mom ? &bv.x : nullptr, a);
      rmsprop_ex_elem(pv.y, gv.y, sv.y, ga ? &av.y : nullptr, mom ? &bv.y : nullptr, a);
      rmsprop_ex_elem(pv.z, gv.z, sv.z, ga ? &av.z : nullptr, mom ? &bv.z : nullptr, a);
      rmsprop_ex_elem(pv.w, gv.w, sv.w, ga ? &av.w : nullptr, mom ? &bv.w : nullptr, a);
      p4[i] = pv; g4[i] = gv; s4[i] = sv;
      if (ga) a4[i] = av;
      if (mom) b4[i] = bv;
    }
    done = n4 * 4;
  }
  for (int64_t i = done + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    rmsprop_ex_elem(p[i], g[i], sq[i], ga ? ga + i : nullptr, mom ? mom + i : nullptr, a);
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

// hp == NULL takes the scalar arguments and checks them; else the kernels read the scalars from hp, and momentum_buf is
// passed as given: the caller passes it exactly when momentum is non-zero.
int tb_clip_rmsprop_step_f32(float* params, float* grads, float* square_avg, float* momentum_buf, int64_t n,
                             const float* sumsq, float max_norm, const float* lr_device, float lr, float alpha,
                             float eps, float momentum, const tb_hparams* hp, float* grad_norm_out, void* stream) {
  TB_REQUIRE(n >= 0 && sumsq, "tb_clip_rmsprop_step_f32: bad arguments");
  if (n == 0) return 0;
  TB_REQUIRE(params && grads && square_avg, "tb_clip_rmsprop_step_f32: null buffer");
  if (!hp) {
    TB_REQUIRE(momentum == 0.0f || momentum_buf, "tb_clip_rmsprop_step_f32: momentum needs a buffer");
    if (momentum == 0.0f) momentum_buf = nullptr;
  }
  int64_t blocks = (n + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  ProfScope prof("clip_rmsprop", (cudaStream_t)stream);
  clip_rmsprop_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      params, grads, square_avg, momentum_buf, n, sumsq, max_norm, lr_device, lr, alpha, eps, momentum, hp,
      grad_norm_out);
  return check_launch("clip_rmsprop_kernel");
}

int tb_clip_adam_step_f32(float* params, float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, const float* sumsq,
                          float max_norm, const float* lr_device, float lr, double beta1, double beta2, float eps,
                          float weight_decay, int decoupled, int64_t* step_device, const tb_hparams* hp,
                          float* grad_norm_out, void* stream) {
  TB_REQUIRE(n >= 0 && sumsq && step_device, "tb_clip_adam_step_f32: bad arguments");
  TB_REQUIRE(n == 0 || (params && grads && exp_avg && exp_avg_sq), "tb_clip_adam_step_f32: null buffer");
  TB_REQUIRE(hp || (beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0),
             "tb_clip_adam_step_f32: betas must be in [0, 1)");
  int64_t blocks = (n + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  if (blocks < 1) blocks = 1;  // n == 0 still counts the step
  ProfScope prof("clip_adam", (cudaStream_t)stream);
  clip_adam_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      params, grads, exp_avg, exp_avg_sq, n, sumsq, max_norm, lr_device, lr, beta1, beta2, eps, weight_decay,
      decoupled, step_device, hp, grad_norm_out);
  if (int rc = check_launch("clip_adam_kernel")) return rc;
  adam_step_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_device);
  return check_launch("adam_step_advance_kernel");
}

int tb_clip_rmsprop_ex_step_f32(float* params, float* grads, float* square_avg, float* grad_avg, float* momentum_buf,
                                int64_t n, const float* sumsq, float max_norm, const float* lr_device, float lr,
                                float alpha, float eps, float weight_decay, float momentum, const tb_hparams* hp,
                                float* grad_norm_out, void* stream) {
  TB_REQUIRE(n >= 0 && sumsq, "tb_clip_rmsprop_ex_step_f32: bad arguments");
  if (n == 0) return 0;
  TB_REQUIRE(params && grads && square_avg, "tb_clip_rmsprop_ex_step_f32: null buffer");
  if (!hp) {
    TB_REQUIRE(momentum == 0.0f || momentum_buf, "tb_clip_rmsprop_ex_step_f32: momentum needs a buffer");
    if (momentum == 0.0f) momentum_buf = nullptr;
  }
  int64_t blocks = (n + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  ProfScope prof("clip_rmsprop_ex", (cudaStream_t)stream);
  clip_rmsprop_ex_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      params, grads, square_avg, grad_avg, momentum_buf, n, sumsq, max_norm, lr_device, lr, alpha, eps, weight_decay,
      momentum, hp, grad_norm_out);
  return check_launch("clip_rmsprop_ex_kernel");
}

}  // extern "C"
