// Policy / baseline heads (monobeast.py:613-614, polybeast_learner.py:251-252): two tiny linear layers over the
// core output, fused.  A GEMM tile is the wrong shape for [N, F] x [F, A+1] with A+1 ~ 7 outputs: the tiled
// GEMM would read core_out many times; these kernels stream it once.
#pragma once
#include "common.cuh"

namespace tb {

// V value outputs (V = 1: the reference's single baseline; V > 1: one per task, PopArt)
constexpr int kHeadsMaxValues = 64;
// The backward's weight-gradient partials: at most this many slabs of rows (64 rows each up to N = 64 * kHeadsMaxSlabs,
// longer slabs beyond), so heads_scratch_floats stops growing with N.  Sized so that every A < 32, V <= 64, F <= 700
// case fits in 8 M floats: 120 * (31 + 64) * 701 = 7.99 M.
constexpr int kHeadsMaxSlabs = 120;

// logits[n, a] = x[n, :] . Wp[a, :] + bp[a];  baseline[n, v] = x[n, :] . Wb[v, :] + bb[v]
int heads_forward(const float* x, int64_t ldx, const float* Wp, const float* bp, const float* Wb, const float* bb, int64_t N, int F,
                  int A, float* logits, float* baseline, cudaStream_t stream, int V = 1);

// dx[n, f] = sum_v dbaseline[n, v] Wb[v, f] + sum_a dlogits[n, a] Wp[a, f]
// dWp[a, f] = sum_n dlogits[n, a] x[n, f];  dbp[a] = sum_n dlogits[n, a];  dWb[v, f] = sum_n dbaseline[n, v] x[n, f];
// dbb[v] = sum_n dbaseline[n, v]  (fixed-order two-stage reductions; scratch >= heads_scratch_floats(N, F, A, V) floats,
// at most kHeadsMaxSlabs * (A + V) * (F + 1))
int64_t heads_scratch_floats(int64_t N, int F, int A, int V = 1);
int heads_backward(const float* x, int64_t ldx, const float* Wp, const float* Wb, const float* dlogits, const float* dbaseline,
                   int64_t N, int F, int A, float* dx, int64_t lddx, float* dWp, float* dbp, float* dWb, float* dbb, float* scratch,
                   cudaStream_t stream, int V = 1);

}  // namespace tb
