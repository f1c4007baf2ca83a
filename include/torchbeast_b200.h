/* torchbeast_b200 C-ABI: the drop-in boundary of the H100-native IMPALA learner hot path.
 *
 * Plain C, raw device pointers + sizes + a cudaStream_t passed as void*; no torch types.
 * The reference (facebookresearch/torchbeast) has NO FFI for this path - its boundary is
 * the Python function surface (SURVEY.md section 8(b) B1) - so every entry point below
 * names the reference Python function (file:line under /root/reference) whose device-side
 * work it replaces.  The Python mirror of that surface lives in torchbeast_b200/ and binds
 * these symbols with ctypes (see INTEGRATION.md for the stub a maintainer would add).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; tb_last_error() returns a
 *     thread-local message for the calling thread's last failure.
 *   - all pointers are DEVICE pointers unless the name ends in _host; buffers are owned by
 *     the caller (PyTorch caching allocator); outputs are written in place; nothing is
 *     allocated or freed by the library on the data path.
 *   - launches go to `stream` (the caller's current stream) and never synchronise.
 *   - layouts are the reference's: time-major, element (t,b) at offset t*B+b
 *     (logits: (t*B+b)*A + a), i.e. contiguous [T,B] / [T,B,A] tensors.
 *   - clip thresholds: a negative or NaN value means Python `None` (no clipping).
 *   - thread-safety: no global mutable state; reductions use the caller's `workspace`
 *     (tb_workspace_bytes() bytes, zero-initialised ONCE by the caller, self-cleaning).
 */
#ifndef TORCHBEAST_B200_H_
#define TORCHBEAST_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB_ABI_VERSION 1

int tb_abi_version(void);
const char* tb_last_error(void);
/* Number of SMs / compute capability of the current device (host query). */
int tb_device_info(int* sm_count_host, int* cc_major_host, int* cc_minor_host);
/* Bytes of zero-initialised scratch the reducing kernels need (counter + per-CTA partials). */
size_t tb_workspace_bytes(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
uint64_t tb_launch_count(void);
/* Optional per-op device timing: tb_profile_enable(1) clears and starts recording a CUDA event pair
 * around every op (GEMM, im2col, scan, ...) on its stream; tb_profile_collect synchronises the
 * device and returns the number of records, writing newline-separated op names to names_host and
 * the elapsed milliseconds to ms_host.  Off by default.                                      */
int tb_profile_enable(int on);
int tb_profile_collect(char* names_host, size_t names_cap, float* ms_host, int max_records);

/* ---- V-trace ----------------------------------------------------------------------- */

/* torchbeast/core/vtrace.py:50-55  action_log_probs(policy_logits, actions)
 * logits [N,A] f32, actions [N] i64 -> out [N] f32 = log_softmax(logits)[actions].       */
int tb_action_log_probs_f32(const float* logits, const int64_t* actions, int64_t N, int64_t A,
                            float* out, void* stream);
int tb_action_log_probs_f64(const double* logits, const int64_t* actions, int64_t N, int64_t A,
                            double* out, void* stream);

/* torchbeast/core/vtrace.py:91-139  from_importance_weights(...) -> VTraceReturns(vs, pg_advantages)
 * log_rhos/discounts/rewards/values [T,B], bootstrap [B]; outputs vs, pg_adv [T,B].
 * One launch; reverse-time scan, T split over warps with an affine-map combine.          */
int tb_vtrace_from_importance_weights_f32(const float* log_rhos, const float* discounts,
                                          const float* rewards, const float* values,
                                          const float* bootstrap, int64_t T, int64_t B,
                                          float clip_rho, float clip_pg_rho, float* vs,
                                          float* pg_adv, void* stream);
int tb_vtrace_from_importance_weights_f64(const double* log_rhos, const double* discounts,
                                          const double* rewards, const double* values,
                                          const double* bootstrap, int64_t T, int64_t B,
                                          double clip_rho, double clip_pg_rho, double* vs,
                                          double* pg_adv, void* stream);

/* Fused learner loss block: torchbeast/core/vtrace.py:58-88 (from_logits) +
 * monobeast.py:107-125 / polybeast_learner.py:113-131 (three losses) +
 * monobeast.py:245-277 / polybeast_learner.py:332-361 (reward clip, discounts, weighting)
 * and their closed-form backward (SURVEY.md section 8(a) A4), ONE launch.
 *
 * inputs (already shifted: batch[1:], learner_outputs[:-1]):
 *   behavior_logits, target_logits [T,B,A] f32; actions [T,B] i64; rewards [T,B] f32 (raw);
 *   done [T,B] u8 (bool) if `discounts`==NULL, else discounts [T,B] f32 used as is;
 *   values [T,B] f32; bootstrap [B] f32.
 * flags: clip_rewards!=0 clamps rewards to [-1,1] (reward_clipping == "abs_one").
 * outputs:
 *   vs, pg_adv, log_rhos, behavior_alp, target_alp [T,B] f32 (all required);
 *   losses_out [4] f32 = {pg_loss, baseline_cost*baseline_loss, entropy_cost*entropy_loss, total};
 *   grad_logits [T(+1),B,A], grad_values [T(+1),B] f32 = d total / d target_logits, d values
 *   (may both be NULL: forward only).  If zero_tail!=0 they have T+1 rows and row T is
 *   zero-filled (the bootstrap row of the learner outputs gets no gradient, vtrace.py:91).
 * workspace: tb_workspace_bytes() zero-initialised bytes (see conventions).                */
int tb_impala_loss_fwd_bwd_f32(const float* behavior_logits, const float* target_logits,
                               const int64_t* actions, const float* rewards,
                               const uint8_t* done, const float* discounts, const float* values,
                               const float* bootstrap, int64_t T, int64_t B, int64_t A,
                               float discounting, float baseline_cost, float entropy_cost,
                               int clip_rewards, float clip_rho, float clip_pg_rho, float* vs,
                               float* pg_adv, float* log_rhos, float* behavior_alp,
                               float* target_alp, float* losses_out, float* grad_logits,
                               float* grad_values, int zero_tail, void* workspace, void* stream);

/* ---- seeded action sampling for the acting forward ------------------------------------ */

/* monobeast.py:618-619 / polybeast_learner.py:256-257  torch.multinomial(F.softmax(policy_logits, dim=1), 1) as a
 * stateless, counter-based sampler: an action depends only on (seed, step, stream id, logits row), never on batch
 * composition, threads or torch's generator.  logits [T,B,A] f32 contiguous; stream_ids [B] i64, or NULL: column b
 * uses stream id b; actions [T,B] i64 out.  For row (t,b), with sid = stream_ids[b]:
 *   1. x = word 0 of Philox4x32-10(counter, key), counter = (lo32(step+t), hi32(step+t), lo32(sid), hi32(sid)),
 *      key = (lo32(seed), hi32(seed))  (all arithmetic mod 2^64, sid taken as its two's-complement bits);
 *   2. u = (x >> 8) * 2^-24, a 24-bit uniform in [0,1), exact in fp32;
 *   3. m = the row's maximum; e_a = expf(l_a - m) (precise expf, not __expf); S = sum of e_a in fp32, in index order;
 *   4. action = the smallest a whose fp32 running sum e_0 + ... + e_a is strictly greater than the fp32 product u*S;
 *      if rounding leaves no such a, the last a with e_a > 0;
 *   5. -inf logits are never chosen.  A row that contains a NaN, whose logits are all -inf, or that has a +inf logit
 *      gets action -1 (the kernel does not trap).
 * Because the counter is step + t, one [T,B] call gives the same actions as T calls of [1,B] at step, step+1, ...
 * Sizes: T, B >= 0, A >= 1; T*B == 0 is a no-op success.                                                        */
int tb_sample_actions_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                          const int64_t* stream_ids, int64_t* actions, void* stream);
/* The same contract, bit for bit, with seed = seed_step[0] and step = seed_step[1] read from device memory when the
 * kernel runs: a launch captured in a CUDA graph samples at whatever (seed, step) was written there before each
 * replay.  Same host validation, and a null seed_step is rejected.                                              */
int tb_sample_actions_dev_f32(const float* logits, int64_t T, int64_t B, int64_t A, const uint64_t* seed_step,
                              const int64_t* stream_ids, int64_t* actions, void* stream);

/* ---- the three loss functions on their own (API mirror; tests pass float64) ---------- */

/* monobeast.py:107-108 compute_baseline_loss: out[0] = 0.5*sum(adv^2); grad (nullable) = adv. */
int tb_baseline_loss_f32(const float* adv, int64_t N, float* out, float* grad, void* workspace, void* stream);
int tb_baseline_loss_f64(const double* adv, int64_t N, double* out, double* grad, void* workspace, void* stream);
/* monobeast.py:111-115 compute_entropy_loss: out[0] = sum(p*log p) over [N,A]; grad nullable [N,A]. */
int tb_entropy_loss_f32(const float* logits, int64_t N, int64_t A, float* out, float* grad, void* workspace, void* stream);
int tb_entropy_loss_f64(const double* logits, int64_t N, int64_t A, double* out, double* grad, void* workspace, void* stream);
/* monobeast.py:118-125 compute_policy_gradient_loss: out[0] = sum(-log pi(a)*adv); grad nullable
 * [N,A] = adv*(p - onehot(a)) (advantages get no gradient).                               */
int tb_pg_loss_f32(const float* logits, const int64_t* actions, const float* adv, int64_t N, int64_t A,
                   float* out, float* grad, void* workspace, void* stream);
int tb_pg_loss_f64(const double* logits, const int64_t* actions, const double* adv, int64_t N, int64_t A,
                   double* out, double* grad, void* workspace, void* stream);

/* ---- AtariNet (monobeast.py:545-635) forward / backward --------------------------------- */

/* Parameters live in ONE flat f32 buffer in the reference's state_dict order and shapes
 * (BASELINE.md section 5): conv1.weight (32,4,8,8), conv1.bias, conv2.weight (64,32,4,4), conv2.bias,
 * conv3.weight (64,64,3,3), conv3.bias, fc.weight (512,3136), fc.bias, [core.weight_ih_l0,
 * core.weight_hh_l0, core.bias_ih_l0, core.bias_hh_l0, ...l1 (2076 x 519 each)], policy.weight (A,519),
 * policy.bias, baseline.weight (1,519), baseline.bias.  Gradients use the same layout.       */
int64_t tb_atarinet_param_count(int num_actions, int use_lstm);
/* Bytes of caller-owned workspace for a [T1,B] rollout (T1 = unroll_length + 1): patch matrices,
 * activations kept for backward, packed weights, split-K scratch.                            */
size_t tb_atarinet_workspace_bytes(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision);

/* monobeast.py:582-632 AtariNet.forward (without the action sampling, which the learner never
 * uses - SURVEY.md K8).  frame u8 [T1,B,4,84,84]; reward f32 [T1,B]; last_action i64 [T1,B];
 * notdone f32 [T1,B] = (~done).float() (LSTM only; multiplies the state before each step,
 * monobeast.py:607-609); h0,c0 / hN,cN f32 [2,B,519] (LSTM only).
 * -> policy_logits f32 [T1,B,A], baseline f32 [T1,B].  Activations stay in `workspace`.
 * precision: 0 = fp32 SIMT GEMMs (bit-comparable with the reference's fp32 CPU arithmetic);
 *            1 = bf16 operands with fp32 accumulation: conv/fc trunk (implicit-GEMM convolutions) and LSTM
 *                projections on wgmma tensor cores, LSTM recurrence products as bf16 mma.sync; LSTM state and
 *                gate math, heads, losses, optimizer, master weights and gradients stay fp32.             */
int tb_atarinet_forward(const uint8_t* frame, const float* reward, const float* notdone,
                        const int64_t* last_action, const float* h0, const float* c0,
                        const float* params, int64_t T1, int64_t B, int num_actions, int use_lstm,
                        int precision, void* workspace, float* policy_logits, float* baseline, float* hN,
                        float* cN, void* stream);
/* Backward of the above (replaces the autograd graph of total_loss.backward(), monobeast.py:290):
 * grad_logits [T1,B,A], grad_baseline [T1,B] -> grads (flat, parameter layout, overwritten).
 * Must follow a tb_atarinet_forward on the same workspace and parameters.                    */
int tb_atarinet_backward(const float* grad_logits, const float* grad_baseline, const float* notdone,
                         const float* params, int64_t T1, int64_t B, int num_actions, int use_lstm,
                         int precision, void* workspace, float* grads, void* stream);

/* The same backward in two calls, for data-parallel learners (the reference has a single learner device,
 * polybeast_learner.py:402-405; SURVEY 8(e) G1 "bucket order = reverse of forward"): phase 1 = policy/baseline heads +
 * LSTM, phase 2 = conv/fc trunk.  After phase 2 everything is final; after phase 1 the slice
 * [tb_atarinet_grad_split(), param_count) of `grads` (LSTM + heads: 17 of 24 MB) is final when the LSTM weight-gradient
 * GEMMs ran on the caller's stream; when they were forked onto the side stream (tensor-core backends), the slice is
 * final in STREAM ORDER on that side stream: pass your own with tb_set_aux_stream() (thread-local; NULL = library-owned)
 * before phase 1, make it wait for `stream`, and enqueue the slice's all-reduce on it - it then overlaps phase 2.      */
int tb_set_aux_stream(void* stream);
int64_t tb_atarinet_grad_split(int num_actions, int use_lstm);
int tb_atarinet_backward_phase(const float* grad_logits, const float* grad_baseline, const float* notdone,
                               const float* params, int64_t T1, int64_t B, int num_actions, int use_lstm,
                               int precision, void* workspace, float* grads, int phase, void* stream);

/* ---- stacked LSTM over the unroll with per-step done-reset -------------------------------------------
 * Replaces the reference's loop of seq_len-1 nn.LSTM calls and its autograd graph (monobeast.py:603-611,
 * polybeast_learner.py:241-249):   for t: state *= notdone_t;  y_t, state = LSTM(x_t, state).
 * torch.nn.LSTM conventions: params[4*l + {0,1,2,3}] = weight_ih_l [4H, In|H], weight_hh_l [4H, H], bias_ih_l [4H],
 * bias_hh_l [4H] (gate order i, f, g, o); 1 or 2 layers; hidden size, input size, batch and unroll are free
 * (BASELINE configs[4]: T = 600, B = 128, H = 512).  x [T1*B, In], notdone [T1*B] (float 0/1), h0/c0/hN/cN [layers, B, H],
 * y [T1*B, H].  precision 0 = fp32 everywhere (any shape); 1 / 2 = bf16 / split-bf16 tensor-core products for the hoisted
 * projections.  tb_lstm_backward must follow tb_lstm_forward on the same workspace; grads[] mirrors params[] and is
 * overwritten; dx [T1*B, In].                                                                                        */
size_t tb_lstm_workspace_bytes(int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision);
int tb_lstm_forward(const float* x, const float* notdone, const float* h0, const float* c0, const float* const* params,
                    int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision, void* workspace,
                    float* y, float* hN, float* cN, void* stream);
int tb_lstm_backward(const float* dy, const float* x, const float* notdone, const float* const* params, float* const* grads,
                     int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision, void* workspace,
                     float* dx, void* stream);

/* ---- IMPALA ResNet (polybeast_learner.py:134-266 `Net`) forward / backward ------------------------- */

/* Flat parameter layout = the reference's state_dict order: feat_convs.{0,1,2}.0.{weight,bias}
 * ((16,4,3,3) (32,16,3,3) (32,32,3,3)), resnet1.{0,1,2}.{1,3}.{weight,bias}, resnet2.{0,1,2}.{1,3}.{weight,bias},
 * fc.{weight (256,3872), bias}, [core.weight_ih_l0 (1024,257), core.weight_hh_l0 (1024,256), core.bias_ih_l0,
 * core.bias_hh_l0], policy.{weight (A,257|256), bias}, baseline.{weight, bias}.                       */
int64_t tb_resnet_param_count(int num_actions, int use_lstm);
size_t tb_resnet_workspace_bytes(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision);
/* polybeast_learner.py:214-266 Net.forward without the action sampling: frame u8 [T1,B,4,84,84], reward f32
 * [T1,B], notdone f32 [T1,B] and h0,c0/hN,cN f32 [1,B,256] (LSTM only) -> policy_logits [T1,B,A], baseline [T1,B].
 * precision: 0 = fp32 SIMT patch-matrix GEMMs; 1 = bf16 activations + patch-matrix wgmma GEMMs (not parity-grade);
 * 2 = split-bf16 (the Python default): fp32 activations, every 3x3 conv as a shifted-window implicit GEMM over padded
 * channel-chunk-planar hi/lo images (csrc/conv3x3_sw.cu), the H=256 LSTM on one thread-block cluster.  T1*B < 65536.
 * The same precision and workspace must be used for forward and backward.                                            */
int tb_resnet_forward(const uint8_t* frame, const float* reward, const float* notdone, const float* h0,
                      const float* c0, const float* params, int64_t T1, int64_t B, int num_actions, int use_lstm,
                      int precision, void* workspace, float* policy_logits, float* baseline, float* hN, float* cN,
                      void* stream);
/* Backward of the forward pass that last ran on `workspace` (it keeps the conv input images / activations it needs). */
int tb_resnet_backward(const uint8_t* frame, const float* grad_logits, const float* grad_baseline,
                       const float* notdone, const float* params, int64_t T1, int64_t B, int num_actions,
                       int use_lstm, int precision, void* workspace, float* grads, void* stream);

/* ---- learner-queue ingest, host side (SURVEY 8(f) N1) --------------------------------------------------
 * One actor writes its [T1, ...] rollout into batch column b of a pinned [T1, B, ...] slot (replaces the per-rollout
 * tensors + torch::cat of src/cc/actorpool.cc:49-55,493-506): leaf l of the slot starts at slot_base + leaf_offset[l], one
 * (time step, column) row of it is row_bytes[l] bytes, src[l] is the actor's contiguous [T1, row] array (NULL = skip).
 * Pure host memcpy on the calling thread; no CUDA call.                                                           */
int tb_host_write_rollout_column(uint8_t* slot_base, const int64_t* leaf_offset, const int64_t* row_bytes, int num_leaves,
                                 int64_t T1, int64_t B, int64_t b, const uint8_t* const* src);

/* ---- flat-buffer optimizer step ------------------------------------------------------------ */

/* out_sumsq[0] = sum(grads^2) (double accumulation, deterministic).  First half of
 * nn.utils.clip_grad_norm_ (monobeast.py:291); grads must be 16-byte aligned.                */
int tb_grad_sumsq_f32(const float* grads, int64_t n, float* out_sumsq, void* workspace, void* stream);
/* Second half of clip_grad_norm_ fused with torch.optim.RMSprop.step() (monobeast.py:292,388-394):
 *   coef = min(1, max_norm/(sqrt(sumsq)+1e-6)) (max_norm < 0: no clipping); grads *= coef (left
 *   clipped in place like the reference); square_avg = alpha*square_avg + (1-alpha)*g^2;
 *   params -= lr * g/(sqrt(square_avg)+eps)   (momentum != 0: buf = momentum*buf + g/avg; params -= lr*buf).
 * lr_device (nullable) overrides `lr` with a device scalar; grad_norm_out (nullable) receives the
 * pre-clip norm.  No host synchronisation.                                                   */
int tb_clip_rmsprop_step_f32(float* params, float* grads, float* square_avg, float* momentum_buf, int64_t n,
                             const float* sumsq, float max_norm, const float* lr_device, float lr, float alpha,
                             float eps, float momentum, float* grad_norm_out, void* stream);

/* ---- bf16 tensor-core GEMM (wgmma + TMA), the throughput backend of the network -------- */

/* C[M,N] = relu?( scale * (A[M,K] . B[N,K]^T) + bias[N] );  A, B bf16 with K contiguous ("K-major"),
 * lda/ldb multiples of 8, 16-byte aligned; outputs fp32 C (ldc) and/or bf16 C_bf16 (ldc16), either may
 * be NULL.  Replaces the cuBLAS/cuDNN calls behind F.linear / F.conv2d-as-GEMM (monobeast.py:587-591). */
int tb_gemm_bf16_tn(const void* A_bf16, const void* B_bf16, int64_t M, int64_t N, int64_t K, int64_t lda,
                    int64_t ldb, float* C, int64_t ldc, void* C_bf16, int64_t ldc16, const float* bias,
                    float scale, int relu, void* stream);
/* General operand layouts of the same kernel: a_mn / b_mn != 0 mark an operand stored with the
 * REDUCTION index as its row index (A as [K,M], B as [K,N], row-major) - the dgrad (b_mn) and wgrad
 * (a_mn and b_mn) forms, so no transposed copies are needed.  splits > 1 reduces K over grid.z through
 * `partial` (splits*M*roundup(N,32) floats: rows padded so the tiles store 16 bytes) with a fixed-order second pass.  C fp32 [M,N] (ldc).            */
int tb_gemm_bf16_ex(const void* A_bf16, const void* B_bf16, int64_t M, int64_t N, int64_t K, int64_t lda,
                    int64_t ldb, int a_mn, int b_mn, float* C, int64_t ldc, int splits, float* partial,
                    void* stream);
/* ---- implicit-GEMM convolutions (bf16 tensor-core backend) -------------------------------------------
 * The nn.Conv2d layers of AtariNet (monobeast.py:560-562: 8x8/4, 4x4/2, 3x3/1, no padding) as wgmma GEMMs whose
 * patch operand is read by TMA straight from the bf16 NHWC activation [Nf,H,W,C] (conv2/conv3) or gathered from a
 * bf16 image of the uint8 NCHW frames (conv1) - no patch matrix is materialised.  weight / dweight are fp32 in the
 * reference layout [O,C,KH,KW]; outputs bf16 NHWC.  *_scratch buffers are caller-owned device memory:
 * pack_scratch_bf16 >= max(O,4*C)*KH*KW*max(C,O) bf16, partial >= 132*O*KH*KW*C floats (one split per SM), image_bf16 = N*4*H*W bf16. */
int tb_conv_nhwc_bf16_fwd(const void* act_bf16, const float* weight, const float* bias, int64_t Nf, int H, int W, int C,
                          int KH, int KW, int S, int O, int relu, void* out_bf16, void* pack_scratch_bf16, void* stream);
/* dx = conv_transpose(dy, weight) * (act > 0)   (act_bf16 nullable: no ReLU mask); O must be 64, stride 1 or 2 (4x4) */
int tb_conv_nhwc_bf16_dgrad(const void* dy_bf16, const float* weight, const void* act_bf16, int64_t Nf, int H, int W, int C,
                            int KH, int KW, int S, int O, void* dx_bf16, void* pack_scratch_bf16, void* stream);
int tb_conv_nhwc_bf16_wgrad(const void* dy_bf16, const void* act_bf16, int64_t Nf, int H, int W, int C, int KH, int KW, int S,
                            int O, float* dweight, float* partial, int64_t partial_floats, void* stream);
/* conv1: frame u8 [N,4,H,W] -> relu(conv(frame/255) + b) bf16 [N,OH,OW,32]; leaves the bf16 image for the wgrad */
int tb_conv1_u8_fwd(const uint8_t* frame, const float* weight, const float* bias, int64_t N, int H, int W, int S, int relu,
                    void* out_bf16, void* image_bf16, void* pack_scratch_bf16, void* stream);
int tb_conv1_u8_wgrad(const void* dy_bf16, const void* image_bf16, int64_t N, int H, int W, int S, float* dweight,
                      float* partial, int64_t partial_floats, void* stream);
/* out_bf16[r, c] = bf16(in[r*ld + c]) for c < cols, 0 for cols <= c < ld16 (operand staging). */
int tb_f32_to_bf16(const float* in, void* out_bf16, int64_t rows, int64_t cols, int64_t ld, int64_t ld16,
                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TORCHBEAST_B200_H_ */
