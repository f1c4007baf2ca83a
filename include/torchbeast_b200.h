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

/* ---- hyper-parameters read from device memory ------------------------------------------
 * The scalar arguments of the loss and optimizer steps, as one block in device memory.  Given a non-NULL `hp`,
 * tb_impala_loss_f32 and the tb_clip_*_step_f32 entry points read their values from it when the kernel runs, so a
 * captured CUDA graph follows changes the caller publishes between replays (annealed costs, population-based
 * training).  Every value derived from them (1 - alpha, 1 - beta, the clip coefficient, the bias corrections) is
 * computed in the kernel by the same expression as from the float arguments, so both give bit-identical results for
 * the same values.  Layout is fixed: tb_hparams_layout() reports it, so a binding can check its packing without a
 * GPU.                                                                                                            */
typedef struct tb_hparams {
  double beta1, beta2;         /* Adam / AdamW, in [0, 1); double as in tb_clip_adam_step_f32                  */
  float discounting;           /* used where done is given; a `discounts` array is used as is                  */
  float baseline_cost, entropy_cost;
  float clip_rho, clip_pg_rho; /* negative or NaN: no clipping (Python None)                                   */
  int32_t clip_rewards;        /* != 0: clamp rewards to [-1, 1]                                               */
  float max_norm;              /* gradient-norm clip; negative: no clipping                                    */
  float alpha, eps, momentum, weight_decay; /* RMSprop: alpha, eps, momentum, weight_decay; Adam: eps, weight_decay */
} tb_hparams;
/* Host only: out[0] = sizeof(tb_hparams), out[1..13] = offsetof of discounting, baseline_cost, entropy_cost,
 * clip_rho, clip_pg_rho, clip_rewards, max_norm, alpha, eps, momentum, weight_decay, beta1, beta2.           */
int tb_hparams_layout(int64_t* out_host);

/* Fused learner loss block: torchbeast/core/vtrace.py:58-88 (from_logits) +
 * monobeast.py:107-125 / polybeast_learner.py:113-131 (three losses) +
 * monobeast.py:245-277 / polybeast_learner.py:332-361 (reward clip, discounts, weighting)
 * and their closed-form backward (SURVEY.md section 8(a) A4), ONE launch.  Each feature group below (hp, importance
 * weights, PopArt, trust region) is off when its pointer is NULL; with all of them NULL this is the plain loss block.
 *
 * inputs (already shifted: batch[1:], learner_outputs[:-1]):
 *   behavior_logits, target_logits [T,B,A] f32; actions [T,B] i64; rewards [T,B] f32 (raw);
 *   done [T,B] u8 (bool) if `discounts`==NULL, else discounts [T,B] f32 used as is;
 *   values [T,B] f32; bootstrap [B] f32.
 * flags: clip_rewards!=0 clamps rewards to [-1,1] (reward_clipping == "abs_one").
 * hp: NULL takes discounting, baseline_cost, entropy_cost, clip_rewards, clip_rho and clip_pg_rho from the
 *   arguments; else they are read from hp (device pointer, see tb_hparams) when the kernel runs, and the scalar
 *   arguments are not read.
 * outputs:
 *   vs, pg_adv, log_rhos, behavior_alp, target_alp [T,B] f32 (all required);
 *   losses_out [4] f32 = {pg_loss, baseline_cost*baseline_loss, entropy_cost*entropy_loss, total};
 *   grad_logits [T(+1),B,A], grad_values [T(+1),B] f32 = d total / d target_logits, d values
 *   (may both be NULL: forward only).  If zero_tail!=0 they have T+1 rows and row T is
 *   zero-filled (the bootstrap row of the learner outputs gets no gradient, vtrace.py:91).
 * workspace: tb_workspace_bytes() zero-initialised bytes (see conventions).
 *
 * ---- importance weights: column_weights [B] f32 (device; NULL: unweighted).  The pg, baseline and entropy terms of
 * every row (t, b) are multiplied by column_weights[b], in losses_out and in grad_logits / grad_values (after the
 * unweighted term is formed, so weights of 1.0f give the bits of column_weights = NULL; a weight of 0 gives zero
 * gradient rows).  vs, pg_adv, log_rhos and the log-probabilities are not weighted.
 *
 * ---- trust region for off-policy V-trace (Schmitt, Hessel & Simonyan, ICML 2020, "Off-Policy Actor-Critic with
 * Shared Experience Replay": LASER's beta trust region): trust_beta (f32 [1], device, read when the kernel runs; NULL:
 * no trust region), kl_out [T,B] f32 and trust_out [2] f32 (both required with trust_beta).  For every row (t, b) of
 * the shifted inputs:
 *   kl_t = sum_a pi_t(a) (log pi_t(a) - log mu_t(a)) in fp32, pi = softmax(target_logits), mu = softmax(behavior_logits),
 *          both log-softmaxes from the max / log-sum-exp the action log-probabilities are formed with (behavior_alp and
 *          target_alp keep their bits); written to kl_out.
 *   m_t  = (kl_t <= beta), a comparison: a NaN kl_t is untrusted.
 *   V-trace and the policy gradient use rho_t * m_t in place of rho_t: at an untrusted row the clipped rho, c_t and the
 *   pg clip ratio are all 0, so its TD error adds nothing, the trace is cut there and its pg_adv is 0 (no pg loss, no
 *   pg gradient).  The baseline and entropy terms are unchanged; where every later trace is cut, vs_t = V_t.  m is a
 *   constant for the backward: no gradient flows through kl.
 *   log_rhos, behavior_alp and target_alp are the true, unmasked values; vs and pg_adv are the masked ones.
 * trust_out = {number of trusted rows, sum of kl_t over all T*B rows}: fp64 sums in a fixed order (no atomics), bit-
 * identical from run to run, rounded to f32 once.  beta = +inf on finite inputs gives the bits of trust_beta = NULL
 * (with the same hp, column_weights and PopArt arguments) in every output; identical behaviour and target logits give
 * kl = 0 exactly, so beta = 0 trusts those rows.  With PopArt the per-task sums come from the masked vs.
 *
 * ---- PopArt value normalisation (van Hasselt et al. 2016; Hessel et al. 2019): task non-NULL.
 * Per task k, statistics mu[k], nu[k] (f64, device; start at 0 and 1) with
 *   sigma_k = clamp(sqrt(max(nu_k - mu_k^2, 0)), 1e-4, 1e6).
 * The loss block then runs on a normalised value head:
 *   values [T+1,B,K] f32 = normalised head outputs n, bootstrap row T included (bootstrap is not read); task [T+1,B]
 *   i64, row (t,b) uses k = task[t*B+b].  1. v = sigma_k * n[k] + mu_k (fp32, mu / sigma rounded once), the bootstrap
 *   with its own task.  2. V-trace on v as without PopArt: vs, pg_adv stay unnormalised.  3. policy gradient
 *   -log pi(a) * pg_adv / sigma_k, entropy unchanged.  4. baseline loss baseline_cost * 1/2 ((vs - mu_k)/sigma_k -
 *   n[k])^2; its gradient goes to column k of grad_values [T+1,B,K], every other column and row T get zero.
 *   A row whose task id is outside [0, K) adds no loss and gets zero gradient rows (its v is 0 in the V-trace); ids
 *   are not checked otherwise.  task_sums [3K] f64 out: count, sum vs and sum vs^2 of each task over rows t < T,
 *   bit-identical from run to run (no atomics).
 *   Requires 1 <= K <= 64, T >= 1, B >= 1, non-NULL mu, nu and task_sums, and zero_tail = 1; column_weights must be
 *   NULL.  Two launches.  NULL task: K, mu, nu and task_sums are not read.                                       */
int tb_impala_loss_f32(const float* behavior_logits, const float* target_logits, const int64_t* actions,
                       const float* rewards, const uint8_t* done, const float* discounts, const float* values,
                       const float* bootstrap, int64_t T, int64_t B, int64_t A, float discounting,
                       float baseline_cost, float entropy_cost, int clip_rewards, float clip_rho, float clip_pg_rho,
                       const tb_hparams* hp, const float* column_weights, const int64_t* task, const double* mu,
                       const double* nu, int64_t K, double* task_sums, const float* trust_beta, float* kl_out,
                       float* trust_out, float* vs, float* pg_adv, float* log_rhos, float* behavior_alp,
                       float* target_alp, float* losses_out, float* grad_logits, float* grad_values, int zero_tail,
                       void* workspace, void* stream);

/* UPGO, the upgoing policy gradient (Vinyals et al. 2019, "Grandmaster level in StarCraft II", Nature 575): a second
 * launch enqueued right after tb_impala_loss_f32 on the same stream.  It reads that launch's log_rhos and, with a
 * trust region, its kl_out, so rho and the mask have the same bits.  The other inputs are the loss call's own: target
 * logits, actions, rewards, done or discounts, values and bootstrap (or the PopArt values, task, mu, nu and K),
 * column_weights, hp (discounting, clip_rewards and clip_pg_rho are read from it when non-NULL, else from the
 * arguments) and trust_beta.  In the loss block's row notation (rows t = 0..T-1 of column b, shifted inputs):
 *   r_t    reward after the reward clip; g_t the discount, from done or discounts as the loss builds it;
 *   V_t    the value, V_T the bootstrap (PopArt: V_t = sigma_k n_t[k] + mu_k, 0 for a task out of range);
 *   rho_t  = exp(log_rhos_t).
 *   Trace switch, t = 0..T-2: lambda_{t+1} = 1 when r_{t+1} + g_{t+1} V_{t+2} >= V_{t+1}, else 0 (a comparison: NaN
 *     gives 0).
 *   Return: G_{T-1} = r_{T-1} + g_{T-1} V_T;  G_t = r_t + g_t (lambda_{t+1} G_{t+1} + (1 - lambda_{t+1}) V_{t+1}).
 *     A lambda-return whose lambda is 0 or 1 at each step; the split-T layout composes it as the loss composes V-trace.
 *   Advantage: A_t = rhobar_t (G_t - V_t), rhobar_t = min(rho_t m_t, clip_pg_rho) (unclipped when clip_pg_rho is
 *     negative or NaN, as in the V-trace policy gradient); m_t = (kl_t <= beta) with trust_beta, else 1.  PopArt: A_t
 *     is divided by sigma_k; a row whose task is out of range gets A_t = 0 and adds nothing.
 *   Loss: upgo_cost * sum_{t,b} w_b (-log pi_t(a_t)) A_t, with A constant; w_b = column_weights[b], or 1.
 *     Gradient: upgo_cost * w_b * A_t * (pi_t - onehot(a_t)), ADDED into grad_logits (NULL: forward only); row T and
 *     the values get nothing.
 * upgo_cost f32 [1] (device, read when the kernel runs).  outputs: upgo_adv [T,B] f32 = A; upgo_out [1] f32 = the
 * loss; losses_out[3] (the loss launch's total) becomes float(double(total) + double(upgo_out)).  When *upgo_cost == 0
 * grad_logits and losses_out are not written, so a zero cost leaves the loss launch's bits.  The sum is fp64 in a fixed
 * order (no atomics): bit-identical from run to run.  workspace: the one the loss launch used (or any other).  PopArt
 * requires T >= 1, B >= 1, 1 <= K <= 64, non-NULL mu and nu, and NULL column_weights; trust_beta requires kl.  One
 * launch.                                                                                                          */
int tb_upgo_loss_f32(const float* target_logits, const int64_t* actions, const float* rewards, const uint8_t* done,
                     const float* discounts, const float* values, const float* bootstrap, int64_t T, int64_t B,
                     int64_t A, float discounting, int clip_rewards, float clip_pg_rho, const tb_hparams* hp,
                     const float* column_weights, const int64_t* task, const double* mu, const double* nu, int64_t K,
                     const float* log_rhos, const float* trust_beta, const float* kl, const float* upgo_cost,
                     float* upgo_adv, float* upgo_out, float* losses_out, float* grad_logits, void* workspace,
                     void* stream);

/* Kickstarting (Schmitt et al. 2018, "Kickstarting Deep Reinforcement Learning", arXiv:1803.03835): distils a frozen
 * teacher policy into the learner.  A launch enqueued after tb_impala_loss_f32 (and tb_upgo_loss_f32) on the same
 * stream, before the network backward.  teacher_logits and target_logits are [T,B,A]: the [:-1] prefixes of the
 * teacher's and the learner's [T+1,B,A] forward outputs.  In the loss block's row notation (rows t = 0..T-1 of column b):
 *   log p_T, log p_S  the row log-softmaxes of the two, by the max / log-sum-exp code the loss uses;
 *   KL_t = sum_a p_T(a) (log p_T(a) - log p_S(a)) in fp32; a term with p_T(a) == 0 adds exactly 0, so a teacher that
 *     masks actions with -inf logits gives no NaN.  Identical rows give KL_t = 0 and a gradient of +-0.
 *   Loss: kickstart_cost * sum_{t,b} w_b KL_t; w_b = column_weights[b], or 1.  Gradient: kickstart_cost * w_b *
 *     (p_S - p_T), ADDED into grad_logits rows t < T (NULL: forward only); row T, the values and the teacher get
 *     nothing.  The trust region's mask and PopArt do not apply.
 * kickstart_cost f32 [1] (device, read when the kernel runs).  outputs: kickstart_out [2] f32 = {the loss, sum_{t,b}
 * KL_t unweighted}, always written; losses_out[3] (the loss launch's total) becomes float(double(total) +
 * double(kickstart_out[0])).  When *kickstart_cost == 0 grad_logits and losses_out are not written, so a zero cost
 * leaves the loss launch's bits.  The sums are fp64 in a fixed order (no atomics): bit-identical from run to run.
 * workspace: the one the loss launch used (or any other).  Requires T, B, A >= 1.  One launch.                    */
int tb_kickstart_loss_f32(const float* teacher_logits, const float* target_logits, int64_t T, int64_t B, int64_t A,
                          const float* column_weights, const float* kickstart_cost, float* kickstart_out,
                          float* losses_out, float* grad_logits, void* workspace, void* stream);

/* tb_popart_update:for each task k with task_sums count > 0 (data-parallel callers SUM all-reduce task_sums
 *   first), with beta read from device memory and sigma_k as in tb_impala_loss_f32:
 *     mu'_k = (1 - beta) mu_k + beta * sum vs / count,   nu'_k = (1 - beta) nu_k + beta * sum vs^2 / count
 *   then rescales value-head row k so that its unnormalised outputs do not change:
 *     weight[k, :] *= sigma_k / sigma'_k,   bias[k] = (sigma_k * bias[k] + mu_k - mu'_k) / sigma'_k
 *   weight [K,F] and bias [K] f32 (e.g. inside a flat parameter buffer).  It runs after the optimizer step and does
 *   not touch optimizer state.  One launch, no host sync; graph-capturable.                                    */
int tb_popart_update(const double* task_sums, const double* beta, double* mu, double* nu, int64_t K, float* weight,
                     float* bias, int64_t F, void* stream);

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

/* ---- multi-discrete (factored) action spaces ------------------------------------------------------------------------
 * An action is a tuple (a_1 .. a_D) of D independent choices, component k taking one of A_k values (gym's MultiDiscrete).
 * The policy is a product of D categoricals, pi(a) = prod_k pi_k(a_k), each pi_k a softmax over a segment of the row:
 *   logits [.., A], A = A_1 + ... + A_D: component k owns columns [off_k, off_k + A_k), off_k = A_1 + ... + A_{k-1}
 *     (off_1 = 0; components are counted from 0 below, so off_0 = 0);
 *   actions and last_action int64 [.., D]: column k is a_k, in [0, A_k).
 * The space reaches the library as a host tb_action_space, read before the call returns.  1 <= num_components <=
 * TB_MAX_ACTION_COMPONENTS, dims[k] >= 1 for k < num_components (later entries are not read), and sum dims = A; an entry
 * given anything else fails with tb_last_error set.  Per row, every segment quantity below is formed by the code the flat
 * contract uses for its whole row, on the segment alone:
 *   log pi_k(a_k) = (l[off_k + a_k] - m_k) - logs_k, with m_k and logs_k the segment's max and log-sum-exp formed as
 *     tb_action_log_probs_f32 forms them; an a_k outside [0, A_k) gives NaN, which poisons the row as in the flat loss;
 *   log pi(a) = the fp32 sum over k in index order, from log pi_0(a_0) (no leading 0 is added);
 *   entropy term: ent_k = sum_{j in k} p_j lp_j in index order, ent = the sum of ent_k over k in index order;
 *   trust-region KL: KL_k = sum_{j in k} pi_j (lp_j - lmu_j) in index order, KL = the sum of KL_k over k in index order;
 *   gradient of segment k: adv * (p - onehot(a_k)) + entropy_cost * p * (lp - ent_k), weighted as in the flat loss.
 * Two properties follow: a component with A_k = 1 contributes exactly 0 to log pi, the entropy and the KL, and a
 * gradient of +-0; and a space whose components all have size 1 but one gives the flat contract's bits on that one.   */
#define TB_MAX_ACTION_COMPONENTS 16
typedef struct tb_action_space {
  int32_t num_components;                  /* D */
  int32_t dims[TB_MAX_ACTION_COMPONENTS];  /* A_k */
} tb_action_space;
/* Host only: out[0] = sizeof(tb_action_space), out[1] = offsetof num_components, out[2] = offsetof dims. */
int tb_action_space_layout(int64_t* out_host);
/* tb_impala_loss_f32 on a factored policy: the same arguments and outputs (hp block, column_weights, PopArt, trust
 * region; A = sum dims), with actions [T,B,D] and the per-segment rules above in place of the flat row's.  V-trace runs
 * on log rho = log pi(a) - log mu(a) of the whole tuple; the pg loss is -log pi(a) * pg_adv; target_alp / behavior_alp
 * are the summed log-probabilities.  With D = 1 it gives tb_impala_loss_f32's bits.  tb_upgo_loss_f32 and
 * tb_kickstart_loss_f32 take flat rows only.                                                                        */
int tb_impala_loss_factored_f32(const float* behavior_logits, const float* target_logits, const int64_t* actions,
                                const float* rewards, const uint8_t* done, const float* discounts, const float* values,
                                const float* bootstrap, int64_t T, int64_t B, int64_t A, float discounting,
                                float baseline_cost, float entropy_cost, int clip_rewards, float clip_rho,
                                float clip_pg_rho, const tb_hparams* hp, const float* column_weights,
                                const int64_t* task, const double* mu, const double* nu, int64_t K, double* task_sums,
                                const float* trust_beta, float* kl_out, float* trust_out, float* vs, float* pg_adv,
                                float* log_rhos, float* behavior_alp, float* target_alp, float* losses_out,
                                float* grad_logits, float* grad_values, int zero_tail, const tb_action_space* space,
                                void* workspace, void* stream);
/* Seeded sampling of a factored policy: logits [T,B,A] -> actions [T,B,D].  Component k of row (t,b) takes x = word
 * (k mod 4) of Philox4x32-10 with tb_sample_actions_f32's counter and key (lo32(seed), hi32(seed) + k/4) (mod 2^32),
 * then steps 2-5 of that contract on its segment (a segment with a NaN, all -inf or a +inf logit gets -1).  So D = 1
 * gives tb_sample_actions_f32's actions.  seed_step (device, nullable) wins over (seed, step), as in
 * tb_sample_actions_dev_f32, so one entry serves eager and graphed acting.  Sizes as tb_sample_actions_f32.          */
int tb_sample_actions_factored_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                                   const uint64_t* seed_step, const int64_t* stream_ids, const tb_action_space* space,
                                   int64_t* actions, void* stream);

/* ---- continuous (diagonal-Gaussian) action spaces -------------------------------------------------------------------
 * An action is a real vector a of D dimensions, 1 <= D <= TB_MAX_CONTINUOUS_DIM, drawn from a diagonal Gaussian:
 *   policy row [.., A], A = 2D: columns [0, D) are the mean mu, columns [D, 2D) the log standard deviation l, taken as
 *     the head outputs it (no clamp, no squash), sigma = exp(l).  A Gaussian head is a policy layer of width 2D.
 *   rollout leaves: policy_logits keeps its name and holds the actor's (mu, l) rows [T+1,B,2D]; action and last_action
 *     are float32 [.., D].  The action is the unclipped sample: an actor clips it to the environment's bounds itself,
 *     before stepping the environment, and stores the unclipped value.
 * Per row, with z_k = (a_k - mu_k) * exp(-l_k) and c = TB_GAUSSIAN_HALF_LOG_2PI (0.5 log 2 pi, one fp32 constant),
 * each quantity is an fp32 sum over k in index order that starts from the k = 0 term:
 *   log pi(a) = sum_k (-0.5 z_k^2 - l_k - c);
 *   entropy term (the sign the flat loss uses for sum p log p): ent = sum_k -(l_k + 0.5 + c);
 *   trust-region KL(pi || mu_b) = sum_k ((lb_k - l_k) + 0.5 (exp(2 (l_k - lb_k)) + ((mu_k - mub_k) exp(-lb_k))^2) - 0.5);
 *   gradient of mu_k: -adv * z_k * exp(-l_k); gradient of l_k: adv * (1 - z_k^2) - entropy_cost; both multiplied by
 *     the column weight where the flat loss applies one.
 * A NaN or +-inf mu, l or action entry gives NaN for its row: log pi(a), the entropy term and the whole gradient row of a
 * row with one, and the KL of a pair of rows with one (the flat loss's "poison the row" convention).                */
#define TB_MAX_CONTINUOUS_DIM 64
#define TB_GAUSSIAN_HALF_LOG_2PI 0.918938533204672742f
/* tb_impala_loss_f32 on a Gaussian policy: the same arguments and outputs (hp block, column_weights, PopArt, trust
 * region, single-launch and split-T layouts), with actions float32 [T,B,D] and the rules above in place of the flat
 * row's.  A must be 2D with 1 <= D <= TB_MAX_CONTINUOUS_DIM (an odd A is rejected).  V-trace runs on
 * log rho = log pi(a) - log mu(a); the pg loss is -log pi(a) * pg_adv; target_alp / behavior_alp are the Gaussian
 * log-densities.  tb_upgo_loss_f32 and tb_kickstart_loss_f32 take categorical rows only.                            */
int tb_impala_loss_gaussian_f32(const float* behavior_logits, const float* target_logits, const float* actions,
                                const float* rewards, const uint8_t* done, const float* discounts, const float* values,
                                const float* bootstrap, int64_t T, int64_t B, int64_t A, float discounting,
                                float baseline_cost, float entropy_cost, int clip_rewards, float clip_rho,
                                float clip_pg_rho, const tb_hparams* hp, const float* column_weights,
                                const int64_t* task, const double* mu, const double* nu, int64_t K, double* task_sums,
                                const float* trust_beta, float* kl_out, float* trust_out, float* vs, float* pg_adv,
                                float* log_rhos, float* behavior_alp, float* target_alp, float* losses_out,
                                float* grad_logits, float* grad_values, int zero_tail, void* workspace, void* stream);
/* Seeded sampling of a Gaussian policy: rows [T,B,A = 2D] -> actions float32 [T,B,D].  Component k of row (t,b) takes
 * the Philox4x32-10 block with tb_sample_actions_f32's counter (step + t, stream id) and key (lo32(seed),
 * hi32(seed) + k/2) (mod 2^32), and its words x0, x1 = words 2 (k mod 2) and 2 (k mod 2) + 1.  Then
 *   u1 = ((x0 >> 8) + 1) * 2^-24 in (0, 1], u2 = (x1 >> 8) * 2^-24;
 *   z = sqrtf(-2 logf(u1)) * cospif(2 u2);  a_k = mu_k + expf(l_k) * z;
 * a non-finite mu_k or l_k gives NaN for a_k.  The greedy (eval-mode) action is mu.  seed_step (device, nullable) wins
 * over (seed, step), as in tb_sample_actions_factored_f32, so one entry serves eager and graphed acting.  Sizes:
 * T, B >= 0 (T*B == 0 is a no-op success), A = 2D as in the loss.                                                  */
int tb_sample_gaussian_f32(const float* logits, int64_t T, int64_t B, int64_t A, uint64_t seed, uint64_t step,
                           const uint64_t* seed_step, const int64_t* stream_ids, float* actions, void* stream);

/* ---- legal-action masks ("invalid action masking": the policy renormalised over each step's legal actions) ---------
 * A rollout may carry a leaf legal_actions bool / uint8 [T+1,B,A], nonzero = legal, indexed like frame: row t holds the
 * actions legal at frame t (an env output, stored beside the frame it came with).  Behaviour logits row t+1 and action
 * row t+1 were formed at frame t, so:
 *   - the learner's forward output row t is masked by legal_actions row t;
 *   - the behaviour logits policy_logits[1:] are masked by legal_actions[:-1];
 *   - action[1:] is checked against legal_actions[:-1].
 * An illegal logit becomes TB_MASKED_LOGIT = -FLT_MAX (torch.finfo(torch.float32).min), finite on purpose: expf of it
 * minus any realistic row maximum is exactly 0, so the loss, UPGO, kickstarting, trust-region and sampling kernels
 * above give p = 0, p * log p = -0 and a logit gradient of +-0 at an illegal entry, and the legal entries' sums keep
 * their bits (adding +0 changes no float sum).  What they compute is the softmax over the legal set.  -inf would make
 * 0 * (-inf) = NaN in the entropy, its gradient and the trust region's KL.                                         */
#define TB_MASKED_LOGIT (-3.40282346638528859812e+38F)
/* in, out [N,A] f32 (out == in allowed: in place); legal [N,A] u8, nonzero = legal; actions [N] i64 or NULL.  For each
 * row i:
 *   - no legal entry (some environments send an empty mask on terminal frames): out[i,:] = in[i,:], unmasked;
 *   - else, with actions given and 0 <= actions[i] < A and legal[i, actions[i]] == 0 (an illegal taken action, a
 *     caller bug the kernel cannot raise): out[i,:] = NaN.  On the target logits this makes the step's losses NaN, as
 *     an out-of-range action does in tb_impala_loss_f32 (on the behaviour logits alone it does not: the rho clips
 *     drop a NaN log-rho); an out-of-range action is left to the loss;
 *   - else out[i,a] = legal[i,a] ? in[i,a] : fill, bit for bit.
 * fill: TB_MASKED_LOGIT for logits; 0 for the gradient of the mask (d out / d in = legal on a masked row).  Sizes:
 * N >= 0 (0: a no-op success), A >= 1.  One launch, no host sync, no atomics; graph-capturable.                    */
int tb_mask_logits_f32(const float* in, float* out, const uint8_t* legal, const int64_t* actions, int64_t N, int64_t A,
                       float fill, void* stream);

/* ---- experience replay: a device ring of earlier batch columns mixed into the learner batch --------------------------
 * A replay buffer is a device ring of `capacity` batch columns.  A stored column holds every learner leaf of one rollout
 * column (frame, stacked [T+1,...] or unstacked [T+4,...]; reward, done, policy_logits, action, and last_action,
 * episode_return, task and legal_actions when present) and, for a net with an LSTM, its initial agent state (h, c: [layers, H] each).
 * Each of these is one leaf of the table below: the fresh batch holds it as [outer, Bf, row], the ring as
 * [capacity, outer, row] (one slot's rows contiguous), the mixed batch as [outer, Bf+R, row]; the agent state has
 * outer = layers.  Device state: head_size = (head: the next slot to write, size: the number of valid slots) and
 * seed_step = (seed, step); slot (head - 1 - k) mod capacity is the k-th newest column.
 *
 * One tb_replay_mix call with Bf fresh columns and R replayed columns, read against the device state when it runs:
 *   1. n = min(size, capacity - Bf) survivors: the newest columns this call's insert leaves in place.  Replayed column
 *      j in [0,R) takes x = word 0 of Philox4x32-10 with counter (lo32(step), hi32(step), j, stream_id) and key
 *      (lo32(seed), hi32(seed)), k = (uint64(x) * n) >> 32, slot = (head - 1 - k) mod capacity.  Draws are with
 *      replacement, and no slot drawn is one of the Bf slots this call writes, so the gather and the insert never race.
 *      The caller guarantees n >= 1 when R > 0 (with n = 0 every draw names slot head - 1, whose contents are undefined).
 *   2. out columns [0,Bf) = the fresh columns; columns [Bf,Bf+R) = the drawn slots, for every leaf whose out != NULL.
 *   3. the fresh columns are written to slots head, head+1, ... (mod capacity).
 *   4. slots_out[j] (int64 [R], nullable) = the slot of replayed column j.
 * tb_replay_advance, the next launch on the stream, then sets head = (head + Bf) mod capacity,
 * size = min(size + Bf, capacity), step = step + 1.  R = 0 inserts only.  Both read their state from device memory when
 * they run, so a launch pair captured in a CUDA graph draws new slots on every replay.  Copies are exact byte copies.
 * Sizes: 1 <= num_leaves <= TB_REPLAY_MAX_LEAVES, 0 <= R <= TB_REPLAY_MAX_R, Bf >= 1, capacity > Bf,
 * 0 <= stream_id < 2^32, outer >= 1 and row_bytes >= 1 per leaf; fresh and ring must not be NULL.
 * Algorithmic bytes of one call: sum over leaves of outer * row_bytes * (3*Bf + 2*R).                              */
#define TB_REPLAY_MAX_LEAVES 16
#define TB_REPLAY_MAX_R 4096
typedef struct tb_replay_leaf {
  const void* fresh; /* [outer, Bf, row_bytes] */
  void* out;         /* [outer, Bf+R, row_bytes], or NULL: this leaf is inserted only */
  void* ring;        /* [capacity, outer, row_bytes] */
  int64_t outer;
  int64_t row_bytes;
} tb_replay_leaf;
/* leaves_host: a host array of num_leaves entries, read before the call returns (the kernel gets it by value). */
int tb_replay_mix(const tb_replay_leaf* leaves_host, int num_leaves, int64_t Bf, int64_t R, int64_t capacity,
                  const uint64_t* seed_step, const int64_t* head_size, int64_t stream_id, int64_t* slots_out,
                  void* stream);
/* One-thread launch: the state advance of one tb_replay_mix call with Bf fresh columns. */
int tb_replay_advance(int64_t* head_size, uint64_t* seed_step, int64_t Bf, int64_t capacity, void* stream);
/* tb_replay_mix with the R replayed slots read from slots (int64 [R], device) instead of drawn: steps 2 and 3 above,
 * with slot j = slots[j]; seed_step is not read.  The caller guarantees every slot is a survivor (tb_replay_sample_
 * prioritized writes such slots).  Same sizes and validation as tb_replay_mix; stream id 0.                          */
int tb_replay_mix_slots(const tb_replay_leaf* leaves_host, int num_leaves, int64_t Bf, int64_t R, int64_t capacity,
                        const int64_t* slots, const int64_t* head_size, void* stream);

/* ---- prioritised replay (Schaul et al. 2016; sequence priorities as in R2D2, Kapturowski et al. 2019) -----------------
 * A prioritised buffer adds, on the device: priorities f32 [capacity], one value per slot (>= 0; never-written slots
 * are never drawn), and prio f64 [4] = {alpha, beta, eta, eps} (alpha >= 0, 0 <= beta <= 1, 0 <= eta <= 1, eps > 0),
 * read when the kernels run, so a captured graph follows the values published between replays.
 *
 * tb_replay_sample_prioritized, before tb_replay_mix_slots and tb_replay_advance, reads head_size, seed_step, prio and
 * priorities and writes batch_slots (int64 [Bf+R]) and column_weights (f32 [Bf+R]):
 *   Fresh column c: batch_slots[c] = (head + c) mod capacity, column_weights[c] = 1.  R = 0 writes these only.
 *   Survivors as for tb_replay_mix: n = min(size, capacity - Bf), survivor k is slot (head - 1 - k) mod capacity; the
 *   caller guarantees n >= 1 when R > 0.  q_k = pow((double)priorities[slot_k] + eps, alpha) in double.
 *   Summation order (every + below a double add, rounded to nearest):
 *     L = ceil(n / 1024); chunk i in [0, 1024) holds k in [i*L, min(i*L + L, n)) (possibly empty).
 *     r_k = the running sum of q over chunk i up to k, in k order, from 0; T_i = its total (0 if empty).
 *     Warp g in [0, 32) holds chunks 32g .. 32g+31.  P_i = the sum of T over the chunks of i's warp before i, in
 *     order, from 0; G_g = the sum of all 32 T of warp g, in order, from 0; B_g = G_0 + ... + G_{g-1}, in order, from 0.
 *     C_k = B_g + (P_i + r_k) for k in chunk i of warp g;  S = C_{n-1}.  C is non-decreasing.
 *   Replayed column j in [0, R): (w0, w1) = words 0 and 1 of Philox4x32-10 with the counter and key of tb_replay_mix
 *   (counter (lo32(step), hi32(step), j, stream_id), key (lo32(seed), hi32(seed))); u = ((w1 << 32 | w0) >> 11) * 2^-53;
 *   k_j = the smallest k with C_k > u * S (the product rounded to double), or n - 1 if there is none.
 *   batch_slots[Bf + j] = slot_{k_j}; column_weights[Bf + j] = (float)pow(q_min / q_{k_j}, beta) with q_min the
 *   minimum of q over the survivors: (n P)^-beta normalised by its largest value over the buffer, in (0, 1].
 *   Draws are with replacement and never name a slot the call overwrites.  One CTA; no atomics, so the results are
 *   bit-identical from run to run.  Host validation as tb_replay_mix (null pointers, R, Bf, capacity, stream_id).
 *
 * tb_replay_update_priorities, after the loss, on the batch the loss used (vs, values [T, B] f32, B = Bf + R):
 *   e_t = |(double)vs[t,c] - (double)values[t,c]|; p_c = eta * max_t e_t + (1 - eta) * (sum_t e_t / T), the sum in t
 *   order, every operation rounded to double (no fused multiply-add); stored as (float)p_c, or 0 if that is not finite.
 *   Column c writes priorities[batch_slots[c]] unless a later column c' > c names the same slot: of a slot drawn
 *   more than once, the largest j wins.  Slots not in batch_slots are untouched.  One launch, deterministic.        */
int tb_replay_sample_prioritized(const float* priorities, const double* prio, const int64_t* head_size,
                                 const uint64_t* seed_step, int64_t Bf, int64_t R, int64_t capacity, int64_t stream_id,
                                 int64_t* batch_slots, float* column_weights, void* stream);
int tb_replay_update_priorities(const float* vs, const float* values, int64_t T, int64_t B, const int64_t* batch_slots,
                                const double* prio, float* priorities, void* stream);

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

/* ---- AtariNet (monobeast.py:545-635) forward / backward ---------------------------------
 * Parameters live in ONE flat f32 buffer in the reference's state_dict order and shapes
 * (BASELINE.md section 5): conv1.weight (32,4,8,8), conv1.bias, conv2.weight (64,32,4,4), conv2.bias,
 * conv3.weight (64,64,3,3), conv3.bias, fc.weight (512,3136), fc.bias, [core.weight_ih_l0,
 * core.weight_hh_l0, core.bias_ih_l0, core.bias_hh_l0, ...l1 (2076 x 519 each)], policy.weight (A,519),
 * policy.bias, baseline.weight (num_values,519), baseline.bias (num_values).  num_values (1..64) is the number of value
 * outputs, one per PopArt task; 1 is the reference's net.  Gradients use the same layout.
 * tb_atarinet_workspace_bytes: bytes of caller-owned workspace for a [T1,B] rollout (T1 = unroll_length + 1): patch
 * matrices, activations kept for backward, packed weights, split-K scratch.  Neither it nor tb_atarinet_grad_split
 * depends on num_values.
 *
 * tb_atarinet_forward: monobeast.py:582-632 AtariNet.forward (without the action sampling, which the learner never
 * uses - SURVEY.md K8).  reward f32 [T1,B]; last_action i64 [T1,B]; notdone f32 [T1,B] = (~done).float() (LSTM only;
 * multiplies the state before each step, monobeast.py:607-609); h0,c0 / hN,cN f32 [2,B,519] (LSTM only).
 * -> policy_logits f32 [T1,B,A], baseline f32 [T1,B,num_values].  Activations stay in `workspace`.
 *   done == NULL: frame is the stacked u8 [T1,B,4,84,84]; stacked_scratch is not read.
 *   done != NULL: frame is an unstacked rollout u8 [T1+3,B,84,84] with done [T1,B] (see "unstacked rollouts" below),
 *     and stacked_scratch is device memory of tb_unstacked_scratch_bytes(0, T1, B, precision) bytes (NULL allowed, and
 *     not touched, when that is 0).  Outputs and workspace contents are bit-identical to the stacked forward on the
 *     restacked frames.
 * precision: 0 = fp32 SIMT GEMMs (bit-comparable with the reference's fp32 CPU arithmetic);
 *            1 = bf16 operands with fp32 accumulation: conv/fc trunk (implicit-GEMM convolutions) and LSTM
 *                projections on wgmma tensor cores, LSTM recurrence products as bf16 mma.sync; LSTM state and
 *                gate math, heads, losses, optimizer, master weights and gradients stay fp32;
 *            2 = split-bf16 (hi + lo planes) tensor-core products over fp32 activations.
 *
 * tb_atarinet_backward: the backward of the forward that last ran on `workspace` with the same parameters (replaces
 * the autograd graph of total_loss.backward(), monobeast.py:290): grad_logits [T1,B,A], grad_baseline
 * [T1,B,num_values] -> grads (flat, parameter layout, overwritten).  It reads only the workspace, never the frames.
 *   phase 3: the whole backward.
 *   phase 1, then phase 2: the same backward in two calls, for data-parallel learners (the reference has a single
 *     learner device, polybeast_learner.py:402-405; SURVEY 8(e) G1 "bucket order = reverse of forward"): phase 1 =
 *     policy/baseline heads + LSTM, phase 2 = conv/fc trunk.  After phase 2 everything is final; after phase 1 the slice
 *     [tb_atarinet_grad_split(), param_count) of `grads` (LSTM + heads: 17 of 24 MB) is final when the LSTM
 *     weight-gradient GEMMs ran on the caller's stream; when they were forked onto the side stream (tensor-core
 *     backends), the slice is final in STREAM ORDER on that side stream: pass your own with tb_set_aux_stream()
 *     (thread-local; NULL = library-owned) before phase 1, make it wait for `stream`, and enqueue the slice's
 *     all-reduce on it - it then overlaps phase 2.
 *   Any other phase is rejected.                                                                                      */
int64_t tb_atarinet_param_count(int num_actions, int num_values, int use_lstm);
size_t tb_atarinet_workspace_bytes(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision);
int64_t tb_atarinet_grad_split(int num_actions, int use_lstm);
int tb_set_aux_stream(void* stream);
int tb_atarinet_forward(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                        const int64_t* last_action, const float* h0, const float* c0, const float* params,
                        int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                        void* workspace, void* stacked_scratch, float* policy_logits, float* baseline,
                        float* hN, float* cN, void* stream);
/* tb_atarinet_forward of a net with a factored action space (num_actions = sum dims, see "multi-discrete (factored)
 * action spaces"): last_action is int64 [T1,B,D], and the core input takes a K-hot, core[n, 512+1+off_k+a_k] = 1 for
 * each k (a component outside [0, A_k) sets nothing), in place of the one-hot.  Everything else is tb_atarinet_forward;
 * the K-hot gets no gradient, so tb_atarinet_backward is its backward.                                             */
int tb_atarinet_forward_factored(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                                 const int64_t* last_action, const float* h0, const float* c0, const float* params,
                                 int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                                 void* workspace, void* stacked_scratch, float* policy_logits, float* baseline,
                                 float* hN, float* cN, const tb_action_space* space, void* stream);
int tb_atarinet_backward(const float* grad_logits, const float* grad_baseline, const float* notdone,
                         const float* params, int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm,
                         int precision, void* workspace, float* grads, int phase, void* stream);
/* AtariNet with a continuous action space (see "continuous (diagonal-Gaussian) action spaces"): num_actions = 2D is the
 * policy layer's width, and the core input is 512 + D + 1 wide, F = 512 + D + 1 in place of 519 above: column 512 holds
 * the clipped reward and columns 513 .. 512 + D hold last_action[n, k] (float32 [T1,B,D]) as it is.  The parameters are
 * the layout above with that F (the LSTM 4F x F, policy.weight (2D, F)), counted by tb_atarinet_param_count_continuous;
 * the workspace is tb_atarinet_workspace_bytes_continuous bytes; tb_atarinet_grad_split holds unchanged.  The forward
 * and the backward are tb_atarinet_forward / tb_atarinet_backward on that layout; last_action gets no gradient.  An odd
 * num_actions, or D > TB_MAX_CONTINUOUS_DIM, is rejected; the heads take at most 31 outputs, so D <= 15 here.        */
int64_t tb_atarinet_param_count_continuous(int num_actions, int num_values, int use_lstm);
size_t tb_atarinet_workspace_bytes_continuous(int64_t T1, int64_t B, int num_actions, int use_lstm, int precision);
int tb_atarinet_forward_continuous(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                                   const float* last_action, const float* h0, const float* c0, const float* params,
                                   int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                                   void* workspace, void* stacked_scratch, float* policy_logits, float* baseline,
                                   float* hN, float* cN, void* stream);
int tb_atarinet_backward_continuous(const float* grad_logits, const float* grad_baseline, const float* notdone,
                                    const float* params, int64_t T1, int64_t B, int num_actions, int num_values,
                                    int use_lstm, int precision, void* workspace, float* grads, int phase, void* stream);

/* ---- MLPNet: vector observations -------------------------------------------------------------------------------
 * AtariNet with its conv trunk and fc replaced by dense layers, for float32 observation vectors of O features:
 *   x = obs [T1*B, O];  with normalisation x = clamp((x - mean) * inv_std, -10, 10) (below);
 *   x = relu(x W_i^T + b_i) for i = 0 .. L-1, W_i [H_i, H_{i-1}] (H_{-1} = O);
 *   core_in = cat[x, clamp(reward, -1, 1), last-action encoding] of width F = H_{L-1} + 1 + E;
 *   [2-layer LSTM of width F with done-reset]; policy [A, F] / baseline [num_values, F] heads.
 * The last-action encoding is AtariNet's: one-hot over A (E = A, last_action int64 [T1,B]) with space == NULL and
 * continuous_dim == 0; a K-hot (E = A, last_action int64 [T1,B,D]) with a factored space (tb_action_space, see
 * "multi-discrete (factored) action spaces"); the raw values (E = D, last_action float32 [T1,B,D]) with continuous_dim
 * = D > 0 and num_actions = 2D (see "continuous (diagonal-Gaussian) action spaces").  Giving both is rejected.
 * Limits: 1 <= O <= TB_MLP_MAX_OBS; 1 to TB_MLP_MAX_LAYERS hidden widths, each a multiple of 8 in [8, TB_MLP_MAX_WIDTH]
 * (the row stride rule of the bf16 operands); 1 <= A <= 31 (the heads); with the LSTM F <= TB_LSTM_MAX_HIDDEN.
 * Parameters, in one flat fp32 buffer in this order: W_0, b_0, ..., W_{L-1}, b_{L-1}, then AtariNet's LSTM (with F),
 * policy and baseline layout; tb_mlpnet_param_count counts them (-1: a rejected config).
 *
 * Observation normalisation (cfg->normalize != 0): obs_mean / obs_var are float64 [O].  The staged operand is, in fp32,
 *   mean_f[j] = (float)obs_mean[j];  inv_std_f[j] = (float)(1.0 / sqrt(obs_var[j] + 1e-8))   (both formed in float64),
 *   y = (x - mean_f[j]) * inv_std_f[j]  (two fp32 roundings, no FMA);  y < -10 ? -10 : (y > 10 ? 10 : y)
 * so a NaN observation stays NaN.  The clip of 10 and the eps of 1e-8 are fixed (VecNormalize's defaults).  Without
 * normalisation y = x.  precision 0 stages y as fp32 [N, O]; 1 and 2 as bf16 [N, ld] with ld = O rounded up to a
 * multiple of 8 and columns [O, ld) zero: hi = bf16_rn(y), and at precision 2 the lo plane bf16_rn(y - hi) follows at
 * N * ld elements.  tb_obs_stage runs that staging alone into `out`.
 *
 * tb_mlpnet_forward / tb_mlpnet_backward: the contract of tb_atarinet_forward / tb_atarinet_backward (phase 3) with
 * float32 observations in place of the frames: reward, notdone, h0/c0/hN/cN [2,B,F] and the outputs as there;
 * precision 0 = fp32 SIMT GEMMs, 1 = bf16, 2 = split-bf16 tensor-core GEMMs.  The backward reads only the workspace
 * the forward left (tb_mlpnet_workspace_bytes bytes, 0: a rejected config) and overwrites grads; the observations and
 * the statistics get no gradient.                                                                                    */
#define TB_MLP_MAX_OBS 4096
#define TB_MLP_MAX_LAYERS 4
#define TB_MLP_MAX_WIDTH 512
#define TB_OBS_NORM_EPS 1e-8
#define TB_OBS_NORM_CLIP 10.0f
typedef struct tb_mlp_config {
  int obs_dim;                     /* O */
  int num_layers;                  /* L */
  int hidden[TB_MLP_MAX_LAYERS];   /* H_0 .. H_{L-1}; later entries are not read */
  int num_actions;                 /* A: the policy width (2D for a continuous space) */
  int num_values;                  /* value outputs (PopArt tasks), 1 .. 64 */
  int use_lstm;
  int normalize;                   /* stage the observations normalised by obs_mean / obs_var */
} tb_mlp_config;
int64_t tb_mlpnet_param_count(const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim);
size_t tb_mlpnet_workspace_bytes(const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim, int64_t T1,
                                 int64_t B, int precision);
int tb_mlpnet_forward(const float* obs, const float* reward, const float* notdone, const void* last_action,
                      const float* h0, const float* c0, const float* params, const double* obs_mean,
                      const double* obs_var, const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim,
                      int64_t T1, int64_t B, int precision, void* workspace, float* policy_logits, float* baseline,
                      float* hN, float* cN, void* stream);
int tb_mlpnet_backward(const float* grad_logits, const float* grad_baseline, const float* notdone, const float* params,
                       const tb_mlp_config* cfg, const tb_action_space* space, int continuous_dim, int64_t T1,
                       int64_t B, int precision, void* workspace, float* grads, void* stream);
int tb_obs_stage(const float* obs, int64_t N, int O, const double* obs_mean, const double* obs_var, int precision,
                 void* out, void* stream);
/* Running observation statistics, per feature j (count, mean, var: float64 [O], initially 0, 0 and 1).
 * tb_obs_norm_sums: sums [3, O] float64 = {number of finite entries, sum x, sum x^2} of feature j over the rows (t, b)
 *   with t_begin <= t < T1 and b < Bf of obs [T1, B, O]; non-finite entries are skipped.  A fixed summation order and
 *   no atomics: bit-identical from run to run.
 * tb_obs_norm_update: merges sums into the statistics (parallel variance).  With n_b = sums[0][j] > 0:
 *   m_b = S / n_b;  v_b = max(S2 / n_b - m_b^2, 0);  tot = count + n_b;  d = m_b - mean;
 *   mean' = mean + d * n_b / tot;  var' = (var * count + v_b * n_b + d^2 * count * n_b / tot) / tot;  count' = tot;
 *   a feature with n_b = 0 is unchanged.  So the first update takes the batch's own mean and variance.
 * One launch each, no host synchronisation: both can be captured in a CUDA graph.                                    */
int tb_obs_norm_sums(const float* obs, int64_t T1, int64_t B, int O, int64_t t_begin, int64_t Bf, double* sums,
                     void* stream);
int tb_obs_norm_update(const double* sums, double* count, double* mean, double* var, int O, void* stream);

/* ---- stacked LSTM over the unroll with per-step done-reset -------------------------------------------
 * Replaces the reference's loop of seq_len-1 nn.LSTM calls and its autograd graph (monobeast.py:603-611,
 * polybeast_learner.py:241-249):   for t: state *= notdone_t;  y_t, state = LSTM(x_t, state).
 * torch.nn.LSTM conventions: params[4*l + {0,1,2,3}] = weight_ih_l [4H, In|H], weight_hh_l [4H, H], bias_ih_l [4H],
 * bias_hh_l [4H] (gate order i, f, g, o); any number of layers >= 1; input size, batch and unroll are free, hidden size is
 * 1 .. TB_LSTM_MAX_HIDDEN (BASELINE configs[4]: T = 600, B = 128, H = 512).  Above that bound the backward's fp32 step kernel,
 * which every precision falls back to, cannot hold a row of H in shared memory: every tb_lstm_* entry rejects such an H
 * (tb_lstm_workspace_bytes returns 0).  x [T1*B, In], notdone [T1*B] (float 0/1), h0/c0/hN/cN [layers, B, H],
 * y [T1*B, H].  precision 0 = fp32 everywhere (any shape); 1 / 2 = bf16 / split-bf16 tensor-core products for the hoisted
 * projections, and in the recurrence where a tensor-core recurrence fits the shape (tb_lstm_plan).  tb_lstm_backward must
 * follow tb_lstm_forward on the same workspace; grads[] mirrors params[] and is overwritten; dx [T1*B, In].
 * A stack runs as a chain of segments of two layers (layers 2k and 2k+1; the top segment is one layer when the depth is
 * odd), each planned as a stack of its own with input width In for the first segment and H above it, so every upper
 * pair can take a two-layer wavefront.  Every notdone step resets all layers.  Above two layers the workspace also holds
 * each segment's output but the top one's and two [T1*B, H] buffers for the gradient handed between segments.        */
#define TB_LSTM_MAX_HIDDEN 700
size_t tb_lstm_workspace_bytes(int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision);
/* The recurrence kinds tb_lstm_forward (*fwd_kind_host) and tb_lstm_backward (*bwd_kind_host) run for this shape on the
 * current device; host query, runs no kernel.  The choice does not depend on the unroll length.  1 or 2 layers
 * (one segment); tb_lstm_plan_layers reports any depth.                                                               */
#define TB_LSTM_STEP 0            /* one step kernel per time step (any shape) */
#define TB_LSTM_PERSISTENT 1      /* one cooperative fp32 kernel per layer */
#define TB_LSTM_PERSISTENT_MMA 2  /* one cooperative kernel per layer, bf16 tensor-core products (precision 1) */
#define TB_LSTM_CLUSTER 3         /* one 16-CTA thread-block cluster per layer, split-bf16 products (precision 2, H = 256) */
#define TB_LSTM_WAVE_BF16 4       /* both layers in one wavefront kernel, bf16 products (precision 1) */
#define TB_LSTM_WAVE_SPLIT 5      /* both layers in one wavefront kernel, split-bf16 products (precision 2) */
int tb_lstm_plan(int64_t B, int input_size, int hidden_size, int layers, int precision, int* fwd_kind_host,
                 int* bwd_kind_host);
/* Per layer, for any depth: fwd_kinds_host[l] / bwd_kinds_host[l] (each an array of `layers` ints) get the kinds of the
 * segment that runs layer l; both layers of a wavefront segment report its kind.  Host query, runs no kernel.          */
int tb_lstm_plan_layers(int64_t B, int input_size, int hidden_size, int layers, int precision, int* fwd_kinds_host,
                        int* bwd_kinds_host);
int tb_lstm_forward(const float* x, const float* notdone, const float* h0, const float* c0, const float* const* params,
                    int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision, void* workspace,
                    float* y, float* hN, float* cN, void* stream);
int tb_lstm_backward(const float* dy, const float* x, const float* notdone, const float* const* params, float* const* grads,
                     int64_t T1, int64_t B, int input_size, int hidden_size, int layers, int precision, void* workspace,
                     float* dx, void* stream);
/* tb_lstm_backward with the gradients at both ends of the recurrence, each [layers, B, H] and each optional (NULL):
 *   dhN, dcN (in):  dL/dhN and dL/dcN, the gradients arriving at the final state the forward returned (a loss on hN / cN,
 *                   or the next unroll of a truncated-BPTT chain);
 *   dh0, dc0 (out): dL/dh0 and dL/dc0 with respect to the h0 / c0 the forward was given.  Step 0 applies
 *                   state *= notdone_0 first, so both include that mask: a column with notdone_0 = 0 gets exact zeros.
 * dy stays read-only.  With all four NULL this is tb_lstm_backward: the same kernels and bit-identical outputs.       */
int tb_lstm_backward_state(const float* dy, const float* x, const float* notdone, const float* const* params,
                           float* const* grads, int64_t T1, int64_t B, int input_size, int hidden_size, int layers,
                           int precision, void* workspace, float* dx, const float* dhN, const float* dcN, float* dh0,
                           float* dc0, void* stream);

/* ---- IMPALA ResNet (polybeast_learner.py:134-266 `Net`) forward / backward -------------------------
 * Observations u8 [C, H, W] and section widths (ch0, ch1, ch2); the reference's net is (4, 84, 84) with (16, 32, 32).
 * Section i (width ch_i) runs its feat conv at H_i x W_i (H_0 = H, W_0 = W); its max-pool (3, 2, 1) leaves
 * ceil(H_i / 2) x ceil(W_i / 2) = H_{i+1} x W_{i+1}.  Flat parameter layout = the reference's state_dict order:
 *   feat_convs.0.0.weight (ch0, C, 3, 3), feat_convs.{1,2}.0.weight (ch_i, ch_{i-1}, 3, 3), feat_convs.i.0.bias (ch_i),
 *   resnet1.i.{1,3}.{weight (ch_i, ch_i, 3, 3), bias (ch_i)}, resnet2.i.{1,3}.{weight, bias},
 *   fc.{weight (256, ch2 * H_3 * W_3), bias (256)}, [core.weight_ih_l0 (1024,257), core.weight_hh_l0 (1024,256),
 *   core.bias_ih_l0, core.bias_hh_l0], policy.{weight (A,257|256), bias}, baseline.{weight (num_values,257|256),
 *   bias (num_values)}.
 * At (4, 84, 84) x (16, 32, 32): (16,4,3,3) (32,16,3,3) (32,32,3,3) and fc.weight (256,3872).  num_values (1..64) is
 * the number of value outputs, one per PopArt task.  Gradients use the same layout.
 * Supported on every precision: 1 <= C <= 16, 17 <= H <= 126 and 33 <= W <= 126 (17 rows are the fewest that leave the
 * last section 3 high, the smallest image of the split-bf16 conv kernels; 33 columns the fewest that leave it 5 wide,
 * the narrowest row their weight gradient takes; 126 their widest padded row, 128 pixels), each width 16, 32 or 64 in
 * any combination (e.g. (32, 64, 64) is the "IMPALA x2" net).  tb_resnet_obs_range writes the shape bounds as
 * {C min, C max, H min, H max, W min, W max}, tb_resnet_widths writes {16, 32, 64}.  tb_resnet_supported returns 1 for
 * a supported (shape, widths, precision) and otherwise 0 with tb_last_error set; the other entries fail the same way
 * (param count -1, workspace 0, forward / backward non-zero).
 *
 * tb_resnet_forward: polybeast_learner.py:214-266 Net.forward without the action sampling: reward f32 [T1,B], notdone
 * f32 [T1,B] and h0,c0/hN,cN f32 [1,B,256] (LSTM only) -> policy_logits [T1,B,A], baseline [T1,B,num_values].
 *   done == NULL: frame is the stacked u8 [T1,B,C,H,W]; stacked_scratch is not read.
 *   done != NULL: frame is an unstacked rollout u8 [T1+3,B,84,84] with done [T1,B] (see "unstacked rollouts" below);
 *     only (4, 84, 84) with widths (16, 32, 32).  stacked_scratch is device memory of
 *     tb_unstacked_scratch_bytes(1, T1, B, precision) bytes (NULL allowed, and not touched, when that is 0); at
 *     precision 0 / 1 the forward restacks the frames into it.  Outputs, workspace contents and gradients are
 *     bit-identical to the stacked forward on the restacked frames.
 * precision: 0 = fp32 SIMT patch-matrix GEMMs; 1 = bf16 activations + patch-matrix wgmma GEMMs (not parity-grade);
 * 2 = split-bf16 (the Python default): fp32 activations, every 3x3 conv as a shifted-window implicit GEMM over padded
 * channel-chunk-planar hi/lo images (csrc/conv3x3_sw.cu), the H=256 LSTM on one thread-block cluster.  T1*B < 65536.
 * The same precision, shape, widths and workspace must be used for forward and backward.
 *
 * tb_resnet_backward: the backward of the forward pass that last ran on `workspace` (it keeps the conv input images /
 * activations it needs).  grad_logits [T1,B,A], grad_baseline [T1,B,num_values] -> grads (flat, overwritten).  frame
 * is what that forward's first conv read: the stacked frame after a stacked forward, stacked_scratch (still holding
 * the restacked frames) after an unstacked one.  At precision 2 it is not read (the first conv's input image is in the
 * workspace) and may be NULL.                                                                                         */
int tb_resnet_obs_range(int* range);
int tb_resnet_widths(int* widths);
int tb_resnet_supported(int C, int H, int W, int ch0, int ch1, int ch2, int precision);
int64_t tb_resnet_param_count(int C, int H, int W, int ch0, int ch1, int ch2, int num_actions, int num_values,
                              int use_lstm);
size_t tb_resnet_workspace_bytes(int C, int H, int W, int ch0, int ch1, int ch2, int64_t T1, int64_t B,
                                 int num_actions, int use_lstm, int precision);
int tb_resnet_forward(const uint8_t* frame, const uint8_t* done, const float* reward, const float* notdone,
                      const float* h0, const float* c0, const float* params, int C, int H, int W, int ch0, int ch1,
                      int ch2, int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                      void* workspace, void* stacked_scratch, float* policy_logits, float* baseline, float* hN,
                      float* cN, void* stream);
int tb_resnet_backward(const uint8_t* frame, const float* grad_logits, const float* grad_baseline,
                       const float* notdone, const float* params, int C, int H, int W, int ch0, int ch1, int ch2,
                       int64_t T1, int64_t B, int num_actions, int num_values, int use_lstm, int precision,
                       void* workspace, float* grads, void* stream);

/* ---- unstacked rollouts: four-frame stacks rebuilt on the GPU ------------------------------------------------------
 * Each frame sits in four consecutive stacks, so a stacked `frame` leaf u8 [T1,B,4,84,84] is three quarters copies.  An
 * unstacked rollout of T1 = T+1 steps carries the same information as frames u8 [T1+3, B, HW] (HW = 84*84), contiguous:
 *   rows 0..2 = channels 0..2 (oldest first) of step 0's stack;  row 3+t = the newest channel of step t's stack;
 * with done [T1,B] bool or uint8, any non-zero value marking the first step of an episode (the environment reports
 * done = 1 on an episode's first frame, and FrameStack.reset fills all four channels with it).  Channel c (0..3) of step t's
 * stack in column b is
 *   stack[t,b,c] = frames[3 + max(t - 3 + c, last_done(t,b)), b],
 *   last_done(t,b) = the largest s in [0,t] with done[s,b] != 0, or -3 if there is none.
 * An actor writes its current stack's four channels into rows 0..3 at the start of a rollout, then one newest frame per
 * step; row 0 of a rollout repeats the previous rollout's last step, as for stacked leaves.  The LSTM's notdone
 * ((~done).float(), a bitwise NOT for uint8) is unaffected: only the restack reads done as "non-zero".             */

/* stacked_out u8 [T1,B,4,HW] = the stacks of frames u8 [T1+3,B,HW] / done [T1,B] (u8 or bool bytes).  HW % 16 == 0;
 * frames and stacked_out 16-byte aligned.  One bandwidth-bound launch.                                               */
int tb_restack_frames_u8(const uint8_t* frames, const uint8_t* done, int64_t T1, int64_t B, int64_t HW, uint8_t* stacked_out,
                         void* stream);
/* Acting on newest frames: a device-resident frame history per actor stream builds rows 0..2 of the unstacked array.
 * history u8 [S,3,HW] (caller-owned; a new one is all zeros) holds for stream s, oldest first, channels 1..3 of the
 * stack of the last step this entry ran for s: channels 0..2 of its next stack unless that step starts an episode.
 * frames u8 [T+3,B,HW] has the newest frames already in rows 3..T+2; done [T,B] (u8 or bool bytes, non-zero = the step
 * starts an episode).  For each column b with s = stream_ids[b] in [0,S), rows 0..2 := history[s], then history[s] :=
 * channels 1..3 of step T-1's stack (the rule above), so T = 1 with done set makes all three the new frame, as
 * FrameStack.reset does.  A column whose id is < 0 or >= S gets zero rows 0..2, and no history is read or written for
 * it (graph padding uses -1).  The ids of one call must be distinct: this is not checked, and two columns naming one
 * stream race.  Calls that share a history must be ordered on one stream.  HW % 16 == 0; frames and history 16-byte
 * aligned.  One launch; the output feeds tb_atarinet_forward / tb_resnet_forward (done != NULL) with T1 = T.          */
int tb_frame_history_fill_u8(uint8_t* frames, const uint8_t* done, const int64_t* stream_ids, int64_t T, int64_t B,
                             int64_t HW, uint8_t* history, int64_t S, void* stream);
/* Bytes of stacked_scratch the forwards need with done != NULL, for net (0 = AtariNet, 1 = ResNet) at this precision:
 * 0 where the restack is fused into the backend's frame-image pass (AtariNet bf16 / bf16x3, ResNet bf16x3),
 * T1*B*4*84*84 where the backend reads stacked frames (AtariNet fp32, ResNet fp32 / bf16).  SIZE_MAX for an unknown net,
 * precision or a size < 1.                                                                                           */
size_t tb_unstacked_scratch_bytes(int net, int64_t T1, int64_t B, int precision);

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
 *   coef = min(1, max_norm/(sqrt(sumsq)+1e-6)), NaN when sumsq is NaN as torch.clamp gives it (max_norm < 0: no
 *   clipping); grads *= coef (left clipped in place like the reference); square_avg = alpha*square_avg + (1-alpha)*g^2;
 *   params -= lr * g/(sqrt(square_avg)+eps)   (momentum != 0: buf = momentum*buf + g/avg; params -= lr*buf).
 * lr_device (nullable) overrides `lr` with a device scalar; grad_norm_out (nullable) receives the
 * pre-clip norm.  No host synchronisation.
 * hp, in this and the two steps below: NULL takes max_norm and the optimizer's values from the arguments.  Non-NULL:
 * they are read from hp (device pointer, see tb_hparams) when the kernel runs, and the scalar arguments are not read;
 * lr_device / lr as above.  The host cannot see hp's values, so the caller checks what the NULL case checks:
 * momentum != 0 needs momentum_buf, betas in [0, 1).  With hp, momentum_buf != NULL selects the momentum update, so
 * pass NULL when momentum is 0 (with hp NULL the buffer is ignored when momentum is 0).                          */
int tb_clip_rmsprop_step_f32(float* params, float* grads, float* square_avg, float* momentum_buf, int64_t n,
                             const float* sumsq, float max_norm, const float* lr_device, float lr, float alpha,
                             float eps, float momentum, const tb_hparams* hp, float* grad_norm_out, void* stream);
/* The same clip fused with one torch.optim.Adam (decoupled = 0, L2 weight decay) or AdamW (decoupled = 1) step,
 * non-amsgrad, in torch's op order:  g *= coef (written back);  Adam: g' = g + wd*p,  AdamW: p *= 1 - lr*wd;
 *   exp_avg = beta1*exp_avg + (1-beta1)*g';  exp_avg_sq = beta2*exp_avg_sq + (1-beta2)*g'^2;
 *   p -= lr/(1-beta1^t) * exp_avg / (sqrt(exp_avg_sq)/sqrt(1-beta2^t) + eps).
 * step_device is a device int64 holding the number of completed steps: t = step_device[0] + 1, and the call
 * increments it on the stream after the update (a second, one-thread launch).  No host read, so the call can be
 * captured into a CUDA graph and every replay takes the next t.  Bias corrections are computed in double.    */
int tb_clip_adam_step_f32(float* params, float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, const float* sumsq,
                          float max_norm, const float* lr_device, float lr, double beta1, double beta2, float eps,
                          float weight_decay, int decoupled, int64_t* step_device, const tb_hparams* hp,
                          float* grad_norm_out, void* stream);
/* The same clip fused with torch.optim.RMSprop's remaining options: weight_decay (g' = g + wd*p after the clip) and
 * centered (grad_avg != NULL: grad_avg = alpha*grad_avg + (1-alpha)*g', avg = sqrt(square_avg - grad_avg^2) + eps),
 * combined with momentum as in tb_clip_rmsprop_step_f32.                                                         */
int tb_clip_rmsprop_ex_step_f32(float* params, float* grads, float* square_avg, float* grad_avg, float* momentum_buf,
                                int64_t n, const float* sumsq, float max_norm, const float* lr_device, float lr,
                                float alpha, float eps, float weight_decay, float momentum, const tb_hparams* hp,
                                float* grad_norm_out, void* stream);

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
/* Split-bf16 ("bf16x3") form of tb_gemm_bf16_ex with the fused epilogue the network's products use: each operand holds
 * its lo plane bf16(x - hi) a_lo / b_lo elements after its hi plane (same leading dimension), and every k-step issues
 * lo.hi, hi.lo, hi.hi into one fp32 accumulator.  C = relu?(scale * acc + bias), then zeroed where mask_bf16 [M,N]
 * (ldmask, nullable) is not positive; C_bf16 (nullable) gets the hi plane and, when c16_lo != 0, the lo plane c16_lo
 * elements further.  splits > 1: fp32 C only, no mask.  A test and diagnostic entry point that reaches the learner's
 * split-mode kernel configurations in isolation; the learner itself calls the kernel from C++, not through it.         */
int tb_gemm_bf16x3_ex(const void* A_bf16, const void* B_bf16, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                      int a_mn, int b_mn, int64_t a_lo, int64_t b_lo, float* C, int64_t ldc, void* C_bf16, int64_t ldc16,
                      int64_t c16_lo, const float* bias, float scale, int relu, const void* mask_bf16, int64_t ldmask,
                      int splits, float* partial, void* stream);
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
/* Split-bf16 ("bf16x3") forms of the five entries above: each bf16 operand / output is a hi plane followed, *_lo elements
 * further, by its lo plane bf16(x - hi), and every k-step issues lo.hi, hi.lo, hi.hi.  The weights are packed as a hi
 * plane of O*KH*KW*C elements with the lo plane right behind it: pack_scratch_bf16 >= 2*O*KH*KW*C bf16 (conv1: 2*32*256).
 * The input gradient's ReLU mask reads the hi plane of act_bf16.  conv1's pixels are exact in bf16, so its image has no
 * lo plane.  Test and diagnostic entry points: the learner calls the same internals from C++.                           */
int tb_conv_nhwc_bf16x3_fwd(const void* act_bf16, int64_t act_lo, const float* weight, const float* bias, int64_t Nf, int H,
                            int W, int C, int KH, int KW, int S, int O, int relu, void* out_bf16, int64_t out_lo,
                            void* pack_scratch_bf16, void* stream);
int tb_conv_nhwc_bf16x3_dgrad(const void* dy_bf16, int64_t dy_lo, const float* weight, const void* act_bf16, int64_t Nf,
                              int H, int W, int C, int KH, int KW, int S, int O, void* dx_bf16, int64_t dx_lo,
                              void* pack_scratch_bf16, void* stream);
int tb_conv_nhwc_bf16x3_wgrad(const void* dy_bf16, int64_t dy_lo, const void* act_bf16, int64_t act_lo, int64_t Nf, int H,
                              int W, int C, int KH, int KW, int S, int O, float* dweight, float* partial,
                              int64_t partial_floats, void* stream);
int tb_conv1_u8_bf16x3_fwd(const uint8_t* frame, const float* weight, const float* bias, int64_t N, int H, int W, int S,
                           int relu, void* out_bf16, int64_t out_lo, void* image_bf16, void* pack_scratch_bf16,
                           void* stream);
int tb_conv1_u8_bf16x3_wgrad(const void* dy_bf16, int64_t dy_lo, const void* image_bf16, int64_t N, int H, int W, int S,
                             float* dweight, float* partial, int64_t partial_floats, void* stream);

/* ---- IMPALA ResNet 3x3 convolutions on shifted-window split-bf16 kernels -----------------------------------------------
 * The building blocks of the precision 2 ResNet trunk, for tests and diagnostics (the learner calls them from C++).
 * Padded planar image of an Nf x H x W x C tensor (C a multiple of 8): one plane of bf16 elements laid out as
 *   [Nf][C/8][(H+2)*(W+2)][8]   (frame, 8-channel chunk, zero-padded pixel in row-major order, channel in chunk),
 * followed by slack (zeros) that a frame's last tile may read past the last plane; tb_sw_image_elems() elements per plane
 * slack included.  The hi plane is at the base, the lo plane lo_off elements further (lo_off > 0, a multiple of 8).
 * Producers write every element of both planes, borders and slack included.                                            */
int64_t tb_sw_image_elems(int64_t Nf, int H, int W, int C);
/* fp32 NHWC x [Nf,H,W,C] (through ReLU if relu_in) -> padded planar hi / lo image.  db != NULL: also db[C] = column sums
 * of x (no ReLU), with scratch of tb_sw_colsum_scratch_floats() floats.                                                  */
int tb_sw_pad_split_f32(const float* x, void* out, int64_t lo_off, int64_t Nf, int H, int W, int C, int relu_in, float* db,
                        float* scratch, int64_t scratch_floats, void* stream);
int64_t tb_sw_colsum_scratch_floats(int64_t Nf, int H, int W, int C);
/* uint8 NCHW frames [Nf, 1 <= Cf <= 16, H, W] -> 16-channel padded planar image (channels >= Cf and the lo plane zero) */
int tb_sw_frames_u8(const uint8_t* frame, void* out, int64_t lo_off, int64_t Nf, int Cf, int H, int W, void* stream);
/* weights fp32 [O,C,3,3] -> the packed hi / lo operand (tb_sw_weight_elems(O, C) bf16) of tb_sw_conv_fwd with CK = C,
 * NO = O (transpose = 0), or of the input-gradient convolution with CK = O, NO = C and flipped taps (transpose = 1).
 * c_real > 0 (forward only): the weights are [O,c_real,3,3] and input channels >= c_real get zeros.                    */
int64_t tb_sw_weight_elems(int O, int C);
int tb_sw_pack_weights(const float* weight, void* out, int O, int C, int transpose, int c_real, void* stream);
/* out fp32 [Nf*H*W, NO] = 3x3 / stride 1 / pad 1 convolution of a CK-channel image (CK, NO in {16, 32, 64}), then the
 * epilogue in this order: * scale, + bias[NO], zeroed where mask [Nf*H*W, NO] is not positive, + addend [Nf*H*W, NO]
 * (each nullable).  emit != NULL: the result (through ReLU if emit_relu) is also written as the complete padded planar
 * image of NO channels (lo plane at emit_lo).  csum != NULL: per (tile, warp) column sums of the result,
 * [tb_sw_csum_rows(Nf, H, W)][NO] floats plus 128*NO floats of scratch behind them for tb_sw_csum_reduce, which folds
 * them into db[C] in a fixed order.                                                                                      */
int tb_sw_conv_fwd(const void* img, int64_t img_lo, const void* wk, float* out, int64_t Nf, int H, int W, int CK, int NO,
                   float scale, const float* bias, const float* mask, const float* addend, void* emit, int64_t emit_lo,
                   int emit_relu, float* csum, void* stream);
int64_t tb_sw_csum_rows(int64_t Nf, int H, int W);
int tb_sw_csum_reduce(float* csum, int64_t rows, int C, float* db, void* stream);
/* dweight fp32 [O, c_real or C, 3, 3] = scale * sum over pixels of dY (x) input windows, from the dY image (O channels)
 * and the input image (C channels); W >= 5; partial >= 132*O*9*C floats.                                              */
int tb_sw_conv_wgrad(const void* dyimg, int64_t dy_lo, const void* ximg, int64_t x_lo, float* dweight, int64_t Nf, int H,
                     int W, int C, int O, float scale, int c_real, float* partial, int64_t partial_floats, void* stream);
/* nn.MaxPool2d(3, 2, 1) backward into an image: dy_pooled fp32 [Nf,OH,OW,C] and the argmax taps of
 * tb_maxpool3x3s2_fwd_f32 -> padded planar image of dL/d(pool input) [Nf,H,W,C] and db[C] = its column sums.          */
int tb_sw_pool_bwd_image_colsum(const uint8_t* argmax, const float* dy_pooled, void* out, int64_t lo_off, int64_t Nf, int H,
                                int W, int C, float* db, float* scratch, int64_t scratch_floats, void* stream);
/* nn.MaxPool2d(3, 2, 1) forward on fp32 NHWC [N,H,W,C] -> y [N,OH,OW,C] and argmax u8 [N,OH,OW,C]: the tap kh*3 + kw
 * (0..8) of each window's first maximum in row-major tap order.                                                       */
int tb_maxpool3x3s2_fwd_f32(const float* x, float* y, uint8_t* argmax, int64_t N, int H, int W, int C, void* stream);
/* out_bf16[r, c] = bf16(in[r*ld + c]) for c < cols, 0 for cols <= c < ld16 (operand staging). */
int tb_f32_to_bf16(const float* in, void* out_bf16, int64_t rows, int64_t cols, int64_t ld, int64_t ld16,
                   void* stream);

/* ---- fp32 network building blocks -----------------------------------------------------------------------------------
 * The kernels of the fp32 backend, the ResNet patch-matrix path, the fused heads and the bias-gradient column sums, for
 * tests and diagnostics (the learner calls the same internals from C++).  Every entry is a thin wrapper that adds no
 * behaviour.
 *
 * fp32 SIMT GEMM: C[M,N] (+)= sum_k A(m,k) B(k,n), A(m,k) = ta ? A[k*lda + m] : A[m*lda + k], B(k,n) = tb ? B[n*ldb + k]
 * : B[k*ldb + n]; a_u8 / b_u8: the operand is uint8, read as x/255.  The five (a_u8, b_u8, ta, tb) combinations the
 * learner runs are (0,0,0,1) forward, (1,0,0,1) uint8 forward, (0,0,0,0) input gradient, (0,0,1,0) weight gradient and
 * (0,1,1,0) uint8 weight gradient; any other is rejected.  splits (clamped to the K tiles of 16) > 1 or permP * permQ > 1
 * takes the split-K path: raw partials [splits][M][N] in scratch, then a fixed-order reduce that applies C = scale * sum
 * + bias, ReLU, and stores column n = p*permQ + q at q*permP + p (permP * permQ = N).  Otherwise the direct path applies
 * C = acc + bias, ReLU, zeroed where mask [M, ldmask] is not positive, + addend [M, ldadd].  Either then stores C, or adds
 * it to C when accumulate.  An epilogue field the chosen path does not apply (mask or addend on the split-K path, scale
 * != 1 on the direct path) is rejected.  tb_gemm_f32_splits is the split count the learner picks for a weight gradient,
 * with tb_splitk_scratch_floats() floats of partials.                                                                  */
int tb_gemm_f32(const void* A, int a_u8, const void* B, int b_u8, int ta, int tb, int64_t M, int64_t N, int64_t K, int64_t lda,
                int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, const float* mask, int64_t ldmask,
                const float* addend, int64_t ldadd, int accumulate, int permP, int permQ, float scale, int splits, float* scratch,
                void* stream);
int tb_gemm_f32_splits(int64_t M, int64_t N, int64_t K, int64_t scratch_floats, int64_t cap);
int64_t tb_splitk_scratch_floats(void);
/* AtariNet patch matrices: frames u8 NCHW [N,C,H,W] -> u8 [N*OH*OW, C*KH*KW] (k = (c*KH + kh)*KW + kw); act f32 NHWC
 * [N,H,W,C] -> f32 [N*OH*OW, KH*KW*C] (k = (kh*KW + kw)*C + c, C % 4 == 0); col2im is the gather-form adjoint of the
 * latter, times (act > 0) when act is not NULL.  No padding.                                                            */
int tb_im2col_u8_nchw(const uint8_t* frame, uint8_t* col, int64_t N, int C, int H, int W, int KH, int KW, int S, void* stream);
int tb_im2col_f32_nhwc(const float* act, float* col, int64_t N, int H, int W, int C, int KH, int KW, int S, void* stream);
int tb_col2im_f32_nhwc(const float* dcol, const float* act, float* dact, int64_t N, int H, int W, int C, int KH, int KW, int S,
                       void* stream);
/* out[o, p*Q + q] = in[o, q*P + p] */
int tb_permute_pq(const float* in, float* out, int64_t O, int P, int Q, void* stream);
/* X[m, n] = 0 where !(Y[m, n] > 0), n < ncols */
int tb_relu_mask_f32(float* X, const float* Y, int64_t M, int64_t ncols, int64_t ldx, int64_t ldy, void* stream);
/* core[n, F] = clamp(reward[n], -1, 1), core[n, F+1+j] = (last_action[n] == j) for j < A */
int tb_core_extras(float* core, int64_t ld, int64_t N, int F, const float* reward, const int64_t* last_action, int A,
                   void* stream);
/* ResNet patch-matrix path; dtype 0 = fp32, 1 = bf16 for every operand.  im2col3x3: x NHWC [N,H,W,C] (through ReLU if
 * relu_in) -> col [N*H*W, ldk], k = (kh*3 + kw)*C + c, 3x3 / stride 1 / zero padding 1.  im2col3x3_u8: frames u8 NCHW
 * [N,1..16,H,W] -> col [N*H*W, ldk] (dtype 0: uint8, 1: bf16), k = (c*3 + kh)*3 + kw.  col2im3x3: its adjoint, dx =
 * gather(dcol) * (relu_src > 0 if relu_src) + addend (each nullable).  maxpool3x3s2: nn.MaxPool2d(3, 2, 1) on NHWC with the
 * argmax taps of tb_maxpool3x3s2_fwd_f32; the backward gathers dy through them.  relu: y = max(x, 0), dx = dy * (x > 0). */
int tb_im2col3x3(const void* x, void* col, int64_t N, int H, int W, int C, int64_t ldk, int relu_in, int dtype, void* stream);
int tb_im2col3x3_u8(const uint8_t* frame, void* col, int64_t N, int C, int H, int W, int64_t ldk, int dtype, void* stream);
int tb_col2im3x3(const void* dcol, const void* relu_src, const void* addend, void* dx, int64_t N, int H, int W, int C, int64_t ldk,
                 int dtype, void* stream);
int tb_maxpool3x3s2_fwd(const void* x, void* y, uint8_t* argmax, int64_t N, int H, int W, int C, int dtype, void* stream);
int tb_maxpool3x3s2_bwd(const uint8_t* argmax, const void* dy, void* dx, int64_t N, int H, int W, int C, int dtype, void* stream);
int tb_relu_fwd(const void* x, void* y, int64_t n, int dtype, void* stream);
int tb_relu_bwd(const void* x, const void* dy, void* dx, int64_t n, int dtype, void* stream);
/* Bias-gradient column sums out[n] = sum_m X[m*ld + n], n < ncols, fp32 accumulation in a fixed order.  bf16: plus the lo
 * plane lo_off elements further when lo_off != 0.  scratch >= tb_colsum_scratch_floats(ncols) floats, and for bf16 at
 * least tb_colsum_scratch_floats(512).                                                                                  */
int64_t tb_colsum_scratch_floats(int64_t ncols);
int tb_colsum_f32(const float* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, void* stream);
int tb_colsum_bf16(const void* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, int64_t lo_off,
                   void* stream);
/* Fused policy / baseline heads: logits [N,A] = x Wp^T + bp, baseline [N,V] = x Wb^T + bb, x [N, ldx >= F]; 1 <= A <= 31,
 * 1 <= V <= 64, F <= 12288.  The backward gives dx [N, lddx] and overwrites dWp, dbp, dWb, dbb, with
 * tb_heads_scratch_floats(N, F, A, V) floats of scratch, at most 120 * (A + V) * (F + 1) whatever N.                  */
int64_t tb_heads_scratch_floats(int64_t N, int F, int A, int V);
int tb_heads_forward(const float* x, int64_t ldx, const float* Wp, const float* bp, const float* Wb, const float* bb, int64_t N,
                     int F, int A, int V, float* logits, float* baseline, void* stream);
int tb_heads_backward(const float* x, int64_t ldx, const float* Wp, const float* Wb, const float* dlogits, const float* dbaseline,
                      int64_t N, int F, int A, int V, float* dx, int64_t lddx, float* dWp, float* dbp, float* dWb, float* dbb,
                      float* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TORCHBEAST_B200_H_ */
