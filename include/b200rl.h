/*
 * b200rl.h -- C-ABI of libb200rl.so: the H100-native (sm_90a) PPO hot path.
 *
 * The reference (vwxyzjn/cleanrl) is pure Python/PyTorch and has NO native
 * interface; this header is the boundary SURVEY.md section 8(b) defines for it.
 * Every entry point replaces a block of torch calls inside the reference's
 * training loop (file:line cited per function, relative to the reference root).
 *
 * Conventions
 *   - plain C: raw DEVICE pointers + explicit sizes, scalars by value.  No
 *     torch / C++ types.  The caller (PyTorch in the shipped host code) owns
 *     every buffer including workspaces; nothing here allocates or frees
 *     device memory, and nothing synchronises the device.
 *   - every function only ENQUEUES work on `stream` (a cudaStream_t passed as
 *     void*; NULL = legacy default stream) and is CUDA-graph capturable.
 *   - return value: 0 on success, negative b200rl_status on failure.  The
 *     failing call's message is kept per host thread: b200rl_last_error().
 *   - "f32" = IEEE binary32.  All matrices are dense row-major unless a leading
 *     dimension / layout is spelled out.
 *   - python-double hyper-parameters (gamma, lr, betas, eps ...) are passed as
 *     double and rounded exactly where the reference rounds them.
 */
#ifndef B200RL_H
#define B200RL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    B200RL_OK = 0,
    B200RL_ERR_INVALID_ARGUMENT = -1,
    B200RL_ERR_CUDA = -2,
    B200RL_ERR_UNSUPPORTED = -3,
    B200RL_ERR_WORKSPACE = -4
} b200rl_status;

/* library version: major*10000 + minor*100 + patch */
int b200rl_version(void);
/* message of the last failing call on this host thread ("" if none) */
const char* b200rl_last_error(void);
/* compute capability the kernels were compiled for (90 = sm_90a) */
int b200rl_compiled_arch(void);

/* Optional per-kernel timing: when enabled, every kernel launch below is bracketed by CUDA events
 * on its stream.  b200rl_profile_summary synchronises the device and writes a JSON array
 * [{"name","launches","ms","flops","bytes"}] (algorithmic flops/bytes per kernel family) into buf.
 * Do not enable during CUDA-graph capture. */
/* number of kernels this library has launched in this process (host-side counter) */
long long b200rl_launch_count(void);
void b200rl_profile_enable(int on);
void b200rl_profile_reset(void);
int b200rl_profile_summary(char* buf, size_t capacity);

/* ---------------------------------------------------------------- GAE -----
 * Reverse-scan generalised advantage estimation over a (T x N) rollout.
 * Replaces the python loop cleanrl/ppo.py:218-231 (identical in
 * ppo_atari_envpool.py:250-263, ppo_atari_multigpu.py:288-301,
 * ppo_continuous_action.py:233-246).
 *   rewards, values, dones : f32 [T, N] (N contiguous)
 *   next_value, next_done  : f32 [N]
 *   advantages, returns    : f32 [T, N] out  (returns = advantages + values)
 *   gamma, gae_lambda      : python doubles; gamma -> f32 once,
 *                            gamma*gae_lambda -> f32 once (ppo.py:230)
 *   mode 0: one thread per env, every op individually rounded (no FMA):
 *           bit-identical to the reference loop.
 *   mode 1: time-chunked affine scan (3 short dependent phases instead of T
 *           steps); re-associated, |err| ~1e-7 relative.
 */
int b200rl_gae_f32(const float* rewards, const float* values, const float* dones,
                   const float* next_value, const float* next_done,
                   float* advantages, float* returns,
                   int64_t T, int64_t N, double gamma, double gae_lambda,
                   int mode, void* stream);

/* ------------------------------------------------ categorical policy head --
 * Rollout-side policy epilogue.  Replaces Categorical(logits) + sample() +
 * log_prob() + entropy() in Agent.get_action_and_value
 * (cleanrl/ppo_atari_envpool.py:143-149, cleanrl/ppo.py:121-126) and the four
 * rollout-buffer stores ppo.py:200-202.
 *   logits  : f32 [n, A], row stride ld_logits elements
 *   noise   : f32 [n, A] Exp(1) draws from the CALLER's generator (torch's
 *             multinomial consumes exactly `empty_like(probs).exponential_(1)`),
 *             action = argmax(softmax(normalised logits) / noise), first max wins.
 *   value_in: optional f32 [n] (stride ld_value) copied to value_out (may be NULL)
 *   outputs : action i64 [n], logprob f32 [n], entropy f32 [n] (entropy may be NULL)
 */
int b200rl_categorical_sample_f32(const float* logits, int64_t ld_logits, const float* noise,
                                  const float* value_in, int64_t ld_value,
                                  int64_t n, int A,
                                  int64_t* action, float* logprob, float* entropy, float* value_out,
                                  void* stream);

/* log_prob and entropy of GIVEN actions (the action != None branch of
 * Agent.get_action_and_value, cleanrl/ppo.py:121-126).  action i64 [n] (clamped to [0,A)). */
int b200rl_categorical_eval_f32(const float* logits, int64_t ld_logits, const int64_t* action,
                                int64_t n, int A, float* logprob, float* entropy, void* stream);

/* -------------------------------------------------------------- PPO loss ---
 * Fused minibatch loss: gather by mb_inds, advantage normalisation (unbiased
 * std), ratio, both KL estimates, clipfrac, clipped surrogate, clipped value
 * loss, entropy bonus, AND the gradients wrt the policy logits / value that
 * autograd would produce.  Replaces cleanrl/ppo.py:250-285 (+ the part of
 * loss.backward() :288 above the network).
 *   new_logits : f32 [M, A] (row stride ld_logits); new_value: f32 [M] (stride ld_value)
 *   mb_inds    : i64 [M] rows of the flat batch (NULL = 0..M-1)
 *   b_*        : flat batch tensors of length B >= max(mb_inds)+1
 *                b_actions i64, b_logprobs/b_advantages/b_returns/b_values f32
 *   dlogits    : f32 [M, A] (row stride ld_dlogits) out; dvalue: f32 [M] (stride ld_dvalue) out
 *   stats      : f32 [16] out: 0 pg_loss, 1 v_loss, 2 entropy, 3 old_approx_kl,
 *                4 approx_kl, 5 clipfrac, 6 loss, 7 adv_mean, 8 adv_std
 *   workspace  : >= b200rl_ppo_loss_workspace_bytes(M) bytes, 16-B aligned.
 * Deterministic: fixed-order two-level reductions, no float atomics.
 */
size_t b200rl_ppo_loss_workspace_bytes(int64_t M);
int b200rl_ppo_loss_f32(const float* new_logits, int64_t ld_logits,
                        const float* new_value, int64_t ld_value,
                        const int64_t* mb_inds,
                        const int64_t* b_actions, const float* b_logprobs,
                        const float* b_advantages, const float* b_returns, const float* b_values,
                        int64_t M, int A,
                        double clip_coef, double ent_coef, double vf_coef,
                        int norm_adv, int clip_vloss,
                        float* dlogits, int64_t ld_dlogits, float* dvalue, int64_t ld_dvalue,
                        float* stats, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------ diagonal Gaussian policy --
 * Continuous-action twin of the three entry points above (cleanrl/ppo_continuous_action.py:134-141:
 * Normal(action_mean, exp(actor_logstd)), log_prob(a).sum(1), entropy().sum(1)).
 *   mean f32 [n, D] (row stride ld_mean), logstd f32 [D] (the state-independent actor_logstd parameter),
 *   noise f32 [n, D] N(0,1) from the caller's generator (torch.normal(mean, std) == randn*std + mean),
 *   action f32 [n, D].  The loss additionally returns dlogstd [D] (deterministic batch reduction).
 */
int b200rl_gaussian_sample_f32(const float* mean, int64_t ld_mean, const float* logstd, const float* noise,
                               const float* value_in, int64_t ld_value, int64_t n, int D,
                               float* action, float* logprob, float* entropy, float* value_out, void* stream);
int b200rl_gaussian_eval_f32(const float* mean, int64_t ld_mean, const float* logstd, const float* action,
                             int64_t n, int D, float* logprob, float* entropy, void* stream);
size_t b200rl_ppo_loss_gaussian_workspace_bytes(int64_t M);
int b200rl_ppo_loss_gaussian_f32(const float* new_mean, int64_t ld_mean, const float* logstd,
                                 const float* new_value, int64_t ld_value, const int64_t* mb_inds,
                                 const float* b_actions, const float* b_logprobs,
                                 const float* b_advantages, const float* b_returns, const float* b_values,
                                 int64_t M, int D, double clip_coef, double ent_coef, double vf_coef,
                                 int norm_adv, int clip_vloss,
                                 float* dmean, int64_t ld_dmean, float* dlogstd, float* dvalue, int64_t ld_dvalue,
                                 float* stats, void* workspace, size_t workspace_bytes, void* stream);
/* The same loss with the policy mean shifted per row (cleanrl/rpo_continuous_action.py:138-142: Normal(mean + z, std)
 * when the update re-evaluates stored actions).  mean_shift f32 [M, D] (row stride ld_shift >= D, minibatch row
 * order, not gathered through mb_inds); each row uses mu = fl(new_mean + mean_shift) wherever the loss above uses
 * new_mean.  dmean is d loss / d new_mean (== d loss / d mu).  Same launches, workspace and other arguments as
 * b200rl_ppo_loss_gaussian_f32; a null mean_shift is refused. */
int b200rl_ppo_loss_gaussian_shift_f32(const float* new_mean, int64_t ld_mean, const float* logstd,
                                       const float* new_value, int64_t ld_value, const int64_t* mb_inds,
                                       const float* b_actions, const float* b_logprobs,
                                       const float* b_advantages, const float* b_returns, const float* b_values,
                                       const float* mean_shift, int64_t ld_shift,
                                       int64_t M, int D, double clip_coef, double ent_coef, double vf_coef,
                                       int norm_adv, int clip_vloss,
                                       float* dmean, int64_t ld_dmean, float* dlogstd, float* dvalue,
                                       int64_t ld_dvalue, float* stats, void* workspace, size_t workspace_bytes,
                                       void* stream);

/* ------------------------------------------------- grad clip + Adam step ---
 * One fused optimiser step over a FLAT f32 parameter vector: optional DP
 * averaging (grads hold the all-reduced SUM; divided by world_size first, as
 * ppo_atari_multigpu.py:369-373 does), global-L2 clip_grad_norm_
 * (torch/nn/utils/clip_grad.py: coef = max_norm/(norm+1e-6) clamped to 1) and
 * Adam (torch/optim/adam.py _single_tensor_adam op order).  Replaces
 * cleanrl/ppo.py:289-290.
 *   params, exp_avg, exp_avg_sq : f32 [P] in/out;  grads: f32 [P] in
 *   step       : 1-based count of this step (bias corrections in double)
 *   max_norm   : < 0 disables clipping (dqn_atari.py has none)
 *   norm_out   : optional f32 [1] device scalar receiving the pre-clip norm
 *   workspace  : >= b200rl_clip_adam_workspace_bytes(P) bytes
 */
size_t b200rl_clip_adam_workspace_bytes(int64_t P);
int b200rl_clip_adam_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                         int64_t P, int64_t step, double lr, double beta1, double beta2, double eps,
                         double max_norm, int world_size, float* norm_out,
                         void* workspace, size_t workspace_bytes, void* stream);
/* The same update with the two scalars that depend on (step, lr) -- sqrt(1 - beta2^step) and -lr / (1 - beta1^step), computed
 * on the host in double by b200rl_adam_step_scalars exactly as the by-value entry point computes them -- read from DEVICE
 * memory (step_scalars f32[2]): a captured CUDA graph of the update can be replayed for every later step / learning rate. */
int b200rl_adam_step_scalars(int64_t step, double lr, double beta1, double beta2, float* out2);
int b200rl_clip_adam_dyn_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                             int64_t P, const float* step_scalars, double beta1, double beta2, double eps,
                             double max_norm, int world_size, float* norm_out,
                             void* workspace, size_t workspace_bytes, void* stream);

/* clip + Adam with per-tensor semantics for a few tensors (torch.optim.Adam keeps one `step` per tensor and, like
 * clip_grad_norm_, skips a tensor whose grad is None; cleanrl/ppg_procgen.py relies on both for `aux_critic`).
 * ranges: HOST array of nranges <= 4 element ranges [ranges[2r], ranges[2r+1]) of the flat vector.
 *   range_step == 0: the ranges are frozen: left out of the clip norm, parameters and both moments untouched;
 *   range_step >= 1: the ranges are updated with (range_step, range_lr), every other element with (step, lr).
 * The clip norm is taken over the elements that are updated; max_norm < 0 disables clipping.  4-B aligned buffers;
 * workspace as b200rl_clip_adam_workspace_bytes(P). */
int b200rl_clip_adam_ranges_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                                int64_t step, double lr, const int64_t* ranges, int nranges, int64_t range_step,
                                double range_lr, double beta1, double beta2, double eps, double max_norm,
                                float* norm_out, void* workspace, size_t workspace_bytes, void* stream);
/* The same with the step-dependent scalars in DEVICE memory (what a captured CUDA graph replays): step_scalars[0..1] =
 * b200rl_adam_step_scalars(step, lr) for every element, [2..3] = those of (range_step, range_lr) for the ranges, not read
 * when `frozen` is non-zero. */
int b200rl_clip_adam_ranges_dyn_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                                    const float* step_scalars, const int64_t* ranges, int nranges, int frozen,
                                    double beta1, double beta2, double eps, double max_norm, float* norm_out,
                                    void* workspace, size_t workspace_bytes, void* stream);

/* grad clip + RAdam (torch/optim/radam.py _single_tensor_radam op order, no weight decay; cleanrl/pqn.py:152,239-240).
 * The clip norm, max_norm, norm_out, buffers and workspace are those of b200rl_clip_adam_f32 (world_size 1).  The
 * step-dependent scalars are python doubles rounded to f32 where the tensor operation that uses each of them rounds it:
 * with bc1 = 1 - beta1^step, bc2 = 1 - beta2^step and rho_t = rho_inf - 2 step beta2^step / bc2,
 *   rho_t <= 5: p -= (m / bc1) * lr
 *   rho_t >  5: p -= (((m / bc1) * lr) * (reciprocal(sqrt(v) + eps) * bc2^0.5)) * rect.
 * The second moment is fma((1 - beta2) g, g, beta2 v), one rounding, as CPU torch's addcmul_ computes it.
 * b200rl_radam_step_scalars writes out4 = (bc1, lr, bc2^0.5, rect) as f32, rect = 0 when rho_t <= 5; the _dyn entry point
 * reads those four from DEVICE memory (step_scalars f32 [4]) so a captured CUDA graph replays for any step / lr. */
int b200rl_radam_step_scalars(int64_t step, double lr, double beta1, double beta2, float* out4);
int b200rl_clip_radam_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                          int64_t step, double lr, double beta1, double beta2, double eps, double max_norm,
                          float* norm_out, void* workspace, size_t workspace_bytes, void* stream);
int b200rl_clip_radam_dyn_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                              const float* step_scalars, double beta1, double beta2, double eps, double max_norm,
                              float* norm_out, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------ phasic policy gradient: auxiliary loss ------
 * cleanrl/ppg_procgen.py:449-461 on the joint head output head_out [n][A + 2] = [logits | value | aux_value] (row stride
 * ld_head): kl_loss = mean KL(Categorical(old_logits) || Categorical(logits)), aux_value_loss = 0.5 mean (aux_value - R)^2,
 * real_value_loss = 0.5 mean (value - R)^2, loss = (aux_value_loss + beta_clone * kl_loss + real_value_loss) * inv_accum.
 * Row i reads old_logits[rows[i]][A] and returns[rows[i]] (rows null = i).  Both logit sets are normalised by
 * log-sum-exp in the kernel; a KL term with p_old == 0 is 0, one with p_new == 0 < p_old is +inf (torch's rule).
 * Writes dhead [n][A + 2] (row stride ld_dhead) = d loss / d head_out and stats[0..2] = kl_loss, aux_value_loss,
 * real_value_loss.  1 <= A <= 22, 1 <= n <= 2^22.  Two launches, sums folded in a fixed order (deterministic). */
size_t b200rl_ppg_aux_loss_workspace_bytes(int64_t n);
int b200rl_ppg_aux_loss_f32(const float* head_out, int64_t ld_head, const int64_t* rows, const float* old_logits,
                            const float* returns, int64_t n, int A, double beta_clone, double inv_accum,
                            float* dhead, int64_t ld_dhead, float* stats, void* workspace, size_t workspace_bytes,
                            void* stream);

/* ------------------------------------------------ fp32 network layers ------
 * Exact-arithmetic (fp32 FMA, CUDA cores) layers in the reference's own NCHW /
 * [out,in] layouts.  They carry configs 1 and 4 (64-wide MLPs,
 * cleanrl/ppo.py:100-116, ppo_continuous_action.py:112-129) and are the
 * validation mode of the NatureCNN (ppo_atari_envpool.py:123-139); the bf16
 * tensor-core path below is the fast path.
 *
 * act: 0 none, 1 ReLU, 2 tanh.  `rows` (i64, may be NULL) gathers the batch
 * dimension of x: sample i of the call reads x[rows[i]] (the minibatch gather
 * ppo.py:250 `b_obs[mb_inds]` without materialising it).
 */
enum { B200RL_ACT_NONE = 0, B200RL_ACT_RELU = 1, B200RL_ACT_TANH = 2 };
enum { B200RL_DT_F32 = 0, B200RL_DT_U8 = 1 };

/* y[n,Cout,OH,OW] = act(conv(x[n,Cin,H,W] / in_div, w[Cout,Cin,KH,KW]) + b)  (in_div = 255 for uint8 obs, 1 otherwise) */
int b200rl_conv2d_fwd_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                          const float* w, const float* b, float* y,
                          int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride,
                          int act, void* stream);
/* Same with zero padding `pad` on every side (IMPALA-CNN 3x3 convolutions, cleanrl/ppo_procgen.py:92-93,110). */
int b200rl_conv2d_fwd_pad_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                              const float* w, const float* b, float* y,
                              int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad,
                              int act, void* stream);
int b200rl_conv2d_bwd_data_pad_f32(const float* dy, const float* w, const float* x_post, int prev_act, float* dx,
                                   int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad, void* stream);
size_t b200rl_conv2d_bwd_weight_pad_workspace_bytes(int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad);
int b200rl_conv2d_bwd_weight_pad_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                                     const float* dy, float* dw, float* db,
                                     int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad,
                                     void* workspace, size_t workspace_bytes, void* stream);
/* IMPALA-CNN glue (cleanrl/ppo_procgen.py:89-150), fp32 NCHW:
 *   maxpool3s2: max_pool2d(kernel 3, stride 2, padding 1) on [nc, H, W] planes -> [nc, (H+1)/2, (W+1)/2]; argmax u8 (0..8)
 *   relu / relu_bwd (dx = dy * (x > 0) + extra, extra may be NULL) / add: pre-activation residual blocks
 *   nhwc_to_nchw_u8: frames [n, H, W, C] (optionally gathered through rows) -> [n, C, H, W] */
int b200rl_maxpool3s2_fwd_f32(const float* x, int64_t nc, int H, int W, float* y, uint8_t* argmax, void* stream);
int b200rl_maxpool3s2_bwd_f32(const float* dy, const uint8_t* argmax, int64_t nc, int H, int W, float* dx, void* stream);
int b200rl_relu_f32(const float* x, int64_t n, float* y, void* stream);
int b200rl_relu_bwd_f32(const float* dy, const float* x, const float* extra, int64_t n, float* dx, void* stream);
int b200rl_add_f32(const float* a, const float* b, int64_t n, float* y, void* stream);
int b200rl_nhwc_to_nchw_u8(const uint8_t* x, const int64_t* rows, int64_t n, int H, int W, int C, uint8_t* y, void* stream);
/* dx = conv_transpose(dy, w) * act'(x_post) ; x_post = the layer input as the
 * previous layer's post-activation output (prev_act selects the derivative). */
int b200rl_conv2d_bwd_data_f32(const float* dy, const float* w, const float* x_post, int prev_act,
                               float* dx,
                               int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride,
                               void* stream);
/* dw[Cout,Cin,KH,KW] = sum_m dy * im2col(x / in_div) ; db[Cout] = sum dy.  Deterministic split
 * reduction through `workspace` (b200rl_conv2d_bwd_weight_workspace_bytes). */
size_t b200rl_conv2d_bwd_weight_workspace_bytes(int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride);
int b200rl_conv2d_bwd_weight_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                                 const float* dy, float* dw, float* db,
                                 int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride,
                                 void* workspace, size_t workspace_bytes, void* stream);
/* y[n,out] = act(x[n,in] @ w[out,in]^T + b) ; x rows optionally gathered */
int b200rl_linear_fwd_f32(const float* x, const int64_t* rows, const float* w, const float* b, float* y,
                          int64_t n, int in_features, int out_features, int act, void* stream);
int b200rl_linear_bwd_data_f32(const float* dy, const float* w, const float* x_post, int prev_act, float* dx,
                               int64_t n, int in_features, int out_features, void* stream);
size_t b200rl_linear_bwd_weight_workspace_bytes(int64_t n, int in_features, int out_features);
int b200rl_linear_bwd_weight_f32(const float* x, const int64_t* rows, const float* dy, float* dw, float* db,
                                 int64_t n, int in_features, int out_features,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------- NatureCNN, bf16 tensor cores ---
 * The throughput path of Agent.network/actor/critic (cleanrl/ppo_atari_envpool.py:123-149):
 * every conv / linear contraction (forward, data-gradient, weight-gradient) is an implicit GEMM
 * on wgmma with bf16 operands and fp32 accumulation in registers, fed by TMA; a minibatch gather
 * (rows) is the image coordinate of conv1's TMA boxes, nothing is materialised; the two heads
 * (A+1 outputs, 1 <= A <= 23) run in fp32 on CUDA cores.  Wide heads (24 <= A+1 <= 2048 outputs, e.g. the
 * A * n_atoms logits of C51) run on wgmma instead: bf16 hidden x bf16 head weights with fp32 output + bias, and in the
 * backward a bf16 copy of dhead feeds the dhid GEMM and the head weight gradient (fixed-order fold over row
 * splits); the head bias gradient is an fp32 column sum of dhead.  A+1 > 2048 is B200RL_ERR_INVALID_ARGUMENT.
 *
 * params / grads: ONE flat f32 vector in libb200rl order
 *     conv1.w[32,4,8,8] conv1.b[32] conv2.w[64,32,4,4] conv2.b[64] conv3.w[64,64,3,3] conv3.b[64]
 *     fc.w[512,3136] fc.b[512] actor.w[A,512] critic.w[1,512] actor.b[A] critic.b[1]
 *   (each tensor in torch's own element order; b200rl_naturecnn_param_count(A) elements).
 * packed : bf16 GEMM operand copies of the weights (b200rl_naturecnn_bf16_packed_bytes), refreshed
 *          by b200rl_naturecnn_bf16_pack after every optimiser step.
 * acts   : activation + activation-gradient workspace for batch n (b200rl_naturecnn_bf16_acts_bytes);
 *          forward fills it, backward consumes it.  The caller must ZERO it once before its first use
 *          with a given n (zero-padded gradient grids rely on never-written positions staying 0).
 * obs    : obs_format B200RL_OBS_U8_NCHW  : uint8 [*, 4, 84, 84] frames as the env delivers them, or
 *          obs_format B200RL_OBS_S2D_BF16 : bf16 [*, 21, 21, 64] space-to-depth frames produced ONCE per
 *          env step by b200rl_frames_to_s2d_bf16 (channel = c*16 + sy*4 + sx of pixel (4Y+sy, 4X+sx)):
 *          conv1 (8x8 stride 4) is then a 2x2 stride-1 convolution over 128-byte pixels and the 16
 *          minibatch passes of an iteration never touch / convert the uint8 frames again.
 *          rows (i64 [n], may be NULL) selects the samples (ppo.py:250 gather) in either format; the
 *          indices are the caller's contract (not range-checked); ascending order keeps the gather
 *          DRAM-page friendly (the engine sorts every minibatch).
 * head_out / dhead : f32 [n, A+1] = [logits | value] and its gradient.
 */
enum { B200RL_OBS_U8_NCHW = 0, B200RL_OBS_S2D_BF16 = 1, B200RL_OBS_S2D_U8 = 2 };
int b200rl_frames_to_s2d_bf16(const uint8_t* obs, const int64_t* rows, int64_t n, void* out_s2d, void* stream);
/* B200RL_OBS_S2D_U8: the rollout keeps each frame as uint8 space-to-depth(4) pixels (28 224 B, the algorithmic minimum;
 * reference: fp32, 112 896 B, ppo_atari_envpool.py:203) in TWO orientations written once per env step:
 *   out_rm u8 [n, 441 grid rows, 64 channels]  -> `obs` of forward and backward: conv1 on the integer tensor cores
 *                                                  (kind::i8) and the conv1 weight gradient (pixels expanded
 *                                                  uint8 -> fp16 in shared memory)
 *   out_cm u8 [n, 64 channels, 448 grid rows]  -> `obs_aux` of backward: required, no longer read
 * channel = c*16 + sy*4 + sx of source pixel (4Y+sy, 4X+sx), grid row = Y*21 + X; rows 441..447 of out_cm are zero. */
int b200rl_frames_to_s2d_u8(const uint8_t* obs, const int64_t* rows, int64_t n, uint8_t* out_rm, uint8_t* out_cm, void* stream);
/* Frame-stack delta upload (csrc/frame_stack.cu).  The Atari observation the reference uploads whole every step
 * (cleanrl/ppo_atari_envpool.py:185-196 stack_num=4, :226,239 `torch.Tensor(next_obs).to(device)`) is a stack of the 4 newest
 * frames: planes 0..2 of an env's observation are planes 1..3 of its previous one unless the env was reset.  Only the newest
 * plane (7 056 B instead of 28 224 B per env) has to cross PCIe; the device rebuilds rollout slot t from slot t-1:
 *   new_planes  u8 [n, 7056]   newest plane of every env
 *   full_slot   i32 [n] or NULL: -1 = shifted stack, k >= 0 = take all 4 planes from full_frames[k] (u8 [*, 4, 84, 84])
 *   prev_rm/prev_cm            the previous slot in the two B200RL_OBS_S2D_U8 orientations (must not alias the outputs) */
int b200rl_frames_delta_s2d_u8(const uint8_t* new_planes, const int32_t* full_slot, const uint8_t* full_frames,
                               const uint8_t* prev_rm, const uint8_t* prev_cm, int64_t n,
                               uint8_t* out_rm, uint8_t* out_cm, void* stream);
/* rows x row_bytes from pitched (pinned) host memory into a dense device buffer (cudaMemcpy2DAsync): the newest planes are
 * uploaded straight from the env's own observation batch, no host-side packing. */
int b200rl_h2d_rows_async(void* dst, const void* src, int64_t src_pitch, int64_t row_bytes, int64_t rows, void* stream);
/* Host-side tracker, one per vector env (HOST pointers; no stream).  It owns a private mirror of every env's last
 * observation and a pool of `threads` worker threads (0 = run inline).
 *   begin(): env i's observation starts at obs + i*env_stride (planes contiguous).  Envs with done[i] != 0 (f32, may be NULL)
 *            -- and every env on the first pass / after invalidate() -- are staged as full frames: full_out[k] (pinned,
 *            [n, planes*plane_bytes]) and slot_out[i] = k; all other envs get slot_out[i] = -1.  new_out (pinned
 *            [n, plane_bytes], may be NULL when the caller uploads the newest planes from `obs` itself) receives the newest
 *            planes.  Returns the number of full frames (>= 0; negative = error) and starts the ASYNCHRONOUS verification:
 *            the workers memcmp the first planes-1 planes of every slot -1 env against the mirror and refresh the mirror.
 *            `obs` must stay unchanged until wait() returns.
 *   wait():  joins the verification; returns how many slot -1 envs did NOT hold the shifted stack (their indices, ascending,
 *            in mismatch_out i32 [n]): the caller must re-stage those as full frames and redo the step.  Every begin() must
 *            be followed by one wait(). */
void* b200rl_stackdelta_create(int64_t n_envs, int planes, int64_t plane_bytes, int threads);
void b200rl_stackdelta_destroy(void* tracker);
void b200rl_stackdelta_invalidate(void* tracker);
int64_t b200rl_stackdelta_begin(void* tracker, const uint8_t* obs, int64_t env_stride, const float* done,
                                uint8_t* new_out, uint8_t* full_out, int32_t* slot_out);
int64_t b200rl_stackdelta_wait(void* tracker, int32_t* mismatch_out);
/* One env group's whole rollout step in ONE host call (the grouped loop of PPOEngine.collect is bounded by per-step host
 * overhead once only a plane per env crosses PCIe).  `plan` is filled once per (step, group):
 *   launch(): begin() on `tracker` (NULL = nothing to upload: the slot is rebuilt from device data only), H2D of the staged
 *             full frames / slot table / newest planes on `copy_stream` (straight from `obs` when it is pinned memory, else
 *             through new_h), then per chunk c: main_stream waits h2d_event[c] and launches graph_exec[c] (a cudaGraphExec_t
 *             holding that chunk's storage rebuild + policy + sampler), records `consumed_event`, copies the actions D2H
 *             (actions_bytes > 0) and records d2h_event.  Returns the number of whole observations staged (or < 0).
 *   join():   cudaEventSynchronize(d2h_event) (may be NULL) + wait() on `tracker` (may be NULL / nothing pending -> 0). */
typedef struct B200rlPartLaunch {
    void* tracker;
    void* copy_stream;
    void* main_stream;
    void* consumed_event;
    int32_t n, nchunks;
    int32_t chunk_lo[4], chunk_hi[4];      /* env ranges of the chunks, relative to the group */
    void* h2d_event[4];
    void* graph_exec[4];
    uint8_t* new_d; int32_t* slot_d; uint8_t* full_d;     /* device staging of the group */
    uint8_t* new_h; uint8_t* full_h; int32_t* slot_h;     /* pinned host staging of the group */
    const void* actions_d; void* actions_h; int64_t actions_bytes; void* d2h_event;
} B200rlPartLaunch;
/* numpy.random.shuffle(x) of an int64 vector on the legacy MT19937 generator (the reference's minibatch shuffle,
 * cleanrl/ppo.py:245, driven by numpy's GLOBAL RandomState), restated natively and bit-exact: key624 / pos are the state
 * words of numpy.random.get_state(); both are advanced exactly as numpy would advance them. */
int b200rl_mt19937_shuffle_i64(uint32_t* key624, int32_t* pos, int64_t* data, int64_t n);
int64_t b200rl_stackdelta_launch(const B200rlPartLaunch* plan, const uint8_t* obs, int64_t env_stride, const float* done);
int64_t b200rl_stackdelta_join(void* tracker, void* d2h_event, int32_t* mismatch_out);
int64_t b200rl_naturecnn_param_count(int A);
size_t b200rl_naturecnn_bf16_packed_bytes(int A);
size_t b200rl_naturecnn_bf16_acts_bytes(int64_t n, int obs_format);
size_t b200rl_naturecnn_bf16_workspace_bytes(int64_t n, int A);
int b200rl_naturecnn_bf16_pack(const float* params, int A, void* packed, void* stream);
int b200rl_naturecnn_bf16_forward(const void* obs, int obs_format, const int64_t* rows, int64_t n, int A,
                                  const float* params, const void* packed, void* acts,
                                  float* head_out, void* stream);
int b200rl_naturecnn_bf16_backward(const void* obs, const void* obs_aux, int obs_format, const int64_t* rows, int64_t n, int A,
                                   const float* params, const void* packed, void* acts,
                                   const float* dhead, float* grads,
                                   void* workspace, size_t workspace_bytes, void* tail_ready_event, void* stream);
/* Data-parallel overlap (cleanrl/ppo_atari_multigpu.py:360-374 exchanges the gradient after the whole backward):
 * the backward finishes the head and fc gradients FIRST; they are the contiguous tail
 * grads[b200rl_naturecnn_grad_tail_offset(A) .. param_count) = 95 % of the vector.  When `tail_ready_event`
 * (a cudaEvent_t, may be NULL) is given, it is recorded on `stream` at that point, so the caller can all-reduce the
 * tail on another stream while the convolution gradients are still being computed. */
int64_t b200rl_naturecnn_grad_tail_offset(int A);

/* ------------------------------------------------------------ IMPALA-CNN, bf16 tensor cores ---
 * cleanrl/ppo_procgen.py:89-150 (three ConvSequences 16/32/32, fc 2048 -> 256, heads), bf16 operands, fp32 accumulation.
 * params : flat fp32 vector in ImpalaAgent._param_order (the trunk in module order, both head weights, both head
 *          biases; b200rl_impala_param_count(A) elements), 16-B aligned.
 * packed : bf16 operand copies (b200rl_impala_bf16_packed_bytes), refreshed by b200rl_impala_bf16_pack after every
 *          optimiser step.
 * acts   : activation + activation-gradient workspace for batch n (b200rl_impala_bf16_acts_bytes), 256-B aligned; the
 *          backward reads what the forward of the same (obs, rows, n) left there.
 * obs    : uint8 NHWC frames [*, 64, 64, 3]; row i of the batch is frame rows[i] (rows may be NULL: frame i).
 * head_out [n, A+1] fp32 = [logits | value]; dhead [n, A+1] its gradient; grads = flat fp32 gradient (overwritten).
 * 1 <= A <= 23 (A+1 <= 24 head outputs), 0 <= n <= 131072.  Bad pointers, alignment, A or n: B200RL_ERR_INVALID_ARGUMENT
 * before any launch.  No host synchronisation or allocation: forward and backward may be captured in a CUDA graph. */
int64_t b200rl_impala_param_count(int A);
size_t b200rl_impala_bf16_packed_bytes(int A);
size_t b200rl_impala_bf16_acts_bytes(int64_t n);
/* Byte offsets of the tensors inside `acts` for batch n (all channel-last; -1 = not stored), written to
 * offsets[B200RL_IMPALA_ACTS_TENSORS] in this order:
 *   c0 bf16 [n,64,64,16], c1 bf16 [n,32,32,32], c2 bf16 [n,16,16,32]      conv outputs in front of each max-pool
 *   for each sequence q (grid 32x32x16, 16x16x32, 8x8x32):
 *     s0 (max-pool output), s1 (after block 0), s2 (after block 1; -1 for q = 2), y0, y1 (relu(conv0) of each block)
 *     bf16 [n,H,W,C]; arg uint8 [n,H,W,C] (arg-max 0..8 in the 3x3 window)
 *   h0 bf16 [n,2048] (relu of the last stream = fc input), mh0 uint32 [n,64] (its > 0 bits), hid bf16 [n,256] (fc
 *   output), mhid uint32 [n,8], then the backward scratch: dc (gradient of the last max-pool input handled, bf16 up to
 *   [n,64,64,16]), ga, gb (stream gradients, bf16 up to [n,16384]), gy (gradient of relu(conv0)), dhid bf16 [n,256]. */
#define B200RL_IMPALA_ACTS_TENSORS 30
int b200rl_impala_bf16_acts_layout(int64_t n, int64_t* offsets);
size_t b200rl_impala_bf16_workspace_bytes(int64_t n, int A);
int b200rl_impala_bf16_pack(const float* params, int A, void* packed, void* stream);
int b200rl_impala_bf16_forward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                               const void* packed, void* acts, float* head_out, void* stream);
int b200rl_impala_bf16_backward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                const void* packed, void* acts, const float* dhead, float* grads,
                                void* workspace, size_t workspace_bytes, void* stream);

/* The PPG variant (cleanrl/ppg_procgen.py:168-211): the same trunk, packed weights and activation workspace
 * (b200rl_impala_bf16_acts_bytes / _acts_layout) with a third head: head_out / dhead are [n][A + 2] =
 * [logits | value | aux_value], 1 <= A <= 22.  Flat parameters in PPGAgent._param_order: the trunk, then actor.weight,
 * critic.weight, aux_critic.weight, actor.bias, critic.bias, aux_critic.bias.  `critic` reads a detached hidden layer:
 * backward uses dhead column A for the critic's own weight and bias only, not for the hidden layer's gradient. */
int64_t b200rl_impala_ppg_param_count(int A);
size_t b200rl_impala_ppg_bf16_packed_bytes(int A);
size_t b200rl_impala_ppg_bf16_workspace_bytes(int64_t n, int A);
int b200rl_impala_ppg_bf16_pack(const float* params, int A, void* packed, void* stream);
int b200rl_impala_ppg_bf16_forward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                   const void* packed, void* acts, float* head_out, void* stream);
int b200rl_impala_ppg_bf16_backward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                    const void* packed, void* acts, const float* dhead, float* grads,
                                    void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------- recurrent agent, bf16 tensor cores ---
 * cleanrl/ppo_atari_lstm.py:117-160: NatureCNN trunk over ONE grayscale frame, nn.LSTM(512, 128) with the state reset by
 * (1 - done) before every step (gate order i, f, g, o), actor / critic on the LSTM output.  bf16 operands, fp32
 * accumulation; the cell state and the gate math stay fp32.
 * params / grads: ONE flat fp32 vector in LSTMAgent._param_order (b200rl_lstm_agent_param_count(A) elements), 16-B aligned:
 *     conv1.w[32,1,8,8] conv1.b[32] conv2.w[64,32,4,4] conv2.b[64] conv3.w[64,64,3,3] conv3.b[64] fc.w[512,3136] fc.b[512]
 *     weight_ih[512,512] weight_hh[512,128] bias_ih[512] bias_hh[512] actor.w[A,128] critic.w[1,128] actor.b[A] critic.b[1]
 * packed : bf16 operand copies (b200rl_lstm_agent_bf16_packed_bytes), refreshed by b200rl_lstm_agent_bf16_pack after every
 *          optimiser step.
 * A sequence is S steps of n envs, time-major: batch row t*n + e is step t of env e (S*n rows, at most 131072).
 * obs    : uint8 frames [*, 1, 84, 84]; row i of the batch is frame rows[i] (rows i64 [S*n], may be NULL: frame i).
 * done   : f32 [S*n]: the state of row (t, e) is multiplied by (1 - done) before step t.
 * h0, c0 : f32 [n, 128] state before step 0; h_out, c_out f32 [n, 128] the state after step S-1 (the rollout calls the
 *          forward with S = 1 once per env step, carrying (h, c)).
 * acts   : activation workspace for (S, n) (b200rl_lstm_agent_bf16_acts_bytes), 256-B aligned, ZEROED once before its first
 *          use; the backward reads what the forward of the same (obs, rows, S, n, done) left there.
 * head_out [S*n, A+1] fp32 = [logits | value]; dhead [S*n, A+1] its gradient; grads = flat fp32 gradient (overwritten).
 * 1 <= A <= 23.  Bad pointers, alignment (rows: 8 B), A, S, n or S*n: B200RL_ERR_INVALID_ARGUMENT before any CUDA call.  No
 * host synchronisation or allocation: forward and backward may be captured in a CUDA graph. */
int64_t b200rl_lstm_agent_param_count(int A);
size_t b200rl_lstm_agent_bf16_packed_bytes(int A);
size_t b200rl_lstm_agent_bf16_acts_bytes(int64_t S, int64_t n);
/* Byte offsets of the tensors inside `acts` (M = S*n rows), written to offsets[B200RL_LSTM_ACTS_TENSORS] in this order:
 *   act1 bf16 [M,10,10,128] (conv1 output as 2x2 cells), m1 uint32 [M,400] (act1 > 0 bits), act2 bf16 [M,9,9,64], act3 bf16
 *   [M,7,7,64] (conv2 / conv3 outputs, channel-last), feats bf16 [M,512] (fc output,
 *   post-ReLU), m4 uint32 [M,16], gx f32 [M,512] (feats W_ih^T + b_ih), hseq bf16 [M,128] (h_t), hm bf16 [M,128] (the
 *   masked state h' entering step t), save f32 [M,5,128] (i, f, g, o, tanh c), cm f32 [M,128] (the masked cell state c'),
 *   dgates f32 [M,512] (backward), dfeats bf16 [M,512] (backward). */
#define B200RL_LSTM_ACTS_TENSORS 13
int b200rl_lstm_agent_bf16_acts_layout(int64_t S, int64_t n, int64_t* offsets);
size_t b200rl_lstm_agent_bf16_workspace_bytes(int64_t S, int64_t n, int A);
int b200rl_lstm_agent_bf16_pack(const float* params, int A, void* packed, void* stream);
int b200rl_lstm_agent_bf16_forward(const uint8_t* obs, const int64_t* rows, int64_t S, int64_t n, int A,
                                   const float* params, const void* packed, const float* h0, const float* c0,
                                   const float* done, void* acts, float* head_out, float* h_out, float* c_out, void* stream);
int b200rl_lstm_agent_bf16_backward(const uint8_t* obs, const int64_t* rows, int64_t S, int64_t n, int A,
                                    const float* params, const void* packed, const float* done, void* acts,
                                    const float* dhead, float* grads, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------ LSTM cell ---
 * Recurrent PPO agent (cleanrl/ppo_atari_lstm.py:117-160: nn.LSTM(512, 128), gate order i, f, g, o; the state is reset
 * by (1 - done) BEFORE the cell, :137-142).  The gate GEMMs are b200rl_linear_fwd_f32 calls (x W_ih^T + b_ih for all
 * steps at once, h' W_hh^T + b_hh per step); these are the elementwise parts, fp32, [n, H] row-major.
 *   mask_state : (h', c') = (1 - done[n]) * (h, c)
 *   cell_fwd   : gates_x, gates_h [n, 4H] -> h_out, c_out [n, H]; save [n, 5H] = (i, f, g, o, tanh c), may be NULL
 *   cell_bwd   : one BPTT step.  dh = dh_heads + (1 - done_next) * dh_rec_raw (dh_rec_raw = dgates_{t+1} W_hh, NULL at the
 *                last step), dc = dc_rec (NULL at the last step) + dh o (1 - tanh(c)^2); writes the pre-activation gate
 *                gradients dgates [n, 4H] and dc_rec_out = (1 - done) dc f for step t-1. */
int b200rl_lstm_mask_state_f32(const float* h, const float* c, const float* done, int64_t n, int H,
                               float* h_masked, float* c_masked, void* stream);
int b200rl_lstm_cell_fwd_f32(const float* gates_x, const float* gates_h, const float* c_masked, int64_t n, int H,
                             float* h_out, float* c_out, float* save, void* stream);
int b200rl_lstm_cell_bwd_f32(const float* dh_heads, const float* dh_rec_raw, const float* done_next, const float* dc_rec,
                             const float* save, const float* c_masked, const float* done, int64_t n, int H,
                             float* dgates, float* dc_rec_out, void* stream);

/* --------------------------------------------------------- DQN TD update ---
 * td_target = r + gamma * max_a' Q_target(s')[a'] * (1 - done); old = Q(s)[a]; loss = mean((td - old)^2)
 * (F.mse_loss, cleanrl/dqn_atari.py:220-224; huber = 1: smooth-L1) and dL/dQ [B, A] in one pass.
 *   q, q_target_next : f32 [B, A] (row strides ld_q, ld_qt); actions i64 [B]; rewards, dones f32 [B]
 *   dq f32 [B, A] out; stats f32 [2] out: td_loss, mean chosen Q (the two logged scalars, dqn_atari.py:227-228)
 * b200rl_argmax_f32: greedy action of the epsilon-greedy policy (dqn_atari.py:192-193), first maximum.
 */
size_t b200rl_dqn_td_loss_workspace_bytes(int64_t B);
int b200rl_dqn_td_loss_f32(const float* q, int64_t ld_q, const float* q_target_next, int64_t ld_qt,
                           const int64_t* actions, const float* rewards, const float* dones,
                           int64_t B, int A, double gamma, int huber,
                           float* dq, int64_t ld_dq, float* stats,
                           void* workspace, size_t workspace_bytes, void* stream);
int b200rl_argmax_f32(const float* q, int64_t ld_q, int64_t n, int A, int64_t* out, void* stream);

/* ------------------------------------------------------------- C51 heads ---
 * Distributional Q-learning (cleanrl/c51_atari.py).  logits f32 [n, A * n_atoms] (row stride ld) are the output of
 * Linear(512, A * n_atoms); action a owns columns [a * n_atoms, (a + 1) * n_atoms).  atoms f32 [n_atoms] is the
 * network's registered `atoms` buffer (linspace(v_min, v_max, n_atoms)); 2 <= n_atoms <= 256.
 *
 * b200rl_c51_act_f32: QNetwork.get_action(x, action) (c51_atari.py:131-138).  Per row: pmf = softmax over atoms for every
 *   action, q = sum(pmf * atoms); the action is the first maximum of q, or action_in[i] when action_in is not NULL.
 *   action_out i64 [n]; q_out f32 [n, A] and pmf_out f32 [n, n_atoms] (the chosen action's pmf) may be NULL.
 * b200rl_c51_loss_f32: the update's target + loss + head gradient (c51_atari.py:233-253) in one pass:
 *   next_pmf = target pmf of the target network's greedy action (next_logits), next_atoms = r + gamma * atoms * (1 - d)
 *   clamped to [v_min, v_max], categorical projection onto the atoms (index_add_ order: all lower, then all upper
 *   neighbours), loss = mean_i -sum_j target_ij * log(clamp(pmf_ij, 1e-5, 1 - 1e-5)) with pmf the online network's pmf
 *   of actions[i].  dlogits f32 [B, A * n_atoms] (row stride ld_d) = dloss/dlogits, zero outside each row's action.
 *   stats f32 [2] = losses/loss, losses/q_values (mean of sum(pmf * atoms) over the unclamped pmf).
 *   gamma, v_min, v_max are rounded to f32 as torch rounds Python scalars.  Fixed-order reductions: bitwise
 *   reproducible.  workspace: b200rl_c51_loss_workspace_bytes(B), 16-byte aligned.
 */
int b200rl_c51_act_f32(const float* logits, int64_t ld, const float* atoms, int64_t n, int A, int n_atoms,
                       const int64_t* action_in, int64_t* action_out, float* q_out, float* pmf_out, void* stream);
size_t b200rl_c51_loss_workspace_bytes(int64_t B);
int b200rl_c51_loss_f32(const float* logits, int64_t ld, const float* next_logits, int64_t ld_next,
                        const float* atoms, const int64_t* actions, const float* rewards, const float* dones,
                        int64_t B, int A, int n_atoms, double gamma, double v_min, double v_max,
                        float* dlogits, int64_t ld_d, float* stats,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------- discrete soft actor-critic ---
 * cleanrl/sac_atari.py on [n, A] head outputs (row strides ld*), 2 <= A <= 32.  The temperature is device memory:
 * alpha f32 [1]; with autotune also log_alpha f32 [1] and its Adam moments exp_avg, exp_avg_sq f32 [1].
 *
 * b200rl_sac_policy_f32: Actor.get_action's log_softmax (logp) and Categorical probabilities (probs) of the logits; either
 *   output may be NULL.  The sampled action is b200rl_categorical_sample_f32 on the same logits.
 * b200rl_sac_critic_loss_f32: the soft-Q target and both critic losses (sac_atari.py:274-290) in one pass:
 *   y = r + ((1 - d) * gamma) * sum_a p'(a) (min(q1t, q2t)(a) - alpha * logp'(a)), p' / logp' from the actor's logits on
 *   next_obs (next_logits); dq_k [B, A] = 2 (q_k[a] - y) / B at the taken action, 0 elsewhere; y f32 [B] may be NULL.
 *   stats f32 [4] = mean q1[a], mean q2[a], qf1_loss, qf2_loss.
 * b200rl_sac_actor_loss_f32: the actor loss and its gradient (sac_atari.py:293-305): f = alpha * logp - min(q1, q2),
 *   actor_loss = mean over B x A of p f, dlogits [B, A] = p (f - sum_a p f) / (B A).  With autotune (sac_atari.py:307-314)
 *   alpha_loss = mean(p (-exp(log_alpha) (logp + target_entropy))) and one Adam step of log_alpha (beta1, beta2, eps,
 *   step_scalars f32 [2] as b200rl_adam_step_scalars in device memory), then alpha = exp(log_alpha); every block reads the
 *   old alpha before it is rewritten.  stats f32 [4] = actor_loss, alpha_loss (0 without autotune), alpha, log_alpha.
 * Fixed-order reductions: bitwise reproducible.  workspace: the matching *_workspace_bytes(B), 16-byte aligned.
 */
int b200rl_sac_policy_f32(const float* logits, int64_t ld, int64_t n, int A, float* logp, int64_t ld_logp,
                          float* probs, int64_t ld_probs, void* stream);
size_t b200rl_sac_critic_loss_workspace_bytes(int64_t B);
int b200rl_sac_critic_loss_f32(const float* next_logits, int64_t ld_next, const float* q1_target, int64_t ld_q1t,
                               const float* q2_target, int64_t ld_q2t, const float* q1, int64_t ld_q1, const float* q2,
                               int64_t ld_q2, const int64_t* actions, const float* rewards, const float* dones,
                               const float* alpha, int64_t B, int A, double gamma, float* y, float* dq1, int64_t ld_dq1,
                               float* dq2, int64_t ld_dq2, float* stats, void* workspace, size_t workspace_bytes,
                               void* stream);
size_t b200rl_sac_actor_loss_workspace_bytes(int64_t B);
int b200rl_sac_actor_loss_f32(const float* logits, int64_t ld, const float* q1, int64_t ld_q1, const float* q2,
                              int64_t ld_q2, int64_t B, int A, float* alpha, int autotune, float* log_alpha,
                              float* exp_avg, float* exp_avg_sq, const float* step_scalars, double target_entropy,
                              double beta1, double beta2, double eps, float* dlogits, int64_t ld_d, float* stats,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------- continuous soft actor-critic ---
 * cleanrl/sac_continuous_action.py, fp32: SoftQNetwork [obs | act] -> 256 -> 256 -> 1 and Actor obs -> 256 -> 256 ->
 * fc_mean / fc_logstd (D each) with the tanh-Gaussian head.  Shapes: 1 <= B <= 8192, 1 <= act_dim (D) <= 32,
 * obs_dim + act_dim <= 1024; any other shape is B200RL_ERR_INVALID_ARGUMENT.  Parameters are flat f32 in nn.Module order
 * (fc1.weight, fc1.bias, fc2.weight, fc2.bias, then fc3 or fc_mean, fc_mean.bias, fc_logstd, fc_logstd.bias); the twin
 * critics are two such blocks net_stride floats apart (critic forward only: 0 = one network, q[0] alone).  Twin
 * outputs are [2, B] (net-major); kept activations are [2, B, 256] for the critics and [B, 256] for the actor.  Every reduction runs in a fixed order: bitwise repeatable.
 * Kernels with a row mean take workspace of b200rl_sacc_workspace_bytes(B) bytes, 16-byte aligned, zeroed once; one
 * buffer may serve all of them on one stream.  Temperature, Adam moments and step scalars live in device memory.
 *
 * Network kinds (``critic``): 0 = the tanh-Gaussian actor, 1 = a critic, 2 = the deterministic TD3 actor (one D-wide
 *   head fc_mu).
 * b200rl_sacc_param_count: floats in one network of that kind; -1 for a shape or kind outside the limits.
 * b200rl_sacc_critic_fwd_f32: q [2, B] of both critics on x = [obs[obs_rows] | act[act_rows]] (either rows vector
 *   (int64) may be NULL for rows 0..B-1); keep_x [B, K] and keep_h1 / keep_h2 (post-ReLU) may be NULL.
 * b200rl_sacc_actor_fwd_f32: Actor.get_action on obs[rows] with noise eps [B, D]: action [B, D], log_pi [B], squashed
 *   mean [B, D], mean_logstd [B, 2D] = Actor.forward's (mean, log_std), the kept x / h1 / h2 and raw head [B, 2D]
 *   (mean | raw log_std); each may be NULL.  With temperature != 0 it also takes the autotune step on these log_pi:
 *   alpha_loss = mean(-exp(log_alpha) (log_pi + target_entropy)), one Adam step of log_alpha (beta1, beta2, adam_eps,
 *   step_scalars f32 [2] as b200rl_adam_step_scalars), alpha = exp(log_alpha); stats[1..3] = alpha_loss, alpha, log_alpha.
 * min is torch.min's: NaN if either operand is NaN.
 * b200rl_sacc_critic_loss_f32: y = r + ((1 - d) gamma) (min(q_next[0], q_next[1]) - alpha next_logpi) with r / d read
 *   through rows (NULL: 0..B-1); dq [2, B] = 2 (q - y) / B; y may be NULL; stats[0..3] = mean q1, mean q2, qf1_loss,
 *   qf2_loss.  next_logpi NULL (TD3): no entropy term, y = r + ((1 - d) gamma) min(q_next[0], q_next[1]); alpha may then
 *   be NULL.
 * b200rl_sacc_critic_bwd_f32: data gradients through both critics.  Critic step: dq given, writes dz1 / dz2 [2, B, 256]
 *   (pre-activation gradients of fc1 / fc2).  Actor step: dq NULL, q [2, B] given; the gradient of -mean(min(q1, q2))
 *   (half to each at a tie, as autograd's min) is carried to the action columns only: dact [2, B, D], one per critic.
 *   Single-network actor step (TD3): net_stride 0, dq and q NULL; the gradient of -mean(q) of the one network goes to
 *   dact [B, D].
 * b200rl_sacc_actor_bwd_f32: actor_loss = mean(alpha log_pi - min(q[0], q[1])) back through the tanh-Gaussian head (raw
 *   head and eps of the forward, dact of the critics) to dhead [B, 2D] = (d mean, d raw log_std), then dz2 / dz1
 *   [B, 256]; stats[0] = actor_loss.
 * b200rl_sacc_wgrad_f32: weight and bias gradients of all three layers of both critics (critic 1: dz1 / dz2 [2, B,
 *   256], dout = dq [2, B], x [B, K], h1 / h2 [2, B, 256]), of the actor (critic 0: dout = dhead [B, 2D]) or of the TD3
 *   actor (critic 2: dout = dhead [B, D]) into grad (flat layout, overwritten), summed over rows in row order, no
 *   atomics.  Critic 1 with net_stride 0: one critic (DDPG), dz1 / dz2 / h1 / h2 [1, B, 256], dout = dq [B].
 * b200rl_sacc_soft_update_f32: dst = tau * src + (1 - tau) * dst, two products and one sum each rounded.
 *
 * cleanrl/td3_continuous_action.py's deterministic Actor (kind 2) on the same trunk, critics and limits:
 * b200rl_td3_actor_fwd_f32: Actor.forward on obs[rows]: mu [B, D] = tanh(z) scale + bias (two roundings), keep_y [B, D]
 *   = tanh(z), the kept x / h1 / h2; each may be NULL.  With eps [B, D] it also writes the smoothed target action
 *   smoothed [B, D] = (mu + (eps policy_noise).clamp(-noise_clip, noise_clip) scale).clamp(low, high) in that rounding
 *   order (eps and smoothed go together; low / high are scalars: the reference clamps to low[0] / high[0]).
 * b200rl_td3_actor_bwd_f32: actor_loss = -mean(q) (q [B] of qf1 on the actor's action, dact [B, D] its gradient from
 *   the single-network critic backward) back through the head: dhead [B, D] = (dact scale) (1 - y^2), then dz2 / dz1
 *   [B, 256]; stats[0] = actor_loss.  Workspace as above.
 *
 * cleanrl/ddpg_continuous_action.py: the TD3 actor and one critic (net_stride 0 everywhere), plus
 * b200rl_ddpg_critic_loss_bwd_f32: the one-critic step in one launch.  y = r + ((1 - d) gamma) q_next (r / d read
 *   through rows, NULL: 0..B-1; q_next [B] of the target critic), dq [B] = 2 (q - y) / B, then, as the critic step of
 *   b200rl_sacc_critic_bwd_f32, dz1 / dz2 [B, 256] from the critic's kept h1 / h2 [B, 256]; y may be NULL;
 *   stats[0..1] = mean q (qf1_values), qf1_loss.  Workspace as above.
 */
int64_t b200rl_sacc_param_count(int obs_dim, int act_dim, int critic);
size_t b200rl_sacc_workspace_bytes(int64_t B);
int b200rl_sacc_critic_fwd_f32(const float* params, int64_t net_stride, const float* obs, int64_t ld_obs,
                               const int64_t* obs_rows, const float* act, int64_t ld_act, const int64_t* act_rows,
                               int64_t B, int obs_dim, int act_dim, float* q, float* keep_x, float* keep_h1,
                               float* keep_h2, void* stream);
int b200rl_sacc_actor_fwd_f32(const float* params, const float* obs, int64_t ld_obs, const int64_t* rows, int64_t B,
                              int obs_dim, int act_dim, const float* eps, const float* scale, const float* bias,
                              float* action, float* log_pi, float* mean_out, float* mean_logstd, float* keep_x,
                              float* keep_h1, float* keep_h2, float* keep_head, int temperature, double target_entropy,
                              float* alpha, float* log_alpha, float* exp_avg, float* exp_avg_sq,
                              const float* step_scalars, double beta1, double beta2, double adam_eps, float* stats,
                              void* workspace, size_t workspace_bytes, void* stream);
int b200rl_sacc_critic_loss_f32(const float* q_next, const float* next_logpi, const float* q, const float* rewards,
                                const float* dones, int64_t ld_rd, const int64_t* rows, const float* alpha, int64_t B, double gamma,
                                float* y, float* dq, float* stats, void* workspace, size_t workspace_bytes, void* stream);
int b200rl_sacc_critic_bwd_f32(const float* params, int64_t net_stride, int64_t B, int obs_dim, int act_dim,
                               const float* dq, const float* q, const float* h1, const float* h2, float* dz1, float* dz2,
                               float* dact, void* stream);
int b200rl_sacc_actor_bwd_f32(const float* params, int64_t B, int obs_dim, int act_dim, const float* head,
                              const float* eps, const float* scale, const float* dact, const float* q,
                              const float* log_pi, const float* alpha, const float* h1, const float* h2, float* dhead,
                              float* dz1, float* dz2, float* stats, void* workspace, size_t workspace_bytes, void* stream);
int b200rl_sacc_wgrad_f32(int critic, int64_t B, int obs_dim, int act_dim, const float* x, const float* h1,
                          const float* h2, const float* dz1, const float* dz2, const float* dout, float* grad,
                          int64_t net_stride, void* stream);
int b200rl_sacc_soft_update_f32(const float* src, float* dst, int64_t n, double tau, void* stream);
int b200rl_td3_actor_fwd_f32(const float* params, const float* obs, int64_t ld_obs, const int64_t* rows, int64_t B,
                             int obs_dim, int act_dim, const float* scale, const float* bias, float* mu, float* keep_y,
                             float* keep_x, float* keep_h1, float* keep_h2, const float* eps, double policy_noise,
                             double noise_clip, double low, double high, float* smoothed, void* stream);
int b200rl_td3_actor_bwd_f32(const float* params, int64_t B, int obs_dim, int act_dim, const float* y,
                             const float* scale, const float* dact, const float* q, const float* h1, const float* h2,
                             float* dhead, float* dz1, float* dz2, float* stats, void* workspace,
                             size_t workspace_bytes, void* stream);
int b200rl_ddpg_critic_loss_bwd_f32(const float* params, int64_t B, int obs_dim, int act_dim, const float* q_next,
                                    const float* q, const float* rewards, const float* dones, int64_t ld_rd,
                                    const int64_t* rows, double gamma, const float* h1, const float* h2, float* y,
                                    float* dq, float* dz1, float* dz2, float* stats, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------ parallel Q-learning ---
 * cleanrl/pqn.py, fp32: QNetwork obs (obs_dim) -> Linear 120 -> LayerNorm -> ReLU -> Linear 84 -> LayerNorm -> ReLU ->
 * Linear A.  Shapes: 1 <= obs_dim <= 512, 2 <= A <= 64; any other shape is B200RL_ERR_INVALID_ARGUMENT.  Parameters are
 * flat f32 in nn.Module order (network.0.weight [120, obs_dim], network.0.bias, network.1.weight / .bias (LN1 gamma /
 * beta), network.3.*, network.4.*, network.6.weight [A, 84], network.6.bias).  obs rows have stride ld_obs floats.
 * Every reduction runs in a fixed order: bitwise repeatable.
 *
 * b200rl_pqn_param_count: floats in the network; -1 for a shape outside the limits.
 * b200rl_pqn_act_f32: the rollout step (pqn.py:180-189) on n rows: Q, max_action = argmax Q (first maximum; a NaN counts
 *   as the maximum), values_slot [n] = Q[max_action].  With random_actions i64 [n] and u f32 [n] (the step's CPU draws,
 *   together or neither) actions_slot i64 [n] = u < eps ? random_actions : max_action, eps rounded to f32 as torch's
 *   `tensor < python_float` rounds it; without them actions_slot (may then be NULL) = max_action, and values_slot is
 *   the greedy bootstrap max Q (pqn.py:209).  obs_slot [n, obs_dim] (dense) may be NULL: a copy of the rows.  The same
 *   launch copies copy_n floats copy_in -> copy_out (the step's done / reward bookkeeping; copy_n 0: none).
 * b200rl_pqn_forward_f32: Q values q [n, A] (QNetwork.forward).
 * b200rl_pqn_loss_bwd_f32: one minibatch (pqn.py:233-238): rows obs[mb_inds] (NULL: 0..M-1), q = Q[b_actions[mb_inds]],
 *   loss = mean((b_returns[mb_inds] - q)^2), dq = F.mse_loss's backward for its target argument, and the data backward
 *   through the head, LN2 + ReLU and LN1 + ReLU (dz = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat))).  It keeps in
 *   the workspace what the weight gradient reads; stats f32 [2] = td_loss, mean(q).
 * b200rl_pqn_wgrad_f32: every weight, bias, gamma and beta gradient of that minibatch into grad (flat layout,
 *   overwritten) from the workspace loss_bwd left, summed over rows in row order, no atomics.  Same obs / mb_inds /
 *   b_actions / M as the loss_bwd call before it.
 * Workspace: b200rl_pqn_workspace_bytes(M) bytes, 16-byte aligned, zeroed once; it serves a loss_bwd and the wgrad
 *   after it, and any smaller M.
 * b200rl_qlambda_f32: Q(lambda) returns (pqn.py:205-218) over rewards / values / dones f32 [T, N], next_value /
 *   next_done f32 [N] into returns [T, N].  One thread per env, every operation separately rounded: bit-identical to the
 *   reference loop.  gamma, q_lambda and 1 - q_lambda (in double) round to f32; the last step is
 *   r + ((gamma nv) (1 - next_done)), the others r + ((gamma ((ql R') + ((1 - ql) v'))) (1 - d')).
 */
int64_t b200rl_pqn_param_count(int obs_dim, int A);
size_t b200rl_pqn_workspace_bytes(int64_t M);
int b200rl_pqn_act_f32(const float* params, const float* obs, int64_t ld_obs, int64_t n, int obs_dim, int A,
                       const int64_t* random_actions, const float* u, double eps, float* obs_slot,
                       int64_t* actions_slot, float* values_slot, const float* copy_in, float* copy_out,
                       int64_t copy_n, void* stream);
int b200rl_pqn_forward_f32(const float* params, const float* obs, int64_t ld_obs, int64_t n, int obs_dim, int A,
                           float* q, void* stream);
int b200rl_pqn_loss_bwd_f32(const float* params, const float* obs, int64_t ld_obs, const int64_t* mb_inds,
                            const int64_t* b_actions, const float* b_returns, int64_t M, int obs_dim, int A,
                            float* stats, void* workspace, size_t workspace_bytes, void* stream);
int b200rl_pqn_wgrad_f32(const float* obs, int64_t ld_obs, const int64_t* mb_inds, const int64_t* b_actions, int64_t M,
                         int obs_dim, int A, const void* workspace, size_t workspace_bytes, float* grad, void* stream);
int b200rl_qlambda_f32(const float* rewards, const float* values, const float* dones, const float* next_value,
                       const float* next_done, float* returns, int64_t T, int64_t N, double gamma, double q_lambda,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H */
