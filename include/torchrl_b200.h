/* torchrl_b200.h -- C ABI of libtorchrl_b200.so (sm_90a kernels for the torchrl hot path).
 *
 * The reference (RchalYang/torchrl, pure Python) has no FFI of its own; these are the
 * entry points a ctypes binding of the reference would call in place of the Python/NumPy
 * code cited beside each declaration (paths relative to the reference root).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller owns
 *     all memory (nothing is allocated or retained by the library);
 *   - arrays are dense, row-major, time-major: (T, N, D) with the env index N contiguous
 *     over D -- the layout of the reference's buffers (replay_buffers/base.py:19-29);
 *   - float data are fp32; 0/1 flags (terminals, time_limits) are uint8;
 *   - `stream` is a cudaStream_t passed as void*; launches are asynchronous, no host sync;
 *   - return value: 0 = ok, <0 = argument error (TRL_E*), >0 = cudaError_t of the launch;
 *     trl_last_error() returns the message of the calling thread's last failure.
 *
 * This header is the one statement of the ABI: every kernel source is compiled against it, and the Python
 * binding (torchrl_b200/_lib.py) reads each entry point's types from it.  The binding accepts declarations of the
 * form `ret trl_name(type name, ...);` (block comments anywhere) with ret int, int64_t or const char*, scalar
 * parameters int, int64_t, unsigned, uint64_t, float or double, and pointers to those, to uint8_t, int32_t or void.
 */
#ifndef TORCHRL_B200_H
#define TORCHRL_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TRL_OK 0
#define TRL_EINVAL (-1)
#define TRL_EALIGN (-2)
#define TRL_EUNSUPPORTED (-3)

const char* trl_last_error(void);
int trl_abi_version(void);
int trl_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* K6 -- replaces OnPolicyReplayBufferBase.generalized_advantage_estimation
 * (torchrl/replay_buffers/on_policy.py:16-44).  variant: 1 = auto (default),
 * 0 = serial-in-T reference-shaped kernel, 2 = force 4-env vectorised, 3 = force scalar. */
int trl_gae_scan(const float* rewards, const float* values, const uint8_t* terminals,
                 const uint8_t* time_limits, const float* last_value, float* advs, float* returns,
                 int64_t T, int64_t N, float gamma, float tau, int time_limit_filter, int variant,
                 void* stream);

/* K6 -- replaces OnPolicyReplayBufferBase.discount_reward (torchrl/replay_buffers/on_policy.py:46-70). */
int trl_discount_return(const float* rewards, const float* values, const uint8_t* terminals,
                        const uint8_t* time_limits, const float* last_value, float* advs, float* returns,
                        int64_t T, int64_t N, float gamma, int time_limit_filter, int variant,
                        void* stream);

/* ---- K1: batched synthetic env (dynamics defined by this build, oracle/synth_env.py) ------------
 * trl_synth_env_step replaces VecEnv.step / SubProcVecEnv.step (torchrl/env/vecenv.py:53-61,
 * subproc_vecenv.py:123-140) with the per-env wrapper chain NormAct.action
 * (env/continuous_wrapper.py:18-20), RewardShift.reward (env/base_wrapper.py:37-41) and
 * TimeLimitAugment.step (env/base_wrapper.py:152-156) fused in, and accumulates the batch moments
 * of Normalizer.update_estimate (env/base_wrapper.py:75-82; merged in-kernel when merge_stats=1).
 * `state` (N,o) is updated in place and IS the raw observation. */
int trl_synth_env_smem_bytes(int obs_dim, int act_dim);
int trl_synth_env_num_ctas(int64_t N);
int trl_synth_env_step(float* state, const float* actions, const float* A, const float* B, const float* c,
                       const float* lb, const float* ub, int* elapsed, const int* step_count, float* reward,
                       uint8_t* done, uint8_t* time_limit, double* partial, double* batch_sums,
                       double* norm_mean, double* norm_var, double* norm_count, unsigned* ticket,
                       int* any_reset, const int* t_ptr, int64_t N, int obs_dim, int act_dim, float rho,
                       float eta, float ctrl_cost, float term_thr, float reward_scale, int max_episode_steps,
                       int max_episode_frames, int merge_stats, void* stream);
/* VecEnv.reset / partial_reset (env/vecenv.py:42-51): mask NULL = all envs. */
int trl_synth_env_reset(float* state, int* elapsed, unsigned* episode, const unsigned* seeds,
                        const uint8_t* mask, int64_t N, int obs_dim, double init_scale, void* stream);
/* VecEnv.seed (env/vecenv.py:63-65): env i gets seed*n_total + first_env + i. */
int trl_synth_env_seed(unsigned* seeds, unsigned* episode, int64_t N, unsigned seed, unsigned n_total,
                       unsigned first_env, void* stream);

/* ---- K2: observation normaliser (env/base_wrapper.py:44-60, 63-94, 103-121) ------------------- */
int trl_obs_norm_moments(const float* x, int64_t N, int obs_dim, double* sums, void* stream);
int trl_obs_norm_merge(const double* sums, double batch_n, int obs_dim, double* mean, double* var,
                       double* count, void* stream);
int trl_obs_norm_filt(const float* raw, const double* mean, const double* var, int64_t N, int obs_dim,
                      double clip, float* out, void* stream);

/* ---- K3: tanh-Gaussian action sampling (policies/continuous_policy.py:92-132,
 * policies/distribution.py:60-76 rsample, :33-45 log_prob).  eps NULL -> in-kernel Philox noise. */
int trl_tanh_gaussian_sample(const float* mean, const float* log_std, int ls_stride, const float* eps,
                             float noise_scale, uint64_t seed, const uint64_t* rng_counter, int64_t M,
                             int act_dim, int tanh_action, float* action, float* pre_tanh, float* log_prob,
                             float* eps_out, int* nan_flag, void* stream);
int trl_tanh_gaussian_sample_bwd(const float* action, const float* eps, const float* log_std, int ls_stride,
                                 const float* g_action, const float* g_logp, int64_t M, int act_dim,
                                 int tanh_action, float* g_mean, float* g_log_std, void* stream);

/* ---- K4/K5: per-step rollout store + timeout bootstrap + partial reset
 * (collector/on_policy.py:115-153, collector/base.py:204-228, replay_buffers/base.py:19-37).
 * state/elapsed/episode/seeds all NULL = host envs behind the pinned-memory bridge (SURVEY 8(f).1): rows are
 * stored and counters updated, the masked reset itself is done by the host env afterwards. */
int trl_collect_finalize(const float* cur_ob_in, const float* next_norm, float* state, const float* act,
                         const float* value, const float* v_next, const float* reward, const uint8_t* done,
                         const uint8_t* tl, int* elapsed, unsigned* episode, const unsigned* seeds,
                         int* step_count, double* ep_return, double* epoch_reward, float* ret_log,
                         int* n_done, const int* any_reset, const double* norm_mean, const double* norm_var,
                         float* cur_ob_out, float* b_obs, float* b_next_obs, float* b_acts, float* b_values,
                         float* b_rewards, uint8_t* b_terminals, uint8_t* b_time_limits, const int* t_ptr,
                         int64_t N, int obs_dim, int act_dim, int max_episode_frames, float discount,
                         double init_scale, double clip, int terminal_includes_surpass,
                         int raw_obs_after_reset, void* stream);
/* BaseReplayBuffer._advance (replay_buffers/base.py:33-37) on device-side counters. */
int trl_step_advance(int* t_ptr, int T, int* size_ptr, uint64_t* rng_counter, void* stream);

/* ---- K7/K9/K4: time-row gather / ring write (replay_buffers/on_policy.py:72-91, base.py:19-51).
 * src/dst/row_bytes are HOST arrays of nkeys entries holding device pointers / byte counts. */
int trl_row_gather(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                   const int64_t* idx, const int* pos_ptr, int rows, void* stream);
int trl_ring_write(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                   const int* row_ptr, void* stream);
/* trl_ring_write + trl_step_advance(row_ptr, T, size_ptr) in one launch (the last CTA to finish advances the index);
 * ticket: one unsigned, zero-initialised once by the caller. */
int trl_ring_write_advance(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                           int* row_ptr, int T, int* size_ptr, unsigned* ticket, void* stream);
/* mean, unbiased std, max, min of a vector (algo/on_policy/ppo.py:141-147). */
int trl_vec_stats(const float* x, int64_t n, float* stats4, void* stream);
/* K12: the same statistics over the union of all ranks' minibatches: local raw moments [sum, sumsq, max, -min]
 * (fp64) -> one all-gather -> combine. */
int trl_vec_moments(const float* x, int64_t n, double* moments4, void* stream);
/* All minibatches of an epoch at once: moments4 (groups,4) = sum, sum of squares, max, -min of the rows
 * idx[u*b .. (u+1)*b) of x; stats4 (groups,4) = mean, unbiased std, max, min from `world` ranks' moments. */
int trl_row_group_moments(const float* x, const int64_t* idx, int groups, int b, int64_t row_elems,
                          double* moments4, void* stream);
int trl_group_stats_from_moments(const double* gathered, int world, int groups, double n_total, float* stats4,
                                 void* stream);
int trl_vec_stats_from_moments(const double* gathered, int world, double n_total, float* stats4, void* stream);

/* ---- K8: PPO losses, value + gradient wrt the network outputs (algo/on_policy/ppo.py:41-122). */
int64_t trl_ppo_actor_scratch_doubles(int64_t B, int act_dim);
/* old_logp == NULL: the plain policy-gradient loss of A2C, L = -mean(logp * adv) - c_ent * mean(ent)
 * (algo/on_policy/a2c.py:66-70), same outputs.
 * ls_min <= ls_max: log_std is the RAW parameter; torch.clamp(log_std, ls_min, ls_max) of
 * GuassianContPolicyBasicBias.forward (policies/continuous_policy.py:173-188) is applied inside, and g_log_std is the
 * gradient with respect to the raw parameter (zero where the clamp is active).  ls_min > ls_max: no clamp. */
int trl_ppo_actor_loss(const float* mean, const float* log_std, int ls_stride, const float* actions,
                       const float* old_logp, const float* advs, const float* adv_stats,
                       const int* adv_stats_pos /* device scalar: row (of 4 floats) of adv_stats to use; NULL: row 0 */,
                       int64_t B,
                       int act_dim, int tanh_action, float clip_para, float entropy_coeff, float ls_min, float ls_max,
                       float* g_mean, float* g_log_std, float* logp_out, float* info16, double* scratch, unsigned* ticket,
                       void* stream);
int trl_ppo_critic_loss(const float* values, const float* returns, const float* old_values, int64_t B,
                        int clipped, float clip_para, float* g_values, float* info1, double* scratch,
                        unsigned* ticket, void* stream);
/* log pi(a|s) of stored actions (policies/continuous_policy.py:134-153). */
int trl_gaussian_log_prob(const float* mean, const float* log_std, int ls_stride, const float* actions,
                          int64_t B, int act_dim, int tanh_action, float* logp, void* stream);

/* ---- K13: categorical distribution of the discrete on-policy path (csrc/categorical.cu), torch's
 * Categorical(probs=softmax(logits)): CategoricalDisPolicy.explore / update (policies/discrete_policies.py:123-160).
 * Logits (M, A) row-major, 1 <= A <= 32; actions are indices stored as float.
 * Sampling by inverse CDF over p with one uniform per row: u (M) given, or (u NULL) Philox4x32-10 keyed by
 * (seed, *rng_counter, row).  Rows with a non-finite logit set *nan_flag (may be NULL) and get action 0. */
int trl_categorical_sample(const float* logits, const float* u, uint64_t seed, const uint64_t* rng_counter, int64_t M,
                           int num_actions, float* action, float* log_prob, int* nan_flag, void* stream);
/* log pi(a|s) of stored actions, log(clamp(p_a, eps, 1-eps)) (the old log-probs of PPO, ppo.py:54-56). */
int trl_categorical_log_prob(const float* logits, const float* actions, int64_t M, int num_actions, float* logp,
                             void* stream);
int64_t trl_ppo_categorical_actor_scratch_doubles(int64_t B);
/* trl_ppo_actor_loss for a categorical policy (ppo.py:41-91 / a2c.py:66-70): old_logp NULL = A2C's plain policy
 * gradient; writes dL/dlogits (B, A) and the same info16 slots (the log-std slots 7-10 are zero). */
int trl_ppo_categorical_actor_loss(const float* logits, const float* actions, const float* old_logp, const float* advs,
                                   const float* adv_stats, const int* adv_stats_pos, int64_t B, int num_actions,
                                   float clip_para, float entropy_coeff, float* g_logits, float* logp_out,
                                   float* info16, double* scratch, unsigned* ticket, void* stream);
/* V-MPO's top-half selection (algo/on_policy/v_mpo.py:65-71: torch.sort(advs, descending) then idx.chunk(2)[0]) for
 * `groups` minibatches in one launch.  Minibatch u is the time rows perm[u*b .. (u+1)*b) x row_elems envs in
 * trl_row_gather order (perm NULL: rows 0..b-1, the explicit vector of eager updates); its B = b * row_elems
 * advantages are normalised with stats4 row u, advn = (adv - mean) / (std + 1e-5), and the positions of the
 * k = B - B/2 largest (ties: the lower position first) are written to sel (groups, k) in ascending order.
 * 1 <= B < 2^31. */
int trl_vmpo_select(const float* advs, const int64_t* perm, int groups, int b, int64_t row_elems, const float* stats4,
                    int64_t* sel, void* stream);
int64_t trl_vmpo_categorical_scratch_doubles(int64_t k);
/* V-MPO's actor loss for a categorical policy on the k selected rows (v_mpo.py:73-99 with
 * CategoricalDisPolicy.update, policies/discrete_policies.py:156-167 and torch's categorical KL):
 * phi = softmax(advn / eta), L = mean(-phi * logp) + alpha * K + eta * eta_eps + eta * log(mean(exp(advn / eta)))
 * + alpha * alpha_eps - alpha * K, with K = sum_i KL_i (per_row_kl = 0: the reference's summed KL) or mean_i KL_i
 * (per_row_kl = 1).  dual (2) = [eta, alpha] on the device.  Writes dL/dlogits (k, A), g_dual (2) = [dL/deta,
 * dL/dalpha] and info12 = [policy_loss, alpha_loss, -, -, logprob mean, std, max, min, KL mean, std, max, min]
 * (the summed KL logs K, NaN, K, K).  The log-mean-exp subtracts the maximum. */
int trl_vmpo_categorical_loss(const float* logits, const float* target_logits, const float* actions,
                              const float* advs, const float* adv_stats, const int* adv_stats_pos, const float* dual,
                              int64_t k, int num_actions, float eta_eps, float alpha_eps, int per_row_kl,
                              float* g_logits, float* g_dual, float* info12, double* scratch, unsigned* ticket,
                              void* stream);
/* TRPO's Fisher-vector product in logit space (algo/on_policy/trpo.py:29-86, the KL over probs of trpo.py:53-61):
 * per row g = scale * (p * t - p <p, t>) with p = softmax(logits) (maximum subtracted) and t (M, A) the tangent of the
 * logits along the parameter direction, J v.  This is the Hessian of the reference's KL at theta0 applied to J v,
 * without its O(1e-8) terms (DESIGN §6 deviation 20); the caller back-propagates g through the logits.  M >= 0. */
int trl_categorical_fisher_vp(const float* logits, const float* tangent, int64_t M, int num_actions, float scale,
                              float* g_logits, void* stream);
/* The bias and activation step of TRPO's tangent forward pass (replaces the elementwise part of trpo.py:65-86's
 * double backward), in place over (M, C, S) -- NCHW conv outputs (S = H * W) or (M, H) linear outputs (S = 1):
 * t <- (t + bias_tangent[c]) * act'(y), act'(y) = 1 - y*y (act 1, tanh), y > 0 (act 2, ReLU) or 1 (act 0, y may be
 * NULL), from the cached layer output y; each operation rounded on its own, as torch evaluates it. */
int trl_tangent_bias_act(float* t, const float* bias_tangent, const float* y, int64_t M, int C, int64_t S, int act,
                         void* stream);
/* TRPO's line-search score of one candidate (trpo.py:113-129): out[0] = -mean(exp(logp - logp_old) * advn), logp
 * as trl_categorical_log_prob; deterministic fp64 sum, one launch.  scratch: ceil(M / 256) doubles; ticket zeroed
 * once. */
int trl_categorical_surrogate(const float* logits, const float* actions, const float* logp_old, const float* advn,
                              int64_t M, int num_actions, float* out, double* scratch, unsigned* ticket, void* stream);

/* ---- K11: flat-buffer grad-norm clip + Adam, Polyak (algo/utils.py:16-25, ppo.py:72-74,117-119). */
int trl_grad_sumsq_blocks(int nseg);
int trl_grad_sumsq(const float* grad, const int64_t* seg_begin_host, int nseg, unsigned active_mask,
                   double* sumsq3_out, int* step_counts, double beta1, double beta2, double* scratch,
                   unsigned* ticket, void* stream);
int trl_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, const int64_t* seg_begin_host,
                  int nseg, unsigned active_mask, const double* sumsq3, const float* lr_dev,
                  const float* max_norm_host, const float* eps_host, float beta1, float beta2,
                  float grad_scale, int zero_grad, float* param_hi, float* param_lo, void* stream);
/* param_hi / param_lo, target_hi / target_lo (both or neither): TF32 planes hi = tf32(w), lo = w - hi of the
 * updated weights, kept current for trl_gemm3_pair's pre-split B operand. */
int trl_polyak_update(float* target, const float* source, int64_t n, float tau, float* target_hi,
                      float* target_lo, void* stream);

/* ---- K10: off-policy TD targets and loss reductions.
 * TwinSACQ.update (algo/off_policy/twin_sac_q.py:84-219), TD3.update (algo/off_policy/td3.py:57-154),
 * QRDQN.update (algo/off_policy/qrdqn.py:22-74) + quantile_regression_loss/huber (algo/utils.py:5-13),
 * DQN.update (algo/off_policy/dqn.py:38-74). */
int64_t trl_offpolicy_scratch_doubles(int64_t B);
/* y = r + (1-d)*gamma*(min(q1',q2') - alpha*logpi')   (logp_next NULL -> TD3 form; q2_next NULL -> one critic) */
int trl_td_target(const float* rewards, const uint8_t* terminals, const float* q1_next, const float* q2_next,
                  const float* logp_next, const float* log_alpha, float fixed_alpha, float gamma, int64_t B,
                  float* y, float* info1, double* scratch, unsigned* ticket, void* stream);
/* a' = clamp(a + clamp(sigma*eps, +-c), +-1); eps NULL -> Philox noise   (td3.py:75-84) */
int trl_td3_smooth_action(const float* action, const float* eps, float sigma, float noise_clip, uint64_t seed,
                          const uint64_t* rng_counter, int64_t n, float* out, void* stream);
/* alpha loss + its one-parameter Adam step (twin_sac_q.py:111-123); info2 = [alpha, alpha_loss] */
int trl_sac_alpha_step(const float* logp, float target_entropy, float* log_alpha, float* adam_state3, float lr,
                       float beta1, float beta2, float eps, int64_t B, float* info2, double* scratch,
                       unsigned* ticket, void* stream);
/* mean(alpha*logpi - min(q1,q2)) and its gradients (twin_sac_q.py:145-153); info5 = [loss, logp mean/std/max/min] */
int trl_sac_policy_loss(const float* logp, const float* q1, const float* q2, const float* log_alpha,
                        float fixed_alpha, int64_t B, float* g_logp, float* g_q1, float* g_q2, float* info5,
                        double* scratch, unsigned* ticket, void* stream);
/* SAC / TwinSAC with a V network (sac.py:128-144, twin_sac.py:138-156): value target min(qn1,qn2) - alpha*logpi
 * (qn2 NULL -> one critic), value MSE and the policy loss (reparameterised: mean(alpha*logpi - min q); otherwise
 * mean(logpi * (alpha*logpi - (min q - v)).detach()), g_qn = 0) with their gradients;
 * info6 = [policy_loss, vf_loss, logp mean/std/max/min] */
int trl_sac_v_loss(const float* logp, const float* qn1, const float* qn2, const float* v_pred, const float* log_alpha,
                   float fixed_alpha, int reparameterization, int64_t B, float* g_logp, float* g_qn1, float* g_qn2,
                   float* g_v, float* info6, double* scratch, unsigned* ticket, void* stream);
/* MSE of one or two critics against the same target (twin_sac_q.py:142-143, td3.py:96-97) */
int trl_twin_mse_loss(const float* q1, const float* q2, const float* y, int64_t B, float* g1, float* g2,
                      float* info2, double* scratch, unsigned* ticket, void* stream);
/* The same with importance weights (prioritised replay; no reference counterpart): loss_k = mean_b w_b (q_k - y)^2,
 * g_k = ((2 (q_k - y)) w_b) / B, td_out (B, 1 or 2 critics) = the unweighted |q_k - y|.  weights and td_out may be
 * NULL; weights NULL gives trl_twin_mse_loss's bits. */
int trl_twin_mse_loss_weighted(const float* q1, const float* q2, const float* y, const float* weights, int64_t B,
                               float* g1, float* g2, float* td_out, float* info2, double* scratch, unsigned* ticket,
                               void* stream);
/* fused QR-DQN / DQN loss incl. greedy target selection; info3 = [loss, mean q_s_a, mean reward] */
int trl_qr_dqn_loss(const float* pred, const float* next, const float* actions, const float* rewards,
                    const uint8_t* terminals, const float* weights, int B, int n_actions, int n_quantiles,
                    float gamma, float kappa, int mse, float* grad, float* td_out, float* info3, double* scratch,
                    unsigned* ticket, void* stream);   /* weights / td_out: prioritised replay (may be NULL) */

/* ---- Bootstrapped DQN (csrc/bootstrapped.cu): BootstrappedDQN.update (algo/off_policy/bootstrapped_dqn.py:66-113).
 * pred / next (H, B, A): all heads of the network and of its target; actions (B) as float; masks (B, H) uint8.
 * Per head y_h = r + gamma*(1-d)*max_a' next[h, b, a'];  loss = sum_{b,h} m_bh (pred[h, b, a_b] - y_h)^2 / (H B).
 * grad (H, B, A) is written completely: 2 m_bh (pred - y_h) / (H B) at the taken action, 0 elsewhere.
 * info3 = [loss, mean over (b, h) of pred[h, b, a_b], mean reward].  scratch: trl_offpolicy_scratch_doubles(B). */
int trl_bootstrapped_dqn_loss(const float* pred, const float* next, const float* actions, const float* rewards,
                              const uint8_t* terminals, const uint8_t* masks, int64_t B, int num_heads,
                              int num_actions, float gamma, float* grad, float* info3, double* scratch,
                              unsigned* ticket, void* stream);
/* The collector's per-step decision for N envs (bootstrapped_dqn.py:22-62, policies/discrete_policies.py:92-115):
 * where current_step[n] == 0 a new head[n] = min(floor(u * H), H - 1); action[n] = the first argmax_a of
 * q_all[head[n], n, a] (q_all (H, N, A)); masks_ring[*top, n, j] = (u_j < bernoulli_p) -- no other ring row is touched.
 * Uniforms: u_head (N) and u_mask (N, H), or (both NULL) Philox4x32-10 keyed by (seed, *rng_counter, n); then the call
 * itself advances *rng_counter by one (ticket: a zero-initialised uint32 the caller owns). */
int trl_bootstrapped_act(const float* q_all, const int* current_step, int* head, float* action, uint8_t* masks_ring,
                         const int* top, const float* u_head, const float* u_mask, uint64_t seed,
                         uint64_t* rng_counter, unsigned* ticket, int64_t N, int num_heads, int num_actions,
                         float bernoulli_p, void* stream);

/* ---- MLP epilogues around the cuBLAS GEMMs of MLPBase (networks/base.py:24-44): z <- act(z + b) in place
 * (act: 0 none, 1 tanh, 2 relu) and its backward g_pre = g * act'(out), dbias = column sums (one launch each). */
int64_t trl_bias_act_bwd_scratch_floats(int64_t M, int H);
int trl_bias_act_fwd(float* z, const float* bias, int64_t M, int H, int act, void* stream);
int trl_bias_act_bwd(const float* grad, const float* out, float* grad_pre, float* dbias, int64_t M, int H,
                     int act, float* scratch, unsigned* tickets, void* stream);
/* x = hi + lo, hi = tf32(x): operand split of the error-compensated 3xTF32 tensor-core GEMM (opt-in). */
int trl_split_tf32(const float* x, int64_t n, float* hi, float* lo, void* stream);

/* ---- K9 (prioritised variant): proportional prioritised sampling of replay time rows.
 * PARITY UNPINNED -- the reference has no prioritised replay (SURVEY.md fact 7); the row-granular
 * definition follows BaseReplayBuffer.random_batch (replay_buffers/base.py:39-51) and is restated in
 * oracle/ref_numpy.py:per_sample/per_update.  u: device doubles in [0,1) (host np.random for parity). */
int trl_per_sample(const float* prio, int size, const double* u, int b, float beta, int64_t* idx,
                   float* weights, void* stream);
/* The same draw for rings of up to 2^24 rows, graph-safe: the live size is *size_ptr (clamped to 1..capacity) and
 * the uniforms are u[*pos_ptr * b ..][0..b), both read on the device.  Two launches (a scan per chunk of 4096 rows,
 * then one CTA over the chunk totals and the draws); for *size_ptr <= 4096 the bits are trl_per_sample's.
 * scratch: trl_per_scratch_doubles(capacity) doubles (-1: capacity not in 1..2^24). */
int trl_per_scratch_doubles(int capacity);
int trl_per_sample_rows(const float* prio, int capacity, const int* size_ptr, const double* u, const int* pos_ptr,
                        int b, float beta, int64_t* idx, float* weights, double* scratch, void* stream);
/* prio[idx_k] = (mean_n |td[k][n]| + eps)^alpha; a row drawn twice keeps its last draw's value (batch order) */
int trl_per_update(float* prio, const int64_t* idx, const float* td, int b, int n, float alpha, float eps,
                   float* max_prio, void* stream);
int trl_per_insert(float* prio, const int* row_ptr, const float* max_prio, void* stream);

/* ---- frame-de-duplicated pixel replay (csrc/frames.cu): the device layout of LazyFrames + MemoryEfficientReplayBuffer
 * (env/atari_wrapper.py:142-168, replay_buffers/memory_efficient_replay_buffer.py:5-33).  The ring keeps the newest
 * frame of obs and of next_obs per (row, env) + an age byte; stacks are rebuilt (as float32 * scale) at gather time. */
int trl_frame_ring_write(const uint8_t* stack, uint8_t* ring, uint8_t* age_ring, const int* elapsed, uint8_t* hist,
                         int* hist_count, const int* top, const int* size, int64_t N, int C, int64_t F, int T, int frame,
                         void* stream);
int trl_frame_hist_advance(int* hist_count, const int* size, int T, void* stream);
int trl_frame_stack_gather(const uint8_t* obs_last, const uint8_t* next_last, const uint8_t* age, const uint8_t* hist,
                           const int* hist_count, const int64_t* idx, const int* pos, int rows, const int* top,
                           const int* size, int64_t N, int C, int64_t F, int T, float scale, float* out_obs,
                           float* out_next, void* stream);

/* ---- K12: one-shot all-reduce over NVLink peer memory (csrc/comm.cu; no reference counterpart, SURVEY.md 8(e)).
 * Communication buffers are cudaMalloc blocks of their own (cudaIpc needs that): the ONLY allocations this library
 * makes.  peer_data / peer_flags: host arrays of `world` device pointers, entry r = rank r's operand buffer / flag
 * pad (trl_comm_flag_bytes() bytes, zero-initialised) as mapped in THIS process (own entries = local pointers).
 * `seq`: device uint32 of the communicator, starts at 0, bumped by every call; all ranks must issue the same calls in
 * the same order.  Sums run in rank order: every rank obtains the bit-identical result. */
int trl_comm_flag_bytes(void);
int trl_comm_ipc_handle_bytes(void);
int trl_comm_alloc(int64_t bytes, void** ptr_out);
int trl_comm_free(void* ptr);
int trl_comm_ipc_get(void* ptr, void* handle_out);
int trl_comm_ipc_open(const void* handle, void** ptr_out);
int trl_comm_ipc_close(void* ptr);
int trl_comm_scratch_doubles(int nseg);
/* out (n) = sum over ranks of the flat gradient + what trl_grad_sumsq computes for `out` (per-segment sum of squares,
 * Adam step counts, bias corrections): the all-reduce before clip_grad_norm_ of ppo.py:72,117 and the norm itself in
 * one kernel.  zero_local: this rank's operand is zeroed once every peer has read it. */
int trl_allreduce_grad(const void* const* peer_data, void* const* peer_flags, int rank, int world, float* out,
                       int64_t n, const int64_t* seg_begin_host, int nseg, unsigned active_mask, double* sumsq3_out,
                       int* step_counts, double beta1, double beta2, double* scratch, unsigned* ticket, unsigned* seq,
                       int zero_local, void* stream);
/* fp64 moment vectors (observation-normaliser sums of base_wrapper.py:75-82, advantage moments of ppo.py:147):
 * gather == 0: out (n) = sum over ranks; gather != 0: out (world, n) = every rank's vector in rank order. */
int trl_allreduce_f64(const void* const* peer_data, void* const* peer_flags, int rank, int world, double* out, int n,
                      int gather, unsigned* seq, void* stream);
/* The same exchange for small vectors (n <= nmax) as ONE NVLink traversal: every rank pushes 16-byte packets
 * {lo32, seq, hi32, seq} into slot [seq & 1][rank] of each peer's receive area and polls its own (NCCL's "LL" scheme; no
 * barrier phases, no fences).  peer_recv: `world` device pointers to receive areas of trl_comm_ll_recv_bytes(world, nmax)
 * zero-initialised bytes; ll_seq: device uint32 of the communicator counting LL exchanges. */
int64_t trl_comm_ll_recv_bytes(int world, int nmax);
int trl_allreduce_f64_ll(const double* local, void* const* peer_recv, int rank, int world, double* out, int n, int nmax,
                         int gather, unsigned* ll_seq, void* stream);

/* ---- fp32-faithful tensor-core GEMM for the 256-wide MLP layers (wgmma tf32, 3xTF32 split in
 * shared memory, TMA operand loads, register accumulator): C (M x 256) = A (M x K) . B (256 x K)^T, A/B row-major.
 * Serves MLPBase's Linear forward / dgrad / wgrad (networks/base.py:24-44) when the layer width is 256.
 * splits > 1: deterministic split-K (workspace: splits*M*256 floats).  bias != NULL (splits == 1): the Linear
 * epilogue C = act(A B^T + bias) is fused (act: 0 none, 1 tanh, 2 relu). */
int trl_gemm_tf32x3_nt(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                       float* workspace, const float* bias, int act, void* stream);
/* C (M x 256) = A (K x M)^T . B (K x 256): the weight-gradient shape (operands M/N-major, no transposes). */
int trl_gemm_tf32x3_tn(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                       float* workspace, void* stream);
int trl_transpose_f32(const float* in, float* out, int64_t rows, int cols, void* stream);
/* The same three shapes for the hot path (csrc/gemm_pair.cu): pre-split weight planes, N-major dgrad operand,
 * MUFU tanh, 8-way split-K reduce.  C (M x 256) = act(A (M x K) . B + bias):
 * b_nmajor == 0: B is (256 x K) row-major (Linear forward, networks/base.py:24-44: x W^T + b);
 * b_nmajor != 0: B is (K x 256) row-major (the dgrad shape g W, no transpose of the weights).
 * b_lo != NULL: (b_hi, b_lo) are pre-split TF32 planes of B (trl_split_tf32 / trl_adam_step / trl_polyak_update);
 * b_lo == NULL: b_hi is the raw fp32 matrix, split in shared memory.  Any M >= 1, K % 32 == 0. */
int trl_gemm3_pair(const float* A, const float* b_hi, const float* b_lo, float* C, int64_t M, int64_t K,
                   int b_nmajor, const float* bias, int act, void* stream);
/* C (M x 256) = A (K x M)^T . B (K x 256), M % 256 == 0, deterministic split-K (the weight-gradient shape). */
int trl_gemm3_pair_tn(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                      float* workspace, void* stream);
/* The same C bit for bit, with the split-K sum inside one launch (thread-block clusters of splits / 8 CTAs).
 * 8 <= splits <= 64, splits % 8 == 0; workspace: 8*M*256 floats; tickets: M/8 int32, zero on entry and left zero,
 * one set per stream. */
int trl_gemm3_pair_tn_cluster(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                              float* workspace, int* tickets, void* stream);
/* The dgrad dH1 = G (M x 256) . W2 of an MLP's second hidden layer with the first layer's backward as its epilogue:
 * writes the slab partials of trl_skinny_act_wgrad_partial(dH1, Y, X, M, 256, K, act, scratch) bit for bit, dH1 itself
 * is never stored.  (w_hi_t, w_lo_t): the transposed pre-split planes of W2 (256 x 256, hi^T and lo^T); Y: h1 (M x 256);
 * X: the first layer's input (M x K).  scratch: trl_skinny_tn_scratch_floats(M, 256, K) floats, summed by
 * trl_skinny_reduce_jobs (kind 1).  1 <= M <= 16896, 1 <= K <= 24; G, W, Y and scratch 16-byte aligned. */
int trl_gemm3_pair_dgrad_act_wgrad(const float* G, const float* w_hi_t, const float* w_lo_t, const float* Y,
                                   const float* X, int64_t M, int K, int act, float* scratch, void* stream);

/* ---- "skinny" Linear layers of the small MLPs (first layer K = obs_dim, output layer N = act_dim / 1;
 * networks/base.py:24-44, networks/nets.py:13-52): memory-bound fp32 kernels, bias / activation fused. */
int trl_skinny_k_fwd(const float* X, const float* W, const float* bias, float* Y, int64_t M, int K, int H,
                     int act, void* stream);                         /* Y = act(X W^T + b), K <= 128 */
int64_t trl_skinny_tn_scratch_floats(int64_t M, int H, int K);
int trl_skinny_tn(const float* A, const float* B, float* Out, float* colsum, int64_t M, int H, int K,
                  int out_transposed, float* scratch, void* stream);  /* Out = A^T B (K <= 32) [+ colsum(B)] */
int trl_skinny_n_fwd(const float* X, const float* W, const float* bias, float* Y, int64_t M, int H, int N,
                     void* stream);                                   /* Y = X W^T + b, N <= 8 */
int trl_skinny_n_dgrad(const float* G, const float* W, float* dX, int64_t M, int H, int N, void* stream);
/* backward fusions (autograd of networks/base.py:43-44 + nets.py:49-52): first-layer weight/bias gradient straight
 * from the upstream gradient and the layer output; output-layer dgrad fused with the hidden activation backward. */
int trl_skinny_act_wgrad(const float* G, const float* Y, const float* X, float* dW, float* db, int64_t M, int H,
                         int K, int act, float* scratch, void* stream);
int64_t trl_skinny_dgrad_act_scratch_floats(int64_t M, int H);
int trl_skinny_n_dgrad_act(const float* G, const float* W, const float* Y, float* gz, float* db, int64_t M, int H,
                           int N, int act, float* scratch, void* stream);
/* First stages alone + ONE launch for all the second stages of a backward pass.  The *_partial entry points run only the
 * pass over the (M x H) matrix and leave the per-CTA slabs in `scratch` (one scratch buffer per pending job, untouched
 * until the reduce); trl_skinny_reduce_jobs finishes up to 8 jobs in one launch.  kind: 0 = trl_skinny_tn (colsum NULL or
 * (K)), 1 = trl_skinny_act_wgrad (colsum = db (H)), 2 = trl_skinny_n_dgrad_act (colsum = db (H); out / K unused). */
int trl_skinny_tn_partial(const float* A, const float* B, int64_t M, int H, int K, int want_colsum, float* scratch,
                          void* stream);
int trl_skinny_act_wgrad_partial(const float* G, const float* Y, const float* X, int64_t M, int H, int K, int act,
                                 float* scratch, void* stream);
int trl_skinny_n_dgrad_act_partial(const float* G, const float* W, const float* Y, float* gz, int64_t M, int H, int N,
                                   int act, float* scratch, void* stream);
int trl_skinny_reduce_jobs(int njobs, const int* kind, const float* const* scratch, float* const* out,
                           float* const* colsum, const int64_t* M, const int* H, const int* K, const int* out_transposed,
                           void* stream);
/* The output layer's whole backward in one pass over Y (H == 256, 1 <= N <= 8): trl_skinny_n_dgrad_act_partial(G, W, Y,
 * gz, M, 256, N, act, db_scratch) and trl_skinny_tn_partial(Y, G, M, 256, N, 1, w_scratch) in one launch, bit for bit.
 * db_scratch (trl_skinny_dgrad_act_scratch_floats(M, 256) floats) is summed by reduce kind 2, w_scratch
 * (trl_skinny_tn_scratch_floats(M, 256, N) floats) by kind 0 with out_transposed = 1.  W, Y, gz, w_scratch 16-byte
 * aligned.  The second form also runs both reduces in one launch: db (256) = colsum(gz), dW (N x 256) = G^T Y,
 * dbias (N) = colsum(G). */
int trl_skinny_n_dgrad_act_wgrad_partial(const float* G, const float* W, const float* Y, float* gz, int64_t M, int H,
                                         int N, int act, float* db_scratch, float* w_scratch, void* stream);
int trl_skinny_n_dgrad_act_wgrad(const float* G, const float* W, const float* Y, float* gz, float* db, float* dW,
                                 float* dbias, int64_t M, int H, int N, int act, float* db_scratch, float* w_scratch,
                                 void* stream);

/* ---- K1 for BASELINE config 4: synthetic Atari-shaped pixel env, obs (N,4,84,84) uint8, 6 actions (defined in
 * oracle/synth_atari.py; the reference only wraps real ALE games, env/atari_wrapper.py).  latent: (N,5) int32. */
int trl_synth_atari_step(uint8_t* obs, int* latent, const float* actions, int* elapsed, float* reward,
                         uint8_t* done, uint8_t* time_limit, int64_t N, int max_steps, void* stream);
int trl_synth_atari_reset(uint8_t* obs, int* latent, int* elapsed, unsigned* episode, const unsigned* seeds,
                          const uint8_t* mask, const int* zero_is_mask, int episode_bias, int bump, int64_t N,
                          void* stream);
/* ---- K1 for CartPole-v0 / CartPole-v1: gym.make(env_id) (torchrl/env/get_env.py:53) with TimeLimitAugment.step
 * (env/base_wrapper.py:152-156), RewardShift.reward (env/base_wrapper.py:37-41) and VecEnv.step (env/vecenv.py:53-61)
 * fused in; gym's closed-form dynamics and Euler step in fp64 from the fp32 state (N,4), rounded once (defined in
 * oracle/cartpole.py).  actions (N) are 0.0 or 1.0 (force -10 / +10); any other value sets *action_error = 1 and
 * leaves that env's state unchanged.  reward = reward_scale on every step.  partial ((trl_cartpole_num_ctas(N), 8)
 * doubles) / batch_sums (8) / norm_*: the NormObs batch moments, as in trl_synth_env_step.  Resets go through
 * trl_synth_env_reset with obs_dim 4 and init_scale 0.05. */
int trl_cartpole_num_ctas(int64_t N);
int trl_cartpole_step(float* state, const float* actions, int* elapsed, const int* step_count, float* reward,
                      uint8_t* done, uint8_t* time_limit, int* action_error, double* partial, double* batch_sums,
                      double* norm_mean, double* norm_var, double* norm_count, unsigned* ticket, int* any_reset,
                      const int* t_ptr, int64_t N, float reward_scale, int max_episode_steps, int max_episode_frames,
                      int merge_stats, void* stream);
/* ---- K1 for Pendulum-v1: gym.make("Pendulum-v1") (torchrl/env/get_env.py:53) with NormAct.action
 * (env/continuous_wrapper.py:18-20), TimeLimitAugment.step (env/base_wrapper.py:152-156), RewardShift.reward
 * (env/base_wrapper.py:37-41) and VecEnv.step / partial_reset (env/vecenv.py:47-61) fused in (defined in
 * oracle/pendulum.py).  phys (N,2) fp64 (theta, theta_dot) in place; obs (N,3) fp32 raw observation (cos, sin,
 * theta_dot).  actions (N) in [-1, 1]: the torque is NormAct's map to [-2, 2] in fp32, widened exactly; the step is fp64
 * in gym's order, the velocity clipped before it moves the angle (v1).  A non-finite action sets *action_error = 1 and
 * leaves that env's state and observation unchanged (reward 0).  done = (elapsed >= max_episode_steps), time_limit =
 * done && elapsed == max_episode_steps.
 * partial ((trl_pendulum_num_ctas(N), 6) doubles) / batch_sums (6) / norm_*: the NormObs batch moments of the three
 * observation columns, as in trl_cartpole_step. */
int trl_pendulum_num_ctas(int64_t N);
int trl_pendulum_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count,
                      float* reward, uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                      double* batch_sums, double* norm_mean, double* norm_var, double* norm_count, unsigned* ticket,
                      int* any_reset, const int* t_ptr, int64_t N, float reward_scale, int max_episode_steps,
                      int max_episode_frames, int merge_stats, void* stream);
/* PendulumEnv.reset + VecEnv.partial_reset (env/vecenv.py:47-51), and for a collector the partial reset of
 * collect_finalize (theta = pi (2U - 1), theta_dot = 2U - 1 in fp64 from the counter hash of trl_synth_env_reset).
 * Selected envs: step_count[n] == 0 when step_count is given (after trl_collect_finalize with external-env arguments
 * this holds exactly for the envs it cut), else mask[n] != 0, else all.  They get a new state and raw observation,
 * elapsed = 0, episode += 1.  With cur_ob (needs step_count, next_norm, any_reset, t_ptr) it also writes the next
 * observation as collect_finalize does: raw without norm_mean; raw for all envs when raw_obs_after_reset and
 * any_reset[*t_ptr & 1]; otherwise clip((raw - mean) / (sqrt(var) + 1e-4)) on reset rows and next_norm on the rest. */
int trl_pendulum_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                       const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                       const int* any_reset, const int* t_ptr, const double* norm_mean, const double* norm_var,
                       int64_t N, double clip, int raw_obs_after_reset, void* stream);
/* ---- K1 for Acrobot-v1: gym.make("Acrobot-v1") (torchrl/env/get_env.py:53) with TimeLimitAugment.step
 * (env/base_wrapper.py:152-156), RewardShift.reward (env/base_wrapper.py:37-41) and VecEnv.step / partial_reset
 * (env/vecenv.py:47-61) fused in (defined in oracle/acrobot.py).  phys (N,4) fp64 (theta1, theta2, dtheta1, dtheta2) in
 * place; obs (N,6) fp32 raw observation (cos theta1, sin theta1, cos theta2, sin theta2, dtheta1, dtheta2).  actions (N)
 * are 0.0, 1.0 or 2.0 (torque -1, 0, +1); any other value sets *action_error = 1 and leaves that env's state and
 * observation unchanged (reward 0).  The step is one RK4 step of gym's "book" dynamics over dt = 0.2 in fp64 in gym's
 * order, the angles wrapped into [-pi, pi] by gym's loop, the velocities bounded by 4 pi and 9 pi.  done = terminal
 * (-cos theta1 - cos(theta1 + theta2) > 1) or elapsed >= max_episode_steps, time_limit = done && elapsed ==
 * max_episode_steps; reward = reward_scale * (terminal ? 0 : -1).
 * partial ((trl_acrobot_num_ctas(N), 12) doubles) / batch_sums (12) / norm_*: the NormObs batch moments of the six
 * observation columns, as in trl_cartpole_step. */
int trl_acrobot_num_ctas(int64_t N);
int trl_acrobot_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count, float* reward,
                     uint8_t* done, uint8_t* time_limit, int* action_error, double* partial, double* batch_sums,
                     double* norm_mean, double* norm_var, double* norm_count, unsigned* ticket, int* any_reset,
                     const int* t_ptr, int64_t N, float reward_scale, int max_episode_steps, int max_episode_frames,
                     int merge_stats, void* stream);
/* AcrobotEnv.reset + VecEnv.partial_reset, and for a collector the partial reset of collect_finalize, as
 * trl_pendulum_reset: every state component 0.1 (2U - 1) in fp64 from the counter hash of trl_synth_env_reset. */
int trl_acrobot_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                      const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                      const int* any_reset, const int* t_ptr, const double* norm_mean, const double* norm_var,
                      int64_t N, double clip, int raw_obs_after_reset, void* stream);
/* ---- K1 for MountainCar-v0 (continuous = 0) and MountainCarContinuous-v0 (continuous = 1): gym.make(env_id)
 * (torchrl/env/get_env.py:53) with, for the continuous variant, NormAct.action (env/continuous_wrapper.py:18-20), and
 * TimeLimitAugment.step (env/base_wrapper.py:152-156), RewardShift.reward (env/base_wrapper.py:37-41) and VecEnv.step /
 * partial_reset (env/vecenv.py:47-61) fused in (defined in oracle/mountain_car.py).  phys (N,2) fp64 (position,
 * velocity) in place; obs (N,2) fp32 raw observation.  v0: actions (N) are 0.0, 1.0 or 2.0 (push left, none, right),
 * reward -1; continuous: actions (N) in [-1, 1], the force is NormAct's map to [-1, 1] in fp32, widened exactly, reward
 * 100 on reaching the goal minus 0.1 force^2.  A refused action (v0: any other value; continuous: not finite) sets
 * *action_error = 1 and leaves that env's state and observation unchanged (reward 0).  done = terminal (position >= 0.5,
 * continuous 0.45, with velocity >= 0) or elapsed >= max_episode_steps; time_limit as in trl_acrobot_step.
 * partial ((trl_mountain_car_num_ctas(N), 4) doubles) / batch_sums (4) / norm_*: the NormObs batch moments, as in
 * trl_cartpole_step. */
int trl_mountain_car_num_ctas(int64_t N);
int trl_mountain_car_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count,
                          float* reward, uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                          double* batch_sums, double* norm_mean, double* norm_var, double* norm_count,
                          unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N, float reward_scale,
                          int max_episode_steps, int max_episode_frames, int merge_stats, int continuous,
                          void* stream);
/* MountainCarEnv.reset + VecEnv.partial_reset, and for a collector the partial reset of collect_finalize, as
 * trl_pendulum_reset: position -0.6 + 0.2 U in fp64 from the counter hash of trl_synth_env_reset, velocity 0. */
int trl_mountain_car_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                           const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                           const int* any_reset, const int* t_ptr, const double* norm_mean, const double* norm_var,
                           int64_t N, double clip, int raw_obs_after_reset, void* stream);

/* ScaledFloatFrame (env/atari_wrapper.py:171-180): out = in * scale */
int trl_u8_to_f32(const uint8_t* in, float* out, int64_t n, float scale, void* stream);

/* ---- Atari frames stepped by host envs (env/atari_host.py; defined in oracle/atari_frames.py): WarpFrame
 * (env/atari_wrapper.py:112-131, OpenCV's RGB2GRAY and INTER_AREA resize to 84x84, bit for bit) and FrameStack
 * (:134-168) in one launch, one CTA per frame.  frames (M, H, W, 3) uint8 RGB, H, W >= 84, 3W % 16 == 0,
 * H*W + 7056 <= 227 KB; stack (N, C, 84, 84) uint8 in place; both 16-byte aligned.  Frame m belongs to env
 * env_idx[m] (env_idx NULL: env m, and M == N; ids outside [0, N) are skipped).  An env with fresh[n] != 0, or every
 * env when fresh is NULL, gets the new frame in all C slots (FrameStack.reset); any other env's stack shifts by one
 * frame and the new frame is appended (FrameStack.step).  tab_i = [xofs (85) | yofs (85) | xsrc | ysrc] int32 and
 * tab_w = [xw | yw] fp32: OpenCV's area tables (computeResizeAreaTab) of W -> 84 and H -> 84 in CSR form, output
 * column dx drawing on entries xofs[dx] .. xofs[dx+1]-1 (env/atari_host.py area_tables builds them). */
int trl_atari_warp_stack(const uint8_t* frames, const int* env_idx, const uint8_t* fresh, uint8_t* stack,
                         const int* tab_i, const float* tab_w, int64_t M, int64_t N, int H, int W, int C,
                         void* stream);
/* out[i] = lut[in[i]] as float32 (n % 4 == 0, in 4-byte and out 16-byte aligned, lut 256 floats): the pixel env's
 * to_float, exact by construction for any map built on the host (ScaledFloatFrame's x / 255.0 - 0.5, or float(x)). */
int trl_u8_lut_f32(const uint8_t* in, float* out, int64_t n, const float* lut, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TORCHRL_B200_H */
