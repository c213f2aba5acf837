// collect.cu -- K3 (action sampling), K4 (rollout row store), K5 (timeout bootstrap / partial reset).
//
// K3 replaces the sampling half of
//   GuassianContPolicyBase.explore   /root/reference/torchrl/policies/continuous_policy.py:92-132
//   TanhNormal.rsample / log_prob    /root/reference/torchrl/policies/distribution.py:60-76, 33-45
// K4+K5 replace, per collector step,
//   VecOnPolicyCollector.take_actions /root/reference/torchrl/collector/on_policy.py:115-153
//   VecCollector.take_actions         /root/reference/torchrl/collector/base.py:204-228
//   BaseReplayBuffer.add_sample       /root/reference/torchrl/replay_buffers/base.py:19-37
// The time row `t` is read from device memory so that one captured CUDA graph of the whole
// step can be replayed for every row of the epoch (pointers in the graph never change).
#include "env_common.cuh"

namespace trl {

constexpr float kLogSqrt2Pi = 0.9189385332046727f;  // 0.5*log(2*pi)

// ------------------------------------------------------------------------------------ K3
struct SampleParams {
  const float* __restrict__ mean;     // (M,a)
  const float* __restrict__ log_std;  // (a) if ls_stride==0 else (M,a)
  const float* __restrict__ eps;      // (M,a) standard-normal noise, or nullptr -> Philox
  float* __restrict__ action;         // (M,a)
  float* __restrict__ pre_tanh;       // (M,a) or nullptr
  float* __restrict__ log_prob;       // (M) or nullptr
  float* __restrict__ eps_out;        // (M,a) or nullptr: the noise actually used (needed by backward)
  int* __restrict__ nan_flag;         // (1) or nullptr
  const unsigned long long* __restrict__ rng_counter;  // (1) device counter (Philox offset)
  unsigned long long seed;
  long long M;
  int a, ls_stride, tanh_action;
  float noise_scale;                  // multiplies eps (1 for Gaussian policies)
};

__global__ void tanh_gaussian_sample_kernel(const SampleParams p) {
  const long long m = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= p.M) return;
  const int a = p.a;
  const unsigned long long ctr = p.rng_counter ? *p.rng_counter : 0ull;
  float lp = 0.f;
  bool bad = false;
  float nrm[4];
  for (int j = 0; j < a; ++j) {
    float e;
    if (p.eps) {
      e = p.eps[m * a + j];
    } else {
      if ((j & 3) == 0) {
        uint32_t r[4];
        Philox::gen(p.seed, ctr * 0x100000000ull + static_cast<unsigned long long>(m), static_cast<uint32_t>(j >> 2), r);
        box_muller(r[0], r[1], nrm[0], nrm[1]);
        box_muller(r[2], r[3], nrm[2], nrm[3]);
      }
      e = nrm[j & 3];
    }
    e *= p.noise_scale;
    const float ls = p.log_std[(p.ls_stride ? m * p.ls_stride : 0) + j];
    const float sd = expf(ls);
    const float mu = p.mean[m * a + j];
    const float z = fmaf(sd, e, mu);
    const float act = p.tanh_action ? tanhf(z) : z;
    p.action[m * a + j] = act;
    if (p.pre_tanh) p.pre_tanh[m * a + j] = z;
    if (p.eps_out) p.eps_out[m * a + j] = e;
    if (p.log_prob) {
      // Normal(mu,sd).log_prob(z) with (z-mu)/sd == e, minus the tanh Jacobian term
      float l = -0.5f * e * e - ls - kLogSqrt2Pi;
      if (p.tanh_action) l -= logf(1.0f - act * act + 1e-6f);
      lp += l;
    }
    bad |= isnan(act);
  }
  if (p.log_prob) p.log_prob[m] = lp;
  if (bad && p.nan_flag) atomicOr(p.nan_flag, 1);
}

// backward of (action, log_prob) wrt (mean, log_std) for the reparameterised sample.
struct SampleBwdParams {
  const float* __restrict__ action;    // (M,a)
  const float* __restrict__ eps;       // (M,a) noise used in forward (already scaled)
  const float* __restrict__ log_std;   // (a) or (M,a)
  const float* __restrict__ g_action;  // (M,a) or nullptr
  const float* __restrict__ g_logp;    // (M)   or nullptr
  float* __restrict__ g_mean;          // (M,a)
  float* __restrict__ g_log_std;       // (M,a) per-row gradient (caller reduces if log_std is shared)
  long long M;
  int a, ls_stride, tanh_action;
};

__global__ void tanh_gaussian_sample_bwd_kernel(const SampleBwdParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= p.M * p.a) return;
  const long long m = i / p.a;
  const int j = static_cast<int>(i - m * p.a);
  const float act = p.action[i], e = p.eps[i];
  const float ls = p.log_std[(p.ls_stride ? m * p.ls_stride : 0) + j];
  const float sd = expf(ls);
  const float ga = p.g_action ? p.g_action[i] : 0.f;
  const float gl = p.g_logp ? p.g_logp[m] : 0.f;
  float dadz = 1.f, dldz = 0.f;
  if (p.tanh_action) {
    dadz = 1.f - act * act;
    dldz = 2.f * act * dadz / (1.f - act * act + 1e-6f);  // -d/dz log(1 - a^2 + eps)
  }
  const float gz = ga * dadz + gl * dldz;       // dz/dmu = 1, dz/dls = sd*e
  p.g_mean[i] = gz;
  p.g_log_std[i] = gz * sd * e - gl;            // -ls term of the Normal log-density
}

// ------------------------------------------------------------------------------------ K4/K5
struct FinalizeParams {
  // step inputs (fixed staging buffers)
  const float* cur_ob_in;                // (N,o) observation the policy acted on (may alias cur_ob_out)
  const float* __restrict__ next_norm;   // (N,o) next observation as returned by env.step (normalised if NormObs)
  float* __restrict__ state;             // (N,o) raw env state (post-step); reset in place
  const float* __restrict__ act;         // (N,a)  (or (N) int64-as-float for discrete; a==1)
  const float* __restrict__ value;       // (N) V(cur_ob) or nullptr (off-policy)
  const float* __restrict__ v_next;      // (N) V(next_norm) or nullptr (no bootstrap this step)
  const float* __restrict__ reward;      // (N)
  const uint8_t* __restrict__ done;      // (N)
  const uint8_t* __restrict__ tl;        // (N)
  // env / collector state
  int* __restrict__ elapsed;             // (N)
  unsigned* __restrict__ episode;        // (N)
  const unsigned* __restrict__ seeds;    // (N)
  int* __restrict__ step_count;          // (N) collector current_step
  double* __restrict__ ep_return;        // (N) running episode return (train_rew)
  double* __restrict__ epoch_reward;     // (N) per-env sum of rewards this epoch
  float* __restrict__ ret_log;           // (T,N) finished-episode returns (NaN = none) or nullptr
  int* __restrict__ n_done;              // (1) number of finished episodes this epoch
  const int* __restrict__ any_reset;     // (2) flag written by the env kernel
  const double* __restrict__ norm_mean;  // (o) or nullptr (no NormObs)
  const double* __restrict__ norm_var;   // (o)
  float* cur_ob_out;                     // (N,o) observation for the next step
  // rollout storage, time-major
  float* __restrict__ b_obs;             // (T,N,o)
  float* __restrict__ b_next_obs;        // (T,N,o)
  float* __restrict__ b_acts;            // (T,N,a)
  float* __restrict__ b_values;          // (T,N) or nullptr
  float* __restrict__ b_rewards;         // (T,N)
  uint8_t* __restrict__ b_terminals;     // (T,N)
  uint8_t* __restrict__ b_time_limits;   // (T,N)
  const int* __restrict__ t_ptr;         // (1) row to write
  long long N;
  int o, a;
  int max_episode_frames;
  float discount;
  double init_scale, clip;
  int terminal_includes_surpass;         // on-policy collector: terminals = done | surpass
  int raw_obs_after_reset;               // reference quirk A.1 (SURVEY.md): raw obs for ALL envs after any reset
};

constexpr int kFinEnvs = 32;

__global__ void __launch_bounds__(256) collect_finalize_kernel(const FinalizeParams p) {
  __shared__ uint8_t s_mask[kFinEnvs];
  const int tid = threadIdx.x, nthr = blockDim.x;
  const long long env_base = static_cast<long long>(blockIdx.x) * kFinEnvs;
  const int ne = static_cast<int>(min(static_cast<long long>(kFinEnvs), p.N - env_base));
  const int t = *p.t_ptr;
  const long long N = p.N;
  const int o = p.o, a = p.a;
  const int any_reset = p.any_reset ? p.any_reset[t & 1] : 0;

  if (tid < ne) {
    const long long n = env_base + tid;
    const int sc = p.step_count[n] + 1;
    const bool dn = p.done[n] != 0;
    const bool surpass = sc >= p.max_episode_frames;
    const bool mask = dn || surpass;
    float r = p.reward[n];
    // train_rew bookkeeping uses the un-bootstrapped reward (on_policy.py:126-130)
    const double er = p.ep_return[n] + static_cast<double>(r);
    p.epoch_reward[n] += static_cast<double>(r);
    if (dn) {
      if (p.ret_log) p.ret_log[static_cast<long long>(t) * N + n] = static_cast<float>(er);
      atomicAdd(p.n_done, 1);
      p.ep_return[n] = 0.0;
    } else {
      p.ep_return[n] = er;
    }
    if (p.v_next && surpass) r = fmaf(p.discount * p.v_next[n], 1.0f, r);  // rewards + discount*V(next)*surpass
    const long long row = static_cast<long long>(t) * N + n;
    p.b_rewards[row] = r;
    p.b_terminals[row] = (dn || (p.terminal_includes_surpass && surpass)) ? 1 : 0;
    p.b_time_limits[row] = p.tl[n];
    if (p.b_values) p.b_values[row] = p.value[n];
    p.step_count[n] = mask ? 0 : sc;
    if (mask && p.elapsed) { p.elapsed[n] = 0; }
    s_mask[tid] = mask ? 1 : 0;
  }
  __syncthreads();

  // rows: obs[t] <- cur_ob ; next_obs[t] <- next_norm ; acts[t] <- act
  {
    const long long src = env_base * o;
    const long long dst = (static_cast<long long>(t) * N + env_base) * o;
    for (int i = tid; i < ne * o; i += nthr) {
      p.b_obs[dst + i] = p.cur_ob_in[src + i];
      p.b_next_obs[dst + i] = p.next_norm[src + i];
    }
    const long long srca = env_base * a;
    const long long dsta = (static_cast<long long>(t) * N + env_base) * a;
    for (int i = tid; i < ne * a; i += nthr) p.b_acts[dsta + i] = p.act[srca + i];
  }
  __syncthreads();  // cur_ob_in may alias cur_ob_out: finish every read before the writes below
  if (!p.seeds) {
    // external (host) envs: the reset happens on the host after this launch (env/bridge.py); carry the
    // stepped observation forward and let the bridge overwrite the rows it resets
    for (int i = tid; i < ne * o; i += nthr) p.cur_ob_out[env_base * o + i] = p.next_norm[env_base * o + i];
    return;
  }
  // partial reset + next current_ob; under quirk A.1 no row is normalised, so a reset without the flag carries over
  const bool all_raw = !p.norm_mean || (p.raw_obs_after_reset && any_reset);
  for (int i = tid; i < ne * o; i += nthr) {
    const int e = i / o, j = i - e * o;
    const long long n = env_base + e;
    float raw;
    if (s_mask[e]) {
      raw = reset_value(p.seeds[n], p.episode[n], j, p.init_scale);
      p.state[n * o + j] = raw;
    } else {
      raw = p.state[n * o + j];
    }
    p.cur_ob_out[n * o + j] = next_observation(all_raw, s_mask[e] && !p.raw_obs_after_reset, raw,
                                               p.next_norm + n * o + j, p.norm_mean, p.norm_var, j, p.clip);
  }
  __syncthreads();
  if (tid < ne && s_mask[tid]) p.episode[env_base + tid] += 1u;
}

// advance the device-side row index (mod T), ring size and Philox offset by one step
__global__ void step_advance_kernel(int* t_ptr, int T, int* size_ptr, unsigned long long* rng_counter) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (t_ptr) *t_ptr = (*t_ptr + 1) % T;
    if (size_ptr && *size_ptr < T) *size_ptr += 1;
    if (rng_counter) *rng_counter += 1ull;
  }
}

}  // namespace trl

TRL_API int trl_tanh_gaussian_sample(const float* mean, const float* log_std, int ls_stride, const float* eps,
                                     float noise_scale, uint64_t seed, const uint64_t* rng_counter, int64_t M,
                                     int act_dim, int tanh_action, float* action, float* pre_tanh, float* log_prob,
                                     float* eps_out, int* nan_flag, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && act_dim >= 1, "trl_tanh_gaussian_sample: bad sizes");
  if (M == 0) return TRL_OK;
  TRL_REQUIRE(mean && log_std && action, "trl_tanh_gaussian_sample: null pointer");
  TRL_REQUIRE(ls_stride == 0 || ls_stride == act_dim, "trl_tanh_gaussian_sample: ls_stride must be 0 or act_dim");
  SampleParams p{mean, log_std, eps, action, pre_tanh, log_prob, eps_out, nan_flag,
                 reinterpret_cast<const unsigned long long*>(rng_counter), seed, M, act_dim, ls_stride, tanh_action,
                 noise_scale};
  tanh_gaussian_sample_kernel<<<static_cast<unsigned>(ceil_div<long long>(M, 128)), 128, 0,
                                static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("tanh_gaussian_sample_kernel");
}

TRL_API int trl_tanh_gaussian_sample_bwd(const float* action, const float* eps, const float* log_std, int ls_stride,
                                         const float* g_action, const float* g_logp, int64_t M, int act_dim,
                                         int tanh_action, float* g_mean, float* g_log_std, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && act_dim >= 1, "trl_tanh_gaussian_sample_bwd: bad sizes");
  if (M == 0) return TRL_OK;
  TRL_REQUIRE(action && eps && log_std && g_mean && g_log_std, "trl_tanh_gaussian_sample_bwd: null pointer");
  TRL_REQUIRE(ls_stride == 0 || ls_stride == act_dim,
              "trl_tanh_gaussian_sample_bwd: ls_stride must be 0 or act_dim");
  SampleBwdParams p{action, eps, log_std, g_action, g_logp, g_mean, g_log_std, M, act_dim, ls_stride, tanh_action};
  tanh_gaussian_sample_bwd_kernel<<<static_cast<unsigned>(ceil_div<long long>(M * act_dim, 256)), 256, 0,
                                    static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("tanh_gaussian_sample_bwd_kernel");
}

TRL_API int trl_collect_finalize(const float* cur_ob_in, const float* next_norm, float* state, const float* act,
                                 const float* value, const float* v_next, const float* reward, const uint8_t* done,
                                 const uint8_t* tl, int* elapsed, unsigned* episode, const unsigned* seeds,
                                 int* step_count, double* ep_return, double* epoch_reward, float* ret_log,
                                 int* n_done, const int* any_reset, const double* norm_mean, const double* norm_var,
                                 float* cur_ob_out, float* b_obs, float* b_next_obs, float* b_acts, float* b_values,
                                 float* b_rewards, uint8_t* b_terminals, uint8_t* b_time_limits, const int* t_ptr,
                                 int64_t N, int obs_dim, int act_dim, int max_episode_frames, float discount,
                                 double init_scale, double clip, int terminal_includes_surpass,
                                 int raw_obs_after_reset, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && obs_dim >= 1 && act_dim >= 1, "trl_collect_finalize: bad sizes");
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(cur_ob_in && next_norm && act && reward && done && tl && step_count && ep_return && epoch_reward &&
                  n_done && cur_ob_out && b_obs && b_next_obs && b_acts && b_rewards && b_terminals && b_time_limits &&
                  t_ptr,
              "trl_collect_finalize: null pointer");
  TRL_REQUIRE((state && elapsed && episode && seeds) || (!state && !elapsed && !episode && !seeds),
              "trl_collect_finalize: state/elapsed/episode/seeds must be all given (device env, in-kernel reset) "
              "or all NULL (host env, external reset)");
  TRL_REQUIRE(!b_values || value, "trl_collect_finalize: b_values given without value");
  FinalizeParams p{cur_ob_in, next_norm, state, act, value, v_next, reward, done, tl, elapsed, episode, seeds,
                   step_count, ep_return, epoch_reward, ret_log, n_done, any_reset, norm_mean, norm_var, cur_ob_out,
                   b_obs, b_next_obs, b_acts, b_values, b_rewards, b_terminals, b_time_limits, t_ptr, N, obs_dim,
                   act_dim, max_episode_frames, discount, init_scale, clip, terminal_includes_surpass,
                   raw_obs_after_reset};
  collect_finalize_kernel<<<static_cast<unsigned>(ceil_div<long long>(N, kFinEnvs)), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("collect_finalize_kernel");
}

TRL_API int trl_step_advance(int* t_ptr, int T, int* size_ptr, uint64_t* rng_counter, void* stream) {
  using namespace trl;
  TRL_REQUIRE(T >= 1, "trl_step_advance: T must be >= 1");
  step_advance_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(
      t_ptr, T, size_ptr, reinterpret_cast<unsigned long long*>(rng_counter));
  return check_launch("step_advance_kernel");
}
