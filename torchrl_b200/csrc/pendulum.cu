// pendulum.cu -- K1 for the classic-control Pendulum-v1: N envs advance (and reset) in one launch.
//
// Replaces, for N Pendulum envs held on the device, the per-env Python chain
//   gym.make("Pendulum-v1") -> PendulumEnv.step / reset   /root/reference/torchrl/env/get_env.py:53
//   NormAct.action                                         /root/reference/torchrl/env/continuous_wrapper.py:18-20
//   TimeLimitAugment.step                                  /root/reference/torchrl/env/base_wrapper.py:152-156
//   RewardShift.reward                                     /root/reference/torchrl/env/base_wrapper.py:37-41
//   VecEnv.step / partial_reset                            /root/reference/torchrl/env/vecenv.py:47-61
// and, like csrc/cartpole.cu, accumulates the batch moments NormObs needs (base_wrapper.py:75-82, :44-60).
// The dynamics are gym's Pendulum-v1 (the clipped velocity moves the angle); oracle/pendulum.py is the NumPy statement
// this file must agree with.
//
// Precision: the physical state (theta, theta_dot) is fp64 as in gym; the torque is NormAct's affine map evaluated in
// fp32 (explicitly rounded, so -fmad=true cannot contract it) and widened exactly; the step is fp64 with every
// operation rounded once in gym's order; the observation (cos, sin, theta_dot) and the reward are rounded to fp32 once.
//
// Layout: phys (N,2) fp64, obs (N,3) fp32 raw observation; one thread per env, kPendThreads envs per CTA.  The reset
// has its own kernel because the observation is not the state: collect_finalize's in-kernel reset cannot serve it.
#include "env_common.cuh"

namespace trl {

constexpr int kPendThreads = 256;

// gym's PendulumEnv constants (classic_control/pendulum.py)
constexpr double kPendG = 10.0;
constexpr double kPendM = 1.0;
constexpr double kPendL = 1.0;
constexpr double kPendDt = 0.05;
constexpr double kPendMaxSpeed = 8.0;
constexpr float kPendMaxTorque = 2.0f;
constexpr double kPi = 3.141592653589793;
constexpr double kTwoPi = 2.0 * 3.141592653589793;
constexpr double kGravTerm = 3.0 * kPendG / (2.0 * kPendL);            // 15.0, exact
constexpr double kTorqueTerm = 3.0 / (kPendM * kPendL * kPendL);       // 3.0, exact

// NormAct (continuous_wrapper.py:18-20) with lb = -2, ub = 2, in fp32: clip(lb + (a + 1) * 0.5 * (ub - lb), lb, ub)
__device__ __forceinline__ float pend_torque(float a) {
  const float lb = -kPendMaxTorque, ub = kPendMaxTorque;
  const float u = __fadd_rn(lb, __fmul_rn(__fmul_rn(__fadd_rn(a, 1.0f), 0.5f), __fadd_rn(ub, -lb)));
  return fminf(fmaxf(u, lb), ub);
}

// angle_normalize(x) = ((x + pi) % (2 pi)) - pi with Python's float %: fmod (exact), shifted into [0, 2 pi)
__device__ __forceinline__ double pend_angle_normalize(double x) {
  double r = fmod(__dadd_rn(x, kPi), kTwoPi);
  if (r < 0.0) r = __dadd_rn(r, kTwoPi);
  return __dadd_rn(r, -kPi);
}

struct PendulumParams {
  double* __restrict__ phys;            // (N,2) in/out: theta, theta_dot
  float* __restrict__ obs;              // (N,3) out: cos theta, sin theta, theta_dot
  const float* __restrict__ actions;    // (N) policy-space actions, [-1, 1] after NormAct's clip
  int* __restrict__ action_error;       // (1) set to 1 when an action is not finite
  EnvStepFields env;                    // D = 3
};

__global__ void __launch_bounds__(kPendThreads) pendulum_step_kernel(const PendulumParams p) {
  const EnvStepFields& f = p.env;
  const long long n = static_cast<long long>(blockIdx.x) * kPendThreads + threadIdx.x;
  float ob[3] = {0.f, 0.f, 0.f};
  bool local_reset = false;
  if (n < f.N) {
    const double th = p.phys[n * 2], thdot = p.phys[n * 2 + 1];
    const float a = p.actions[n];
    float r = 0.f;
    if (isfinite(a)) {
      const double u = static_cast<double>(pend_torque(a));
      const double an = pend_angle_normalize(th);
      const double cost = __dadd_rn(__dadd_rn(__dmul_rn(an, an), __dmul_rn(0.1, __dmul_rn(thdot, thdot))),
                                    __dmul_rn(0.001, __dmul_rn(u, u)));
      double nthdot =
          __dadd_rn(thdot, __dmul_rn(__dadd_rn(__dmul_rn(kGravTerm, sin(th)), __dmul_rn(kTorqueTerm, u)), kPendDt));
      nthdot = fmin(fmax(nthdot, -kPendMaxSpeed), kPendMaxSpeed);
      const double nth = __dadd_rn(th, __dmul_rn(nthdot, kPendDt));   // v1: the clipped velocity moves the angle
      p.phys[n * 2] = nth;
      p.phys[n * 2 + 1] = nthdot;
      ob[0] = static_cast<float>(cos(nth));
      ob[1] = static_cast<float>(sin(nth));
      ob[2] = static_cast<float>(nthdot);
      r = static_cast<float>(__dmul_rn(-cost, static_cast<double>(f.reward_scale)));
    } else {
      // not an action: flag it for the host and leave this env's state and observation where they were
      atomicOr(p.action_error, 1);
#pragma unroll
      for (int j = 0; j < 3; ++j) ob[j] = p.obs[n * 3 + j];
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) p.obs[n * 3 + j] = ob[j];
    local_reset = env_row_end(f, n, false, r);       // no terminal state: only the time limit ends an episode
  }
  update_any_reset(f, local_reset);
  if (f.partial) env_moments<3, kPendThreads>(f, ob);
}

struct PendulumResetParams {
  double* __restrict__ phys;              // (N,2)
  float* __restrict__ obs;                // (N,3) raw observation
  int* __restrict__ elapsed;              // (N)
  unsigned* __restrict__ episode;         // (N)
  const unsigned* __restrict__ seeds;     // (N)
  const uint8_t* __restrict__ mask;       // (N) envs to reset, or nullptr
  const int* __restrict__ step_count;     // (N) reset where 0 (the collector's path), or nullptr
  // collector path (cur_ob != nullptr): the next observation of every env, as collect_finalize writes it
  const float* __restrict__ next_norm;    // (N,3) observation the env step returned (normalised if NormObs)
  float* __restrict__ cur_ob;             // (N,3) or nullptr
  const int* __restrict__ any_reset;      // (2) flag written by the step kernel
  const int* __restrict__ t_ptr;          // (1) ring row (selects the flag slot)
  const double* __restrict__ norm_mean;   // (3) or nullptr (no NormObs)
  const double* __restrict__ norm_var;    // (3)
  long long N;
  double clip;
  int raw_obs_after_reset;                // reference quirk A.1 (SURVEY.md): raw obs for ALL envs after any reset
};

__global__ void __launch_bounds__(kPendThreads) pendulum_reset_kernel(const PendulumResetParams p) {
  const long long n = static_cast<long long>(blockIdx.x) * kPendThreads + threadIdx.x;
  if (n >= p.N) return;
  const bool sel = p.step_count ? p.step_count[n] == 0 : (p.mask ? p.mask[n] != 0 : true);
  float raw[3];
  if (sel) {
    // theta ~ U(-pi, pi), theta_dot ~ U(-1, 1) from the counter hash of (seed, episode, component)
    const unsigned seed = p.seeds[n], ep = p.episode[n];
    const double th = __dmul_rn(kPi, __dadd_rn(__dmul_rn(2.0, double(counter_uniform(seed, ep, 0))), -1.0));
    const double thdot = __dadd_rn(__dmul_rn(2.0, double(counter_uniform(seed, ep, 1))), -1.0);
    p.phys[n * 2] = th;
    p.phys[n * 2 + 1] = thdot;
    raw[0] = static_cast<float>(cos(th));
    raw[1] = static_cast<float>(sin(th));
    raw[2] = static_cast<float>(thdot);
#pragma unroll
    for (int j = 0; j < 3; ++j) p.obs[n * 3 + j] = raw[j];
    p.episode[n] = ep + 1u;
    p.elapsed[n] = 0;
  } else {
#pragma unroll
    for (int j = 0; j < 3; ++j) raw[j] = p.obs[n * 3 + j];
  }
  if (!p.cur_ob) return;
  const bool all_raw = !p.norm_mean || (p.raw_obs_after_reset && p.any_reset[*p.t_ptr & 1]);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    p.cur_ob[n * 3 + j] =
        next_observation(all_raw, sel, raw[j], p.next_norm + n * 3 + j, p.norm_mean, p.norm_var, j, p.clip);
  }
}

}  // namespace trl

TRL_API int trl_pendulum_num_ctas(int64_t N) {
  return static_cast<int>((N + trl::kPendThreads - 1) / trl::kPendThreads);
}

TRL_API int trl_pendulum_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count,
                              float* reward, uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                              double* batch_sums, double* norm_mean, double* norm_var, double* norm_count,
                              unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N, float reward_scale,
                              int max_episode_steps, int max_episode_frames, int merge_stats, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && max_episode_steps >= 1, "trl_pendulum_step: bad sizes N=%lld max_episode_steps=%d",
              (long long)N, max_episode_steps);
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(phys && obs && actions && elapsed && reward && done && time_limit && action_error,
              "trl_pendulum_step: null pointer");
  PendulumParams p{phys, obs, actions, action_error,
                   {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean, norm_var, norm_count,
                    ticket, any_reset, t_ptr, N, reward_scale, max_episode_steps, max_episode_frames, merge_stats}};
  if (const int e = check_env_step("trl_pendulum_step", p.env)) return e;
  pendulum_step_kernel<<<trl_pendulum_num_ctas(N), kPendThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("pendulum_step_kernel");
}

TRL_API int trl_pendulum_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                               const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                               const int* any_reset, const int* t_ptr, const double* norm_mean,
                               const double* norm_var, int64_t N, double clip, int raw_obs_after_reset,
                               void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0, "trl_pendulum_reset: bad size N=%lld", (long long)N);
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(phys && obs && elapsed && episode && seeds, "trl_pendulum_reset: null pointer");
  TRL_REQUIRE(!(mask && step_count), "trl_pendulum_reset: select envs by mask or by step_count, not both");
  TRL_REQUIRE(!cur_ob || (step_count && next_norm && any_reset && t_ptr),
              "trl_pendulum_reset: cur_ob needs step_count, next_norm, any_reset and t_ptr");
  TRL_REQUIRE(!norm_mean || norm_var, "trl_pendulum_reset: norm_mean given without norm_var");
  PendulumResetParams p{phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob, any_reset, t_ptr,
                        norm_mean, norm_var, N, clip, raw_obs_after_reset};
  pendulum_reset_kernel<<<trl_pendulum_num_ctas(N), kPendThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("pendulum_reset_kernel");
}
