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
// Layout: phys (N,2) fp64, obs (N,3) fp32 raw observation; one thread per env (env_step_kernel<Pendulum>).  The reset
// has its own kernel (env_reset_kernel<Pendulum>) because the observation is not the state: collect_finalize's
// in-kernel reset cannot serve it.
#include "env_common.cuh"

namespace trl {

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

struct Pendulum {
  using State = double;
  static constexpr int kPhys = 2, kObs = 3;
  static __device__ __forceinline__ bool accepts(float a) { return isfinite(a); }
  // no terminal state: only the time limit ends an episode; the reward is minus gym's cost
  static __device__ __forceinline__ double step(double (&s)[kPhys], float a, bool&) {
    const double th = s[0], thdot = s[1];
    const double u = static_cast<double>(pend_torque(a));
    const double an = pend_angle_normalize(th);
    const double cost = __dadd_rn(__dadd_rn(__dmul_rn(an, an), __dmul_rn(0.1, __dmul_rn(thdot, thdot))),
                                  __dmul_rn(0.001, __dmul_rn(u, u)));
    double nthdot =
        __dadd_rn(thdot, __dmul_rn(__dadd_rn(__dmul_rn(kGravTerm, sin(th)), __dmul_rn(kTorqueTerm, u)), kPendDt));
    nthdot = fmin(fmax(nthdot, -kPendMaxSpeed), kPendMaxSpeed);
    s[0] = __dadd_rn(th, __dmul_rn(nthdot, kPendDt));   // v1: the clipped velocity moves the angle
    s[1] = nthdot;
    return -cost;
  }
  // not an action: reward 0, no terminal, and the state and observation stay where they were
  static __device__ __forceinline__ float refused(const double (&)[kPhys], float, bool&) { return 0.f; }
  // theta ~ U(-pi, pi), theta_dot ~ U(-1, 1) from the counter hash of (seed, episode, component)
  static __device__ __forceinline__ void reset_state(unsigned seed, unsigned ep, double (&s)[kPhys]) {
    s[0] = __dmul_rn(kPi, __dadd_rn(__dmul_rn(2.0, double(counter_uniform(seed, ep, 0))), -1.0));
    s[1] = __dadd_rn(__dmul_rn(2.0, double(counter_uniform(seed, ep, 1))), -1.0);
  }
  static __device__ __forceinline__ void observe(const double (&s)[kPhys], float (&o)[kObs]) {
    o[0] = static_cast<float>(cos(s[0]));
    o[1] = static_cast<float>(sin(s[0]));
    o[2] = static_cast<float>(s[1]);
  }
};

}  // namespace trl

TRL_API int trl_pendulum_num_ctas(int64_t N) { return trl::env_row_ctas(N); }

TRL_API int trl_pendulum_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count,
                              float* reward, uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                              double* batch_sums, double* norm_mean, double* norm_var, double* norm_count,
                              unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N, float reward_scale,
                              int max_episode_steps, int max_episode_frames, int merge_stats, void* stream) {
  return trl::launch_env_step<trl::Pendulum>(
      "trl_pendulum_step", "pendulum_step_kernel",
      {phys, obs, actions, action_error,
       {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean, norm_var, norm_count, ticket,
        any_reset, t_ptr, N, reward_scale, max_episode_steps, max_episode_frames, merge_stats}},
      stream);
}

TRL_API int trl_pendulum_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                               const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                               const int* any_reset, const int* t_ptr, const double* norm_mean,
                               const double* norm_var, int64_t N, double clip, int raw_obs_after_reset,
                               void* stream) {
  return trl::launch_env_reset<trl::Pendulum>(
      "trl_pendulum_reset", "pendulum_reset_kernel",
      {phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob, any_reset, t_ptr, norm_mean, norm_var,
       N, clip, raw_obs_after_reset},
      stream);
}
