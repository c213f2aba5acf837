// cartpole.cu -- K1 for the classic-control CartPole-v0 / CartPole-v1: N envs advance in one launch.
//
// Replaces, for N CartPole envs held on the device, the per-env Python chain
//   gym.make("CartPole-v1") -> CartPoleEnv.step    /root/reference/torchrl/env/get_env.py:53
//   TimeLimitAugment.step                          /root/reference/torchrl/env/base_wrapper.py:152-156
//   RewardShift.reward                             /root/reference/torchrl/env/base_wrapper.py:37-41
//   VecEnv.step / partial_reset                    /root/reference/torchrl/env/vecenv.py:47-61
// and, like csrc/env_step.cu, accumulates the batch moments NormObs needs (base_wrapper.py:75-82, :44-60).
// The dynamics are gym's closed-form cart-pole with its constants and Euler integrator; oracle/cartpole.py is the
// NumPy statement this file must agree with.
//
// Precision: the state is fp32 (so collect_finalize's in-kernel partial reset serves CartPole unchanged); each step is
// computed in fp64 from the fp32 state with explicitly rounded operations (no contraction into FMAs, which the build's
// -fmad=true would otherwise allow) and rounded to fp32 once.  Thresholds are compared on the rounded state.
//
// Layout: state (N,4) fp32 row-major == the raw observation; one thread per env (env_step_kernel<CartPole>).
#include "env_common.cuh"

namespace trl {

// gym's CartPoleEnv constants (classic_control/cartpole.py), derived quantities computed as gym computes them
constexpr double kGravity = 9.8;
constexpr double kMassCart = 1.0;
constexpr double kMassPole = 0.1;
constexpr double kTotalMass = kMassPole + kMassCart;
constexpr double kLength = 0.5;                       // half the pole's length
constexpr double kPoleMassLength = kMassPole * kLength;
constexpr double kForceMag = 10.0;
constexpr double kTau = 0.02;
constexpr double kFourThirds = 4.0 / 3.0;
constexpr double kThetaThreshold = 12.0 * 2.0 * 3.141592653589793 / 360.0;   // 0.20943951023931953
constexpr double kXThreshold = 2.4;

// One Euler step of gym's CartPoleEnv.step in fp64, every operation rounded once, in gym's evaluation order.
__device__ __forceinline__ void cartpole_dynamics(float (&s)[4], double force) {
  const double x = s[0], x_dot = s[1], theta = s[2], theta_dot = s[3];
  const double costh = cos(theta), sinth = sin(theta);
  const double temp =
      __ddiv_rn(__dadd_rn(force, __dmul_rn(__dmul_rn(kPoleMassLength, __dmul_rn(theta_dot, theta_dot)), sinth)),
                kTotalMass);
  const double denom =
      __dmul_rn(kLength, __dadd_rn(kFourThirds, -__ddiv_rn(__dmul_rn(kMassPole, __dmul_rn(costh, costh)), kTotalMass)));
  const double thetaacc = __ddiv_rn(__dadd_rn(__dmul_rn(kGravity, sinth), -__dmul_rn(costh, temp)), denom);
  const double xacc = __dadd_rn(temp, -__ddiv_rn(__dmul_rn(__dmul_rn(kPoleMassLength, thetaacc), costh), kTotalMass));
  s[0] = static_cast<float>(__dadd_rn(x, __dmul_rn(kTau, x_dot)));            // positions use the old velocities
  s[1] = static_cast<float>(__dadd_rn(x_dot, __dmul_rn(kTau, xacc)));
  s[2] = static_cast<float>(__dadd_rn(theta, __dmul_rn(kTau, theta_dot)));
  s[3] = static_cast<float>(__dadd_rn(theta_dot, __dmul_rn(kTau, thetaacc)));
}

struct CartPole {
  using State = float;                  // the state is the observation
  static constexpr int kPhys = 4, kObs = 4;
  static __device__ __forceinline__ bool accepts(float a) { return a == 1.0f || a == 0.0f; }
  static __device__ __forceinline__ bool terminal(const float (&s)[4]) {
    return fabs(static_cast<double>(s[0])) > kXThreshold || fabs(static_cast<double>(s[2])) > kThetaThreshold;
  }
  // reward 1.0 on every step, the terminating one included
  static __device__ __forceinline__ double step(float (&s)[4], float a, bool& term) {
    cartpole_dynamics(s, a == 1.0f ? kForceMag : -kForceMag);
    term = terminal(s);
    return 1.0;
  }
  // not a CartPole action: the state stays where it was, and its step still counts, ends and pays as one
  static __device__ __forceinline__ float refused(const float (&s)[4], float reward_scale, bool& term) {
    term = terminal(s);
    return reward_scale;
  }
  static __device__ __forceinline__ void observe(const float (&s)[4], float (&o)[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = s[j];
  }
};

}  // namespace trl

TRL_API int trl_cartpole_num_ctas(int64_t N) { return trl::env_row_ctas(N); }

TRL_API int trl_cartpole_step(float* state, const float* actions, int* elapsed, const int* step_count, float* reward,
                              uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                              double* batch_sums, double* norm_mean, double* norm_var, double* norm_count,
                              unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N, float reward_scale,
                              int max_episode_steps, int max_episode_frames, int merge_stats, void* stream) {
  return trl::launch_env_step<trl::CartPole>(
      "trl_cartpole_step", "cartpole_step_kernel",
      {state, state, actions, action_error,
       {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean, norm_var, norm_count, ticket,
        any_reset, t_ptr, N, reward_scale, max_episode_steps, max_episode_frames, merge_stats}},
      stream);
}
