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
// Layout: state (N,4) fp32 row-major == the raw observation; one thread per env, kCartThreads envs per CTA.
#include "env_common.cuh"

namespace trl {

constexpr int kCartThreads = 256;

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

struct CartPoleParams {
  float* __restrict__ state;            // (N,4) in/out: x, x_dot, theta, theta_dot
  const float* __restrict__ actions;    // (N) 0.0 or 1.0
  int* __restrict__ action_error;       // (1) set to 1 when an action is neither 0 nor 1
  EnvStepFields env;                    // D = 4
};

// One Euler step of gym's CartPoleEnv.step in fp64, every operation rounded once, in gym's evaluation order.
__device__ __forceinline__ void cartpole_dynamics(const float s[4], double force, float out[4]) {
  const double x = s[0], x_dot = s[1], theta = s[2], theta_dot = s[3];
  const double costh = cos(theta), sinth = sin(theta);
  const double temp =
      __ddiv_rn(__dadd_rn(force, __dmul_rn(__dmul_rn(kPoleMassLength, __dmul_rn(theta_dot, theta_dot)), sinth)),
                kTotalMass);
  const double denom =
      __dmul_rn(kLength, __dadd_rn(kFourThirds, -__ddiv_rn(__dmul_rn(kMassPole, __dmul_rn(costh, costh)), kTotalMass)));
  const double thetaacc = __ddiv_rn(__dadd_rn(__dmul_rn(kGravity, sinth), -__dmul_rn(costh, temp)), denom);
  const double xacc = __dadd_rn(temp, -__ddiv_rn(__dmul_rn(__dmul_rn(kPoleMassLength, thetaacc), costh), kTotalMass));
  out[0] = static_cast<float>(__dadd_rn(x, __dmul_rn(kTau, x_dot)));          // positions use the old velocities
  out[1] = static_cast<float>(__dadd_rn(x_dot, __dmul_rn(kTau, xacc)));
  out[2] = static_cast<float>(__dadd_rn(theta, __dmul_rn(kTau, theta_dot)));
  out[3] = static_cast<float>(__dadd_rn(theta_dot, __dmul_rn(kTau, thetaacc)));
}

__global__ void __launch_bounds__(kCartThreads) cartpole_step_kernel(const CartPoleParams p) {
  const EnvStepFields& f = p.env;
  const long long n = static_cast<long long>(blockIdx.x) * kCartThreads + threadIdx.x;
  float s2[4] = {0.f, 0.f, 0.f, 0.f};
  bool local_reset = false;
  if (n < f.N) {
    float s[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j] = p.state[n * 4 + j];
    const float a = p.actions[n];
    if (a == 1.0f || a == 0.0f) {
      cartpole_dynamics(s, a == 1.0f ? kForceMag : -kForceMag, s2);
    } else {
      // not a CartPole action: flag it for the host and leave this env's state where it was
      atomicOr(p.action_error, 1);
#pragma unroll
      for (int j = 0; j < 4; ++j) s2[j] = s[j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) p.state[n * 4 + j] = s2[j];
    const bool terminal = fabs(static_cast<double>(s2[0])) > kXThreshold ||
                          fabs(static_cast<double>(s2[2])) > kThetaThreshold;
    // reward 1.0 on every step, the terminating one included
    local_reset = env_row_end(f, n, terminal, f.reward_scale);
  }
  update_any_reset(f, local_reset);
  if (f.partial) env_moments<4, kCartThreads>(f, s2);
}

}  // namespace trl

TRL_API int trl_cartpole_num_ctas(int64_t N) {
  return static_cast<int>((N + trl::kCartThreads - 1) / trl::kCartThreads);
}

TRL_API int trl_cartpole_step(float* state, const float* actions, int* elapsed, const int* step_count, float* reward,
                              uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                              double* batch_sums, double* norm_mean, double* norm_var, double* norm_count,
                              unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N, float reward_scale,
                              int max_episode_steps, int max_episode_frames, int merge_stats, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && max_episode_steps >= 1, "trl_cartpole_step: bad sizes N=%lld max_episode_steps=%d",
              (long long)N, max_episode_steps);
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(state && actions && elapsed && reward && done && time_limit && action_error,
              "trl_cartpole_step: null pointer");
  CartPoleParams p{state, actions, action_error,
                   {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean, norm_var, norm_count,
                    ticket, any_reset, t_ptr, N, reward_scale, max_episode_steps, max_episode_frames, merge_stats}};
  if (const int e = check_env_step("trl_cartpole_step", p.env)) return e;
  cartpole_step_kernel<<<trl_cartpole_num_ctas(N), kCartThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("cartpole_step_kernel");
}
