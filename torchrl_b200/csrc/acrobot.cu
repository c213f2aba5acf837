// acrobot.cu -- K1 for the classic-control Acrobot-v1: N envs advance (and reset) in one launch.
//
// Replaces, for N Acrobot envs held on the device, the per-env Python chain
//   gym.make("Acrobot-v1") -> AcrobotEnv.step / reset   /root/reference/torchrl/env/get_env.py:53
//   TimeLimitAugment.step                              /root/reference/torchrl/env/base_wrapper.py:152-156
//   RewardShift.reward                                 /root/reference/torchrl/env/base_wrapper.py:37-41
//   VecEnv.step / partial_reset                        /root/reference/torchrl/env/vecenv.py:47-61
// and, like csrc/pendulum.cu, accumulates the batch moments NormObs needs (base_wrapper.py:75-82, :44-60).
// The dynamics are gym's "book" Acrobot without torque noise: one RK4 step of _dsdt over [0, dt], the angles wrapped into
// [-pi, pi] by gym's loop and the velocities bounded; oracle/acrobot.py is the NumPy statement this file must agree with.
//
// Precision: the physical state (theta1, theta2, dtheta1, dtheta2) is fp64 as in gym; every fp64 operation is rounded
// once in gym's evaluation order (explicit __dadd_rn / __dmul_rn / __ddiv_rn, so -fmad=true cannot contract them); the
// observation (cos theta1, sin theta1, cos theta2, sin theta2, dtheta1, dtheta2) is rounded to fp32 once.
//
// Layout: phys (N,4) fp64, obs (N,6) fp32 raw observation; one thread per env (env_step_kernel<Acrobot>).  The reset has
// its own kernel (env_reset_kernel<Acrobot>) because the observation is not the state: collect_finalize's in-kernel
// reset cannot serve it.
#include "env_common.cuh"

namespace trl {

// gym's AcrobotEnv constants (classic_control/acrobot.py)
constexpr double kAcroDt = 0.2;
constexpr double kAcroL1 = 1.0;       // LINK_LENGTH_1
constexpr double kAcroM1 = 1.0;       // LINK_MASS_1
constexpr double kAcroM2 = 1.0;       // LINK_MASS_2
constexpr double kAcroLc1 = 0.5;      // LINK_COM_POS_1
constexpr double kAcroLc2 = 0.5;      // LINK_COM_POS_2
constexpr double kAcroI1 = 1.0;       // LINK_MOI
constexpr double kAcroI2 = 1.0;
constexpr double kAcroG = 9.8;
constexpr double kAcroPi = 3.141592653589793;
constexpr double kAcroMaxVel1 = 4.0 * kAcroPi;
constexpr double kAcroMaxVel2 = 9.0 * kAcroPi;
// the constant sub-expressions of _dsdt, grouped as Python evaluates them (left to right, ** before * before +)
constexpr double kAcroHalfPi = kAcroPi / 2.0;
constexpr double kAcroD1a = kAcroM1 * (kAcroLc1 * kAcroLc1);                            // m1 * lc1**2
constexpr double kAcroD1b = kAcroL1 * kAcroL1 + kAcroLc2 * kAcroLc2;                    // l1**2 + lc2**2
constexpr double kAcroD1c = 2.0 * kAcroL1 * kAcroLc2;                                   // 2 * l1 * lc2
constexpr double kAcroLc2Sq = kAcroLc2 * kAcroLc2;                                      // lc2**2
constexpr double kAcroL1Lc2 = kAcroL1 * kAcroLc2;                                       // l1 * lc2
constexpr double kAcroPhi2 = kAcroM2 * kAcroLc2 * kAcroG;                               // m2 * lc2 * g
constexpr double kAcroPhi1a = -kAcroM2 * kAcroL1 * kAcroLc2;                            // -m2 * l1 * lc2
constexpr double kAcroPhi1b = 2.0 * kAcroM2 * kAcroL1 * kAcroLc2;                       // 2 * m2 * l1 * lc2
constexpr double kAcroPhi1c = (kAcroM1 * kAcroLc1 + kAcroM2 * kAcroL1) * kAcroG;        // (m1 lc1 + m2 l1) * g
constexpr double kAcroDd2a = kAcroM2 * kAcroL1 * kAcroLc2;                              // m2 * l1 * lc2
constexpr double kAcroDd2b = kAcroM2 * kAcroLc2Sq + kAcroI2;                            // m2 * lc2**2 + I2

// AcrobotEnv._dsdt ("book") of the state s with torque a: (dtheta1, dtheta2, ddtheta1, ddtheta2)
__device__ __forceinline__ void acrobot_dsdt(const double (&s)[4], double a, double (&ds)[4]) {
  const double theta1 = s[0], theta2 = s[1], dtheta1 = s[2], dtheta2 = s[3];
  const double c2 = cos(theta2), s2 = sin(theta2);
  const double d1 = __dadd_rn(__dadd_rn(__dadd_rn(kAcroD1a, __dmul_rn(kAcroM2, __dadd_rn(kAcroD1b,
                                                                                         __dmul_rn(kAcroD1c, c2)))),
                                        kAcroI1),
                              kAcroI2);
  const double d2 = __dadd_rn(__dmul_rn(kAcroM2, __dadd_rn(kAcroLc2Sq, __dmul_rn(kAcroL1Lc2, c2))), kAcroI2);
  const double phi2 = __dmul_rn(kAcroPhi2, cos(__dadd_rn(__dadd_rn(theta1, theta2), -kAcroHalfPi)));
  const double t1 = __dmul_rn(__dmul_rn(kAcroPhi1a, __dmul_rn(dtheta2, dtheta2)), s2);
  const double t2 = __dmul_rn(__dmul_rn(__dmul_rn(kAcroPhi1b, dtheta2), dtheta1), s2);
  const double t3 = __dmul_rn(kAcroPhi1c, cos(__dadd_rn(theta1, -kAcroHalfPi)));
  const double phi1 = __dadd_rn(__dadd_rn(__dadd_rn(t1, -t2), t3), phi2);
  const double num = __dadd_rn(__dadd_rn(__dadd_rn(a, __dmul_rn(__ddiv_rn(d2, d1), phi1)),
                                         -__dmul_rn(__dmul_rn(kAcroDd2a, __dmul_rn(dtheta1, dtheta1)), s2)),
                               -phi2);
  const double ddtheta2 = __ddiv_rn(num, __dadd_rn(kAcroDd2b, -__ddiv_rn(__dmul_rn(d2, d2), d1)));
  const double ddtheta1 = __ddiv_rn(-__dadd_rn(__dmul_rn(d2, ddtheta2), phi1), d1);
  ds[0] = dtheta1;
  ds[1] = dtheta2;
  ds[2] = ddtheta1;
  ds[3] = ddtheta2;
}

// gym's wrap(x, -pi, pi): whole turns added or removed one at a time (fmod / remainder would round differently).  A
// non-finite x is returned as it is (gym's loop never ends on an infinity).
__device__ __forceinline__ double acrobot_wrap(double x) {
  constexpr double lo = -kAcroPi, hi = kAcroPi, diff = hi - lo;
  if (!isfinite(x)) return x;
  while (x > hi) x = __dadd_rn(x, -diff);
  while (x < lo) x = __dadd_rn(x, diff);
  return x;
}

// One AcrobotEnv.step of the state s with torque a: rk4(_dsdt, s + [a], [0, dt]), wrap, bound.
__device__ __forceinline__ void acrobot_dynamics(double (&s)[4], double a) {
  constexpr double dt2 = kAcroDt / 2.0, dt6 = kAcroDt / 6.0;
  double k1[4], k2[4], k3[4], k4[4], y[4];
  acrobot_dsdt(s, a, k1);
#pragma unroll
  for (int j = 0; j < 4; ++j) y[j] = __dadd_rn(s[j], __dmul_rn(dt2, k1[j]));
  acrobot_dsdt(y, a, k2);
#pragma unroll
  for (int j = 0; j < 4; ++j) y[j] = __dadd_rn(s[j], __dmul_rn(dt2, k2[j]));
  acrobot_dsdt(y, a, k3);
#pragma unroll
  for (int j = 0; j < 4; ++j) y[j] = __dadd_rn(s[j], __dmul_rn(kAcroDt, k3[j]));
  acrobot_dsdt(y, a, k4);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const double sum = __dadd_rn(__dadd_rn(__dadd_rn(k1[j], __dmul_rn(2.0, k2[j])), __dmul_rn(2.0, k3[j])), k4[j]);
    s[j] = __dadd_rn(s[j], __dmul_rn(dt6, sum));
  }
  s[0] = acrobot_wrap(s[0]);
  s[1] = acrobot_wrap(s[1]);
  s[2] = fmin(fmax(s[2], -kAcroMaxVel1), kAcroMaxVel1);
  s[3] = fmin(fmax(s[3], -kAcroMaxVel2), kAcroMaxVel2);
}

struct Acrobot {
  using State = double;
  static constexpr int kPhys = 4, kObs = 6;
  // 0.0, 1.0 or 2.0: torque -1, 0, +1
  static __device__ __forceinline__ bool accepts(float a) { return a == 0.0f || a == 1.0f || a == 2.0f; }
  // _terminal: -cos(theta1) - cos(theta2 + theta1) > 1; reward -1, or 0 on the terminal step
  static __device__ __forceinline__ double step(double (&s)[kPhys], float a, bool& terminal) {
    acrobot_dynamics(s, static_cast<double>(a) - 1.0);
    terminal = __dadd_rn(-cos(s[0]), -cos(__dadd_rn(s[1], s[0]))) > 1.0;
    return terminal ? 0.0 : -1.0;
  }
  // not an Acrobot action: reward 0, no terminal, and the state and observation stay where they were
  static __device__ __forceinline__ float refused(const double (&)[kPhys], float, bool&) { return 0.f; }
  // every state component from U(-0.1, 0.1): 0.1 (2U - 1) in fp64 from the counter hash of (seed, episode, component)
  static __device__ __forceinline__ void reset_state(unsigned seed, unsigned ep, double (&s)[kPhys]) {
#pragma unroll
    for (int j = 0; j < kPhys; ++j)
      s[j] = __dmul_rn(0.1, __dadd_rn(__dmul_rn(2.0, double(counter_uniform(seed, ep, j))), -1.0));
  }
  static __device__ __forceinline__ void observe(const double (&s)[kPhys], float (&o)[kObs]) {
    o[0] = static_cast<float>(cos(s[0]));
    o[1] = static_cast<float>(sin(s[0]));
    o[2] = static_cast<float>(cos(s[1]));
    o[3] = static_cast<float>(sin(s[1]));
    o[4] = static_cast<float>(s[2]);
    o[5] = static_cast<float>(s[3]);
  }
};

}  // namespace trl

TRL_API int trl_acrobot_num_ctas(int64_t N) { return trl::env_row_ctas(N); }

TRL_API int trl_acrobot_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count,
                             float* reward, uint8_t* done, uint8_t* time_limit, int* action_error, double* partial,
                             double* batch_sums, double* norm_mean, double* norm_var, double* norm_count,
                             unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N, float reward_scale,
                             int max_episode_steps, int max_episode_frames, int merge_stats, void* stream) {
  return trl::launch_env_step<trl::Acrobot>(
      "trl_acrobot_step", "acrobot_step_kernel",
      {phys, obs, actions, action_error,
       {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean, norm_var, norm_count, ticket,
        any_reset, t_ptr, N, reward_scale, max_episode_steps, max_episode_frames, merge_stats}},
      stream);
}

TRL_API int trl_acrobot_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                              const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                              const int* any_reset, const int* t_ptr, const double* norm_mean, const double* norm_var,
                              int64_t N, double clip, int raw_obs_after_reset, void* stream) {
  return trl::launch_env_reset<trl::Acrobot>(
      "trl_acrobot_reset", "acrobot_reset_kernel",
      {phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob, any_reset, t_ptr, norm_mean, norm_var,
       N, clip, raw_obs_after_reset},
      stream);
}
