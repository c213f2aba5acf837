// mountain_car.cu -- K1 for the classic-control MountainCar-v0 and MountainCarContinuous-v0: N envs advance (and reset)
// in one launch.
//
// Replaces, for N Mountain Car envs held on the device, the per-env Python chain
//   gym.make("MountainCar-v0" / "MountainCarContinuous-v0") -> step / reset   /root/reference/torchrl/env/get_env.py:53
//   NormAct.action (continuous variant)                                       /root/reference/torchrl/env/continuous_wrapper.py:18-20
//   TimeLimitAugment.step                                                     /root/reference/torchrl/env/base_wrapper.py:152-156
//   RewardShift.reward                                                        /root/reference/torchrl/env/base_wrapper.py:37-41
//   VecEnv.step / partial_reset                                               /root/reference/torchrl/env/vecenv.py:47-61
// and, like csrc/pendulum.cu, accumulates the batch moments NormObs needs (base_wrapper.py:75-82, :44-60).
// One env struct serves both ids; the variant is a template parameter chosen by the entry point's `continuous` flag.
// oracle/mountain_car.py is the NumPy statement this file must agree with.
//
// Precision: the physical state (position, velocity) is fp64; the continuous force is NormAct's affine map evaluated in
// fp32 (explicitly rounded, so -fmad=true cannot contract it) and widened exactly before it meets the fp64 `power`
// (NumPy 1.x promotion); every fp64 operation is rounded once in gym's order; observation and reward are rounded to fp32
// once.
//
// Layout: phys (N,2) fp64, obs (N,2) fp32 raw observation; one thread per env (env_step_kernel<MountainCar<...>>).  The
// reset has its own kernel (env_reset_kernel<MountainCar<false>>, for both ids) because the observation is not the
// state (it is the fp32 rounding of it).
#include "env_common.cuh"

namespace trl {

// gym's MountainCarEnv / Continuous_MountainCarEnv constants (classic_control/mountain_car.py,
// continuous_mountain_car.py)
constexpr double kCarMinPosition = -1.2;
constexpr double kCarMaxPosition = 0.6;
constexpr double kCarMaxSpeed = 0.07;
constexpr double kCarGoalV0 = 0.5;            // MountainCar-v0's goal_position
constexpr double kCarGoalCont = 0.45;         // MountainCarContinuous-v0's goal_position
constexpr double kCarForce = 0.001;           // v0: (action - 1) * force
constexpr double kCarGravity = 0.0025;
constexpr double kCarPower = 0.0015;          // continuous: force * power

// NormAct (continuous_wrapper.py:18-20) with lb = -1, ub = 1, in fp32: clip(lb + (a + 1) * 0.5 * (ub - lb), lb, ub)
__device__ __forceinline__ float car_action(float a) {
  const float lb = -1.0f, ub = 1.0f;
  const float u = __fadd_rn(lb, __fmul_rn(__fmul_rn(__fadd_rn(a, 1.0f), 0.5f), __fadd_rn(ub, -lb)));
  return fminf(fmaxf(u, lb), ub);
}

template <bool kContinuous>
struct MountainCar {
  using State = double;
  static constexpr int kPhys = 2, kObs = 2;
  // v0: 0.0, 1.0 or 2.0; continuous: policy-space actions, finite
  static __device__ __forceinline__ bool accepts(float a) {
    return kContinuous ? isfinite(a) : (a == 0.0f || a == 1.0f || a == 2.0f);
  }
  // v0: -1 per step; continuous: 100 on reaching the goal, minus 0.1 * action[0]**2
  static __device__ __forceinline__ double step(double (&s)[kPhys], float a, bool& terminal) {
    double pos = s[0], vel = s[1];
    const double c = cos(__dmul_rn(3.0, pos));
    double act = 0.0;                       // the continuous env's action[0], widened exactly
    if (kContinuous) {
      act = static_cast<double>(car_action(a));
      const double force = fmin(fmax(act, -1.0), 1.0);
      vel = __dadd_rn(vel, __dadd_rn(__dmul_rn(force, kCarPower), -__dmul_rn(kCarGravity, c)));
    } else {
      vel = __dadd_rn(vel, __dadd_rn(__dmul_rn(static_cast<double>(a) - 1.0, kCarForce), __dmul_rn(c, -kCarGravity)));
    }
    vel = fmin(fmax(vel, -kCarMaxSpeed), kCarMaxSpeed);
    pos = fmin(fmax(__dadd_rn(pos, vel), kCarMinPosition), kCarMaxPosition);
    if (pos == kCarMinPosition && vel < 0.0) vel = 0.0;       // the left wall stops the car
    terminal = pos >= (kContinuous ? kCarGoalCont : kCarGoalV0) && vel >= 0.0;
    s[0] = pos;
    s[1] = vel;
    return kContinuous ? __dadd_rn(terminal ? 100.0 : 0.0, -__dmul_rn(__dmul_rn(act, act), 0.1)) : -1.0;
  }
  // not an action of this env: reward 0, no terminal, and the state and observation stay where they were
  static __device__ __forceinline__ float refused(const double (&)[kPhys], float, bool&) { return 0.f; }
  // position from U(-0.6, -0.4) as -0.6 + 0.2 U in fp64 from the counter hash of (seed, episode, 0); velocity 0
  static __device__ __forceinline__ void reset_state(unsigned seed, unsigned ep, double (&s)[kPhys]) {
    s[0] = __dadd_rn(-0.6, __dmul_rn(0.2, double(counter_uniform(seed, ep, 0))));
    s[1] = 0.0;
  }
  static __device__ __forceinline__ void observe(const double (&s)[kPhys], float (&o)[kObs]) {
    o[0] = static_cast<float>(s[0]);
    o[1] = static_cast<float>(s[1]);
  }
};

}  // namespace trl

TRL_API int trl_mountain_car_num_ctas(int64_t N) { return trl::env_row_ctas(N); }

TRL_API int trl_mountain_car_step(double* phys, float* obs, const float* actions, int* elapsed, const int* step_count,
                                  float* reward, uint8_t* done, uint8_t* time_limit, int* action_error,
                                  double* partial, double* batch_sums, double* norm_mean, double* norm_var,
                                  double* norm_count, unsigned* ticket, int* any_reset, const int* t_ptr, int64_t N,
                                  float reward_scale, int max_episode_steps, int max_episode_frames, int merge_stats,
                                  int continuous, void* stream) {
  using namespace trl;
  // refused after bad sizes (launch_env_step's first check) and before everything else
  TRL_REQUIRE(continuous == 0 || continuous == 1 || N < 0 || max_episode_steps < 1,
              "trl_mountain_car_step: continuous must be 0 or 1, got %d", continuous);
  const EnvStepParams<double> p{phys, obs, actions, action_error,
                                {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean,
                                 norm_var, norm_count, ticket, any_reset, t_ptr, N, reward_scale, max_episode_steps,
                                 max_episode_frames, merge_stats}};
  return continuous == 1
             ? launch_env_step<MountainCar<true>>("trl_mountain_car_step", "mountain_car_step_kernel", p, stream)
             : launch_env_step<MountainCar<false>>("trl_mountain_car_step", "mountain_car_step_kernel", p, stream);
}

TRL_API int trl_mountain_car_reset(double* phys, float* obs, int* elapsed, unsigned* episode, const unsigned* seeds,
                                   const uint8_t* mask, const int* step_count, const float* next_norm, float* cur_ob,
                                   const int* any_reset, const int* t_ptr, const double* norm_mean,
                                   const double* norm_var, int64_t N, double clip, int raw_obs_after_reset,
                                   void* stream) {
  return trl::launch_env_reset<trl::MountainCar<false>>(
      "trl_mountain_car_reset", "mountain_car_reset_kernel",
      {phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob, any_reset, t_ptr, norm_mean, norm_var,
       N, clip, raw_obs_after_reset},
      stream);
}
