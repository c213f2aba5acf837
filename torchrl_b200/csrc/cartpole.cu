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
#include "reduce.cuh"

namespace trl {

constexpr int kCartThreads = 256;
constexpr int kCartWarps = kCartThreads / 32;

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
  int* __restrict__ elapsed;            // (N) env-side step counter (TimeLimit._elapsed_steps)
  const int* __restrict__ step_count;   // (N) collector-side counter or nullptr
  float* __restrict__ reward;           // (N)
  uint8_t* __restrict__ done;           // (N)
  uint8_t* __restrict__ time_limit;     // (N)
  int* __restrict__ action_error;       // (1) set to 1 when an action is neither 0 nor 1
  double* __restrict__ partial;         // (grid, 8) per-CTA column sums / sums of squares, or nullptr
  double* __restrict__ batch_sums;      // (8) reduced sums (written by the last CTA) or nullptr
  double* __restrict__ norm_mean;       // (4) running mean   (merged in-kernel if merge != 0)
  double* __restrict__ norm_var;        // (4)
  double* __restrict__ norm_count;      // (1)
  unsigned* __restrict__ ticket;        // (1) zero-initialised
  int* __restrict__ any_reset;          // (2) double-buffered "some env needs a reset" flag, or nullptr
  const int* __restrict__ t_ptr;        // (1) device step index (selects the flag slot), or nullptr
  long long N;
  float reward_scale;
  int max_episode_steps, max_episode_frames;
  int merge;                            // 1: Chan-merge batch moments into norm_* in the last CTA
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
  __shared__ double sh[kCartWarps][8];
  __shared__ double sred[8];
  const int tid = threadIdx.x;
  const long long n = static_cast<long long>(blockIdx.x) * kCartThreads + tid;
  const bool live = n < p.N;
  float s2[4] = {0.f, 0.f, 0.f, 0.f};
  int local_reset = 0;
  if (live) {
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
    const int el = p.elapsed[n] + 1;
    p.elapsed[n] = el;
    const bool done_dyn = fabs(static_cast<double>(s2[0])) > kXThreshold ||
                          fabs(static_cast<double>(s2[2])) > kThetaThreshold;
    const bool done = done_dyn || el >= p.max_episode_steps;
    p.reward[n] = p.reward_scale;                     // 1.0 on every step, the terminating one included
    p.done[n] = done ? 1 : 0;
    p.time_limit[n] = (done && el == p.max_episode_steps) ? 1 : 0;
    const bool surpass = p.step_count ? (p.step_count[n] + 1 >= p.max_episode_frames) : false;
    local_reset = (done || surpass) ? 1 : 0;
  }
  if (p.any_reset) {
    const int t = p.t_ptr ? *p.t_ptr : 0;
    if (blockIdx.x == 0 && tid == 0) p.any_reset[(t + 1) & 1] = 0;  // slot of the *next* step
    if (__syncthreads_or(local_reset) && tid == 0) atomicOr(&p.any_reset[t & 1], 1);
  }

  if (p.partial) {
    // per-feature batch moments of this CTA's envs: warp shuffles, then thread k folds the warps in order
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double x = static_cast<double>(s2[j]);
      const double ws = warp_sum(x), wq = warp_sum(x * x);
      if (lane == 0) { sh[wid][j] = ws; sh[wid][4 + j] = wq; }
    }
    __syncthreads();
    if (tid < 8) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < kCartWarps; ++w) t += sh[w][tid];
      p.partial[static_cast<long long>(blockIdx.x) * 8 + tid] = t;
    }
    if (last_cta(p.ticket, gridDim.x)) {
      // warp k folds quantity k over the CTAs: lanes stride over CTAs, then one shuffle reduction (fixed order)
      if (wid < 8) {
        double acc = 0.0;
        for (unsigned b = lane; b < gridDim.x; b += 32) acc += __ldcg(p.partial + static_cast<long long>(b) * 8 + wid);
        acc = warp_sum(acc);
        if (lane == 0) sred[wid] = acc;
      }
      __syncthreads();
      if (tid < 4) {
        const double s = sred[tid], q = sred[4 + tid];
        if (p.batch_sums) { p.batch_sums[tid] = s; p.batch_sums[4 + tid] = q; }
        if (p.merge) chan_merge(s, q, static_cast<double>(p.N), *p.norm_count, p.norm_mean[tid], p.norm_var[tid]);
      }
      __syncthreads();   // every thread has read *norm_count
      if (tid == 0 && p.merge) *p.norm_count = *p.norm_count + static_cast<double>(p.N);
    }
  }
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
  TRL_REQUIRE(!partial || ticket, "trl_cartpole_step: statistics requested without a ticket counter");
  TRL_REQUIRE(!(merge_stats && partial) || (norm_mean && norm_var && norm_count),
              "trl_cartpole_step: merge_stats needs norm_mean/var/count");
  TRL_REQUIRE(!t_ptr || any_reset, "trl_cartpole_step: t_ptr given without the any_reset flag");
  CartPoleParams p{state, actions, elapsed, step_count, reward, done, time_limit, action_error, partial, batch_sums,
                   norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, N, reward_scale, max_episode_steps,
                   max_episode_frames, merge_stats};
  cartpole_step_kernel<<<trl_cartpole_num_ctas(N), kCartThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("cartpole_step_kernel");
}
