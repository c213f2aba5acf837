// env_common.cuh -- what the device env kernels share: the reset counter hash, the fields and bookkeeping of a step
// (TimeLimitAugment, the collector's reset flag, NormObs's batch moments), the collector's next-observation rule, and
// the step and own-reset kernels of the one-thread-per-env classic-control envs with their launches.  Each of those
// envs' .cu files keeps its physics in an env struct (see env_step_kernel) and its literal TRL_API entry points.
#pragma once
#include <type_traits>

#include "reduce.cuh"

namespace trl {

// block size of the kernels that run one thread per env
constexpr int kEnvRowThreads = 256;
inline int env_row_ctas(int64_t N) { return static_cast<int>((N + kEnvRowThreads - 1) / kEnvRowThreads); }

// ---- the reset counter hash (oracle/synth_env.py:hash_uniform) ------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t counter_hash(uint32_t seed, uint32_t episode, uint32_t j) {
  uint32_t x = seed * 0x9E3779B1u + episode * 0x85EBCA77u + j * 0xC2B2AE3Du + 0x27D4EB2Fu;
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return x;
}
// U(seed, episode, j): 24 random bits / 2^24 -- exact in fp32
__host__ __device__ __forceinline__ float counter_uniform(uint32_t seed, uint32_t episode, uint32_t j) {
  return float(counter_hash(seed, episode, j) >> 8) * (1.0f / 16777216.0f);
}
__host__ __device__ __forceinline__ float reset_value(uint32_t seed, uint32_t episode, uint32_t j, double init_scale) {
  // INIT_SCALE * (2u - 1) evaluated in fp64 then rounded once, like the float64 oracle cast to fp32
  return float(init_scale * (2.0 * double(counter_uniform(seed, episode, j)) - 1.0));
}

// ---- one step of N envs ---------------------------------------------------------------------------------------------
// The fields every env step kernel has besides its physics; D below is the observation's feature count.
struct EnvStepFields {
  int* __restrict__ elapsed;            // (N) env-side step counter (TimeLimit._elapsed_steps)
  const int* __restrict__ step_count;   // (N) collector-side counter or nullptr
  float* __restrict__ reward;           // (N)
  uint8_t* __restrict__ done;           // (N)
  uint8_t* __restrict__ time_limit;     // (N)
  double* __restrict__ partial;         // (grid, 2*D) per-CTA column sums / sums of squares, or nullptr
  double* __restrict__ batch_sums;      // (2*D) reduced sums (written by the last CTA) or nullptr
  double* __restrict__ norm_mean;       // (D) running mean   (merged in-kernel if merge != 0)
  double* __restrict__ norm_var;        // (D)
  double* __restrict__ norm_count;      // (1)
  unsigned* __restrict__ ticket;        // (1) zero-initialised
  int* __restrict__ any_reset;          // (2) double-buffered "some env needs a reset" flag, or nullptr
  const int* __restrict__ t_ptr;        // (1) device step index (selects the flag slot), or nullptr
  long long N;
  float reward_scale;
  int max_episode_steps, max_episode_frames;
  int merge;                            // 1: Chan-merge batch moments into norm_* in the last CTA
};

// The step arguments' rules that every env step shares; `fn` names the entry point in the message.
inline int check_env_step(const char* fn, const EnvStepFields& f) {
  TRL_REQUIRE(!f.partial || f.ticket, "%s: statistics requested without a ticket counter", fn);
  TRL_REQUIRE(!(f.merge && f.partial) || (f.norm_mean && f.norm_var && f.norm_count),
              "%s: merge_stats needs norm_mean/var/count", fn);
  TRL_REQUIRE(!f.t_ptr || f.any_reset, "%s: t_ptr given without the any_reset flag", fn);
  return TRL_OK;
}

// The end of env n's step (TimeLimitAugment): counts the step and stores its reward (already scaled), done and
// time_limit.  Returns whether the env needs a reset: done, or cut by the collector's max_episode_frames ("surpass").
__device__ __forceinline__ bool env_row_end(const EnvStepFields& f, long long n, bool terminal, float reward) {
  const int el = f.elapsed[n] + 1;
  f.elapsed[n] = el;
  const bool done = terminal || el >= f.max_episode_steps;
  f.reward[n] = reward;
  f.done[n] = done ? 1 : 0;
  f.time_limit[n] = (done && el == f.max_episode_steps) ? 1 : 0;
  const bool surpass = f.step_count ? (f.step_count[n] + 1 >= f.max_episode_frames) : false;
  return done || surpass;
}

// any_reset[t & 1] |= "an env of this CTA needs a reset", and CTA 0 clears the slot of the next step.  Called by every
// thread of the CTA (a barrier).
__device__ __forceinline__ void update_any_reset(const EnvStepFields& f, bool local_reset) {
  if (f.any_reset) {
    const int t = f.t_ptr ? *f.t_ptr : 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) f.any_reset[(t + 1) & 1] = 0;  // slot of the *next* step
    if (__syncthreads_or(local_reset) && threadIdx.x == 0) atomicOr(&f.any_reset[t & 1], 1);
  }
}

// The last CTA's tail for feature j of D, given the batch's sum s and sum of squares q: batch_sums, then the merge.
__device__ __forceinline__ void merge_feature(const EnvStepFields& f, int D, int j, double s, double q) {
  if (f.batch_sums) { f.batch_sums[j] = s; f.batch_sums[D + j] = q; }
  if (f.merge) chan_merge(s, q, static_cast<double>(f.N), *f.norm_count, f.norm_mean[j], f.norm_var[j]);
}
// After every merge_feature of the last CTA (called by all its threads): the count grows by the batch.
__device__ __forceinline__ void merge_count(const EnvStepFields& f) {
  __syncthreads();   // every thread has read *norm_count
  if (threadIdx.x == 0 && f.merge) *f.norm_count = *f.norm_count + static_cast<double>(f.N);
}

// NormObs's batch moments for the envs that run one thread per env (kThreads per CTA): x is this thread's observation
// (zeros past N).  Warp shuffles, then thread k folds the warps' value of quantity k in order into this CTA's partial;
// the last CTA's warp k folds quantity k over the CTAs (lanes stride over them, then one shuffle reduction: a fixed
// order) and merges.  Called by every thread.
template <int D, int kThreads>
__device__ __forceinline__ void env_moments(const EnvStepFields& f, const float (&x)[D]) {
  constexpr int kWarps = kThreads / 32;
  __shared__ double sh[kWarps][2 * D];
  __shared__ double sred[2 * D];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
#pragma unroll
  for (int j = 0; j < D; ++j) {
    const double v = static_cast<double>(x[j]);
    const double ws = warp_sum(v), wq = warp_sum(v * v);
    if (lane == 0) { sh[wid][j] = ws; sh[wid][D + j] = wq; }
  }
  __syncthreads();
  if (tid < 2 * D) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += sh[w][tid];
    f.partial[static_cast<long long>(blockIdx.x) * 2 * D + tid] = t;
  }
  if (last_cta(f.ticket, gridDim.x)) {
    if constexpr (2 * D <= kWarps) {
      if (wid < 2 * D) {
        double acc = 0.0;
        for (unsigned b = lane; b < gridDim.x; b += 32)
          acc += __ldcg(f.partial + static_cast<long long>(b) * 2 * D + wid);
        acc = warp_sum(acc);
        if (lane == 0) sred[wid] = acc;
      }
    } else {
      // more quantities than warps (Acrobot's 12 over 8 warps): warp k also folds k + kWarps, ..., in the same order
      for (int k = wid; k < 2 * D; k += kWarps) {
        double acc = 0.0;
        for (unsigned b = lane; b < gridDim.x; b += 32)
          acc += __ldcg(f.partial + static_cast<long long>(b) * 2 * D + k);
        acc = warp_sum(acc);
        if (lane == 0) sred[k] = acc;
      }
    }
    __syncthreads();
    if (tid < D) merge_feature(f, D, tid, sred[tid], sred[D + tid]);
    merge_count(f);
  }
}

// ---- the collector's next observation -------------------------------------------------------------------------------
// Feature j of the observation the policy acts on next: the raw one when `all_raw` (no NormObs, or reference quirk A.1
// (SURVEY.md) after any reset), the raw one normalised and clipped in fp64 when `normalise` (a reset row), else the
// observation the step returned (*carried).
__device__ __forceinline__ float next_observation(bool all_raw, bool normalise, float raw, const float* carried,
                                                  const double* norm_mean, const double* norm_var, int j, double clip) {
  if (all_raw) return raw;
  if (!normalise) return *carried;
  const double y = (static_cast<double>(raw) - norm_mean[j]) / (sqrt(norm_var[j]) + 1e-4);
  return static_cast<float>(fmin(fmax(y, -clip), clip));
}

// ---- the step of a classic-control env: one thread per env --------------------------------------------------------
// Env supplies its physics:
//   using State = double or float;     the physical state's type (float: CartPole, whose fp32 state is its observation)
//   static constexpr int kPhys, kObs;  state and observation widths
//   static __device__ bool accepts(float a);
//   static __device__ double step(State (&s)[kPhys], float a, bool& terminal);  advances s, returns the unscaled reward
//   static __device__ float refused(const State (&s)[kPhys], float reward_scale, bool& terminal);
//                                      the reward (and terminal) of a row whose action was refused; its state stays
//   static __device__ void observe(const State (&s)[kPhys], float (&o)[kObs]);
template <class State>
struct EnvStepParams {
  State* __restrict__ phys;             // (N, kPhys) in/out physical state; for a float State the same array as obs,
                                        // which the kernel reads and writes it through
  float* __restrict__ obs;              // (N, kObs) in/out raw observation
  const float* __restrict__ actions;    // (N) one action per env
  int* __restrict__ action_error;       // (1) set to 1 when an action is refused
  EnvStepFields env;                    // D = kObs
};

// A refused action is flagged for the host; the observation is reloaded (a float State is the observation itself) and
// only the env's refused() decides the row's reward and terminal.
template <class Env>
__global__ void __launch_bounds__(kEnvRowThreads) env_step_kernel(const EnvStepParams<typename Env::State> p) {
  constexpr int P = Env::kPhys, D = Env::kObs;
  constexpr bool kStateIsObs = std::is_same_v<typename Env::State, float>;
  const EnvStepFields& f = p.env;
  const long long n = static_cast<long long>(blockIdx.x) * kEnvRowThreads + threadIdx.x;
  float ob[D] = {};
  bool local_reset = false;
  if (n < f.N) {
    typename Env::State s[P];
#pragma unroll
    for (int j = 0; j < P; ++j) s[j] = kStateIsObs ? p.obs[n * D + j] : p.phys[n * P + j];
    const float a = p.actions[n];
    bool terminal = false;
    float r;
    if (Env::accepts(a)) {
      // one rounded fp64 product (nothing is added to it, so it cannot contract); CartPole's x 1.0 folds away
      r = static_cast<float>(Env::step(s, a, terminal) * static_cast<double>(f.reward_scale));
      if constexpr (!kStateIsObs) {
#pragma unroll
        for (int j = 0; j < P; ++j) p.phys[n * P + j] = s[j];
      }
      Env::observe(s, ob);
    } else {
      atomicOr(p.action_error, 1);
      r = Env::refused(s, f.reward_scale, terminal);
#pragma unroll
      for (int j = 0; j < D; ++j) ob[j] = kStateIsObs ? s[j] : p.obs[n * D + j];
    }
#pragma unroll
    for (int j = 0; j < D; ++j) p.obs[n * D + j] = ob[j];
    local_reset = env_row_end(f, n, terminal, r);
  }
  update_any_reset(f, local_reset);
  if (f.partial) env_moments<D, kEnvRowThreads>(f, ob);
}

// The body of a trl_<env>_step entry point `fn` after it has gathered its arguments: the argument checks, then the
// launch of env_step_kernel<Env>; `kernel` names it in a launch error.
template <class Env>
int launch_env_step(const char* fn, const char* kernel, const EnvStepParams<typename Env::State>& p, void* stream) {
  const EnvStepFields& f = p.env;
  TRL_REQUIRE(f.N >= 0 && f.max_episode_steps >= 1, "%s: bad sizes N=%lld max_episode_steps=%d", fn, f.N,
              f.max_episode_steps);
  if (f.N == 0) return TRL_OK;
  TRL_REQUIRE(p.phys && p.obs && p.actions && f.elapsed && f.reward && f.done && f.time_limit && p.action_error,
              "%s: null pointer", fn);
  if (const int e = check_env_step(fn, f)) return e;
  env_step_kernel<Env><<<env_row_ctas(f.N), kEnvRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch(kernel);
}

// ---- the own reset of an env whose observation is not its state -----------------------------------------------------
// An fp64 physical state (N, Env::kPhys) and its fp32 raw observation (N, Env::kObs).  Env supplies, besides the
// physics of env_step_kernel,
//   static __device__ void reset_state(unsigned seed, unsigned episode, double (&s)[kPhys]);
struct SelfResetParams {
  double* __restrict__ phys;              // (N, kPhys)
  float* __restrict__ obs;                // (N, kObs) raw observation
  int* __restrict__ elapsed;              // (N)
  unsigned* __restrict__ episode;         // (N)
  const unsigned* __restrict__ seeds;     // (N)
  const uint8_t* __restrict__ mask;       // (N) envs to reset, or nullptr
  const int* __restrict__ step_count;     // (N) reset where 0 (the collector's path), or nullptr
  // collector path (cur_ob != nullptr): the next observation of every env, as collect_finalize writes it
  const float* __restrict__ next_norm;    // (N, kObs) observation the env step returned (normalised if NormObs)
  float* __restrict__ cur_ob;             // (N, kObs) or nullptr
  const int* __restrict__ any_reset;      // (2) flag written by the step kernel
  const int* __restrict__ t_ptr;          // (1) ring row (selects the flag slot)
  const double* __restrict__ norm_mean;   // (kObs) or nullptr (no NormObs)
  const double* __restrict__ norm_var;    // (kObs)
  long long N;
  double clip;
  int raw_obs_after_reset;                // reference quirk A.1 (SURVEY.md): raw obs for ALL envs after any reset
};

// Env n's reset: selected by step_count == 0, else by mask, else always.  A selected env gets a new state from the
// counter hash of (seed, episode), its raw observation, elapsed = 0 and episode += 1.  With cur_ob, every env's next
// observation is written by collect_finalize's rules (next_observation).
template <class Env>
__device__ __forceinline__ void env_self_reset(const SelfResetParams& p, long long n) {
  constexpr int P = Env::kPhys, D = Env::kObs;
  if (n >= p.N) return;
  const bool sel = p.step_count ? p.step_count[n] == 0 : (p.mask ? p.mask[n] != 0 : true);
  float raw[D];
  if (sel) {
    const unsigned ep = p.episode[n];
    double s[P];
    Env::reset_state(p.seeds[n], ep, s);
    Env::observe(s, raw);
#pragma unroll
    for (int j = 0; j < P; ++j) p.phys[n * P + j] = s[j];
#pragma unroll
    for (int j = 0; j < D; ++j) p.obs[n * D + j] = raw[j];
    p.episode[n] = ep + 1u;
    p.elapsed[n] = 0;
  } else {
#pragma unroll
    for (int j = 0; j < D; ++j) raw[j] = p.obs[n * D + j];
  }
  if (!p.cur_ob) return;
  const bool all_raw = !p.norm_mean || (p.raw_obs_after_reset && p.any_reset[*p.t_ptr & 1]);
#pragma unroll
  for (int j = 0; j < D; ++j) {
    p.cur_ob[n * D + j] =
        next_observation(all_raw, sel, raw[j], p.next_norm + n * D + j, p.norm_mean, p.norm_var, j, p.clip);
  }
}

template <class Env>
__global__ void __launch_bounds__(kEnvRowThreads) env_reset_kernel(const SelfResetParams p) {
  env_self_reset<Env>(p, static_cast<long long>(blockIdx.x) * kEnvRowThreads + threadIdx.x);
}

// The body of a trl_<env>_reset entry point `fn` after it has gathered its arguments: the argument checks, then the
// launch of env_reset_kernel<Env>; `kernel` names it in a launch error.
template <class Env>
int launch_env_reset(const char* fn, const char* kernel, const SelfResetParams& p, void* stream) {
  TRL_REQUIRE(p.N >= 0, "%s: bad size N=%lld", fn, p.N);
  if (p.N == 0) return TRL_OK;
  TRL_REQUIRE(p.phys && p.obs && p.elapsed && p.episode && p.seeds, "%s: null pointer", fn);
  TRL_REQUIRE(!(p.mask && p.step_count), "%s: select envs by mask or by step_count, not both", fn);
  TRL_REQUIRE(!p.cur_ob || (p.step_count && p.next_norm && p.any_reset && p.t_ptr),
              "%s: cur_ob needs step_count, next_norm, any_reset and t_ptr", fn);
  TRL_REQUIRE(!p.norm_mean || p.norm_var, "%s: norm_mean given without norm_var", fn);
  env_reset_kernel<Env><<<env_row_ctas(p.N), kEnvRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch(kernel);
}

}  // namespace trl
