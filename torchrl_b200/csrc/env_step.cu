// env_step.cu -- K1 + K2(statistics half): batched synthetic MuJoCo-shaped env transition.
//
// Replaces, for N independent envs held on the device, the per-env Python chain
//   VecEnv.step / SubProcVecEnv.step        /root/reference/torchrl/env/vecenv.py:53-61, subproc_vecenv.py:123-140
//   NormAct.action                          /root/reference/torchrl/env/continuous_wrapper.py:18-20
//   RewardShift.reward                      /root/reference/torchrl/env/base_wrapper.py:37-41
//   TimeLimitAugment.step                   /root/reference/torchrl/env/base_wrapper.py:152-156
//   VecEnv.partial_reset / seed             /root/reference/torchrl/env/vecenv.py:47-51, 63-65
// and accumulates the batch moments that NormObs needs
//   Normalizer.update_estimate              /root/reference/torchrl/env/base_wrapper.py:75-82 (+ :44-60 Chan merge).
// The dynamics themselves are defined by this build (the reference's physics is third-party
// MuJoCo): see oracle/synth_env.py for the CPU definition this file must agree with.
//
// Layout: state (N,o) fp32 row-major == the raw observation.  One CTA owns ENVS_PER_CTA
// consecutive envs: the (E x o) state tile and (E x a) action tile are contiguous in HBM and
// are staged in shared memory with flat coalesced loads; A (o x o), B (a x o), c live in
// shared memory too (49 KB for o=111).  Thread (e, j) produces s'[e][j].  HBM traffic per
// env-step: read 4(o+a), write 4o + 6 bytes -> HBM/latency-bound, no tensor-core work.
#include "env_common.cuh"

namespace trl {

constexpr int kEnvsPerCta = 32;
constexpr int kEnvThreads = 256;

struct EnvParams {
  float* __restrict__ state;            // (N,o) in/out: s -> s'
  const float* __restrict__ actions;    // (N,a) policy-space actions in [-1,1]
  const float* __restrict__ A;          // (o,o)
  const float* __restrict__ B;          // (a,o)
  const float* __restrict__ c;          // (o)
  const float* __restrict__ lb;         // (a)
  const float* __restrict__ ub;         // (a)
  EnvStepFields env;                    // D = o
  int o, a;
  float rho, eta, ctrl_cost, term_thr;
};

// dynamic smem: A[o*o] B[a*o] c[o] lbub[2a] | s[E*o] u[E*a] s2[E*o]
__global__ void __launch_bounds__(kEnvThreads) synth_env_step_kernel(const EnvParams p) {
  extern __shared__ float sm[];
  const int o = p.o, a = p.a, E = kEnvsPerCta;
  float* sA = sm;
  float* sB = sA + o * o;
  float* sc = sB + a * o;
  float* slb = sc + o;
  float* sub = slb + a;
  float* ss = sub + a;
  float* su = ss + E * o;
  float* s2 = su + E * a;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const EnvStepFields& f = p.env;
  const long long env_base = static_cast<long long>(blockIdx.x) * E;
  const int ne = static_cast<int>(min(static_cast<long long>(E), f.N - env_base));

  for (int i = tid; i < o * o; i += nthr) sA[i] = p.A[i];
  for (int i = tid; i < a * o; i += nthr) sB[i] = p.B[i];
  for (int i = tid; i < o; i += nthr) sc[i] = p.c[i];
  for (int i = tid; i < a; i += nthr) { slb[i] = p.lb[i]; sub[i] = p.ub[i]; }
  const float* gs = p.state + env_base * o;
  for (int i = tid; i < ne * o; i += nthr) ss[i] = gs[i];
  __syncthreads();
  const float* gu = p.actions + env_base * a;
  for (int i = tid; i < ne * a; i += nthr) {
    const int k = i % a;
    // NormAct: lb + (act+1)/2*(ub-lb), clipped to [lb,ub]
    const float scaled = slb[k] + (gu[i] + 1.0f) * 0.5f * (sub[k] - slb[k]);
    su[i] = fminf(fmaxf(scaled, slb[k]), sub[k]);
  }
  __syncthreads();

  for (int idx = tid; idx < ne * o; idx += nthr) {
    const int e = idx / o, j = idx - e * o;
    float z = sc[j];
    const float* se = ss + e * o;
    for (int i = 0; i < o; ++i) z = fmaf(se[i], sA[i * o + j], z);
    const float* ue = su + e * a;
    for (int k = 0; k < a; ++k) z = fmaf(ue[k], sB[k * o + j], z);
    s2[idx] = p.rho * se[j] + p.eta * tanhf(z);
  }
  __syncthreads();

  float* gout = p.state + env_base * o;
  for (int i = tid; i < ne * o; i += nthr) gout[i] = s2[i];

  bool local_reset = false;
  if (tid < ne) {
    const float* ue = su + tid * a;
    float usq = 0.f;
    for (int k = 0; k < a; ++k) usq = fmaf(ue[k], ue[k], usq);
    const float r = s2[tid * o + 0] - p.ctrl_cost * usq;
    local_reset = env_row_end(f, env_base + tid, fabsf(s2[tid * o + 1]) > p.term_thr, r * f.reward_scale);
  }
  update_any_reset(f, local_reset);

  if (f.partial) {
    // per-feature batch moments of this CTA's rows (fp64 accumulation)
    double* pp = f.partial + static_cast<long long>(blockIdx.x) * 2 * o;
    for (int j = tid; j < o; j += nthr) {
      double s = 0.0, q = 0.0;
      for (int e = 0; e < ne; ++e) {
        const double x = static_cast<double>(s2[e * o + j]);
        s += x;
        q += x * x;
      }
      pp[j] = s;
      pp[o + j] = q;
    }
    if (last_cta(f.ticket, gridDim.x)) {
      // fold the per-CTA partials with all threads: thread (part, c) sums CTAs b = part, part+P, ... of
      // column c (c < 2*o), then `part` results are combined in fixed order (deterministic); the previous
      // version walked all CTAs serially in `o` threads and dominated the kernel's latency
      double* sred = reinterpret_cast<double*>(sm);          // tile memory is dead by now: reuse as scratch
      const int C = 2 * o;
      const int P = nthr / C > 0 ? (nthr / C < 8 ? nthr / C : 8) : 1;
      if (C <= nthr) {
        const int part = tid / C, c = tid - part * C;
        if (part < P) {
          double acc = 0.0;
          for (unsigned b = part; b < gridDim.x; b += P) acc += f.partial[static_cast<long long>(b) * C + c];
          sred[part * C + c] = acc;
        }
      }
      __syncthreads();
      for (int j = tid; j < o; j += nthr) {
        double s = 0.0, q = 0.0;
        if (C <= nthr) {
          for (int part = 0; part < P; ++part) { s += sred[part * C + j]; q += sred[part * C + o + j]; }
        } else {
          for (unsigned b = 0; b < gridDim.x; ++b) {
            s += f.partial[static_cast<long long>(b) * C + j];
            q += f.partial[static_cast<long long>(b) * C + o + j];
          }
        }
        merge_feature(f, o, j, s, q);
      }
      merge_count(f);
    }
  }
}

struct ResetParams {
  float* __restrict__ state;      // (N,o)
  int* __restrict__ elapsed;      // (N)
  unsigned* __restrict__ episode; // (N) per-env episode counter
  const unsigned* __restrict__ seeds;  // (N)
  const uint8_t* __restrict__ mask;    // (N) or nullptr = all
  long long N;
  int o;
  double init_scale;
};

__global__ void synth_env_reset_kernel(const ResetParams p) {
  // one warp per env: lanes stride over features
  const long long n = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= p.N) return;
  if (p.mask && !p.mask[n]) return;
  const unsigned seed = p.seeds[n], ep = p.episode[n];
  for (int j = lane; j < p.o; j += 32) p.state[n * p.o + j] = reset_value(seed, ep, j, p.init_scale);
  __syncwarp();
  if (lane == 0) { p.episode[n] = ep + 1u; p.elapsed[n] = 0; }
}

// seeds[i] = seed * n_total + first_env + i   (VecEnv.seed, vecenv.py:63-65), episodes <- 0
__global__ void synth_env_seed_kernel(unsigned* seeds, unsigned* episode, long long N, unsigned seed,
                                      unsigned n_total, unsigned first_env) {
  const long long n = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (n >= N) return;
  seeds[n] = seed * n_total + first_env + static_cast<unsigned>(n);
  episode[n] = 0u;
}

}  // namespace trl

namespace trl {
// dynamic shared memory of synth_env_step_kernel in bytes, in double so that no obs_dim / act_dim overflows it
static double synth_env_smem(int obs_dim, int act_dim) {
  const double o = obs_dim, a = act_dim, E = kEnvsPerCta;
  return sizeof(float) * (o * o + a * o + o + 2 * a + 2 * E * o + E * a);
}
}  // namespace trl

// saturates at INT_MAX, far above anything that fits
TRL_API int trl_synth_env_smem_bytes(int obs_dim, int act_dim) {
  const double b = trl::synth_env_smem(obs_dim, act_dim);
  return b > 2147483647.0 ? 2147483647 : static_cast<int>(b);
}

TRL_API int trl_synth_env_num_ctas(int64_t N) {
  return static_cast<int>((N + trl::kEnvsPerCta - 1) / trl::kEnvsPerCta);
}

TRL_API int trl_synth_env_step(float* state, const float* actions, const float* A, const float* B, const float* c,
                               const float* lb, const float* ub, int* elapsed, const int* step_count, float* reward,
                               uint8_t* done, uint8_t* time_limit, double* partial, double* batch_sums,
                               double* norm_mean, double* norm_var, double* norm_count, unsigned* ticket,
                               int* any_reset, const int* t_ptr, int64_t N, int obs_dim, int act_dim, float rho,
                               float eta, float ctrl_cost, float term_thr, float reward_scale, int max_episode_steps,
                               int max_episode_frames, int merge_stats, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && obs_dim >= 2 && act_dim >= 1, "trl_synth_env_step: bad sizes N=%lld o=%d a=%d", (long long)N,
              obs_dim, act_dim);
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(state && actions && A && B && c && lb && ub && elapsed && reward && done && time_limit,
              "trl_synth_env_step: null pointer");
  EnvParams p{state, actions, A, B, c, lb, ub,
              {elapsed, step_count, reward, done, time_limit, partial, batch_sums, norm_mean, norm_var, norm_count,
               ticket, any_reset, t_ptr, N, reward_scale, max_episode_steps, max_episode_frames, merge_stats},
              obs_dim, act_dim, rho, eta, ctrl_cost, term_thr};
  if (const int e = check_env_step("trl_synth_env_step", p.env)) return e;
  const double smem_bytes = synth_env_smem(obs_dim, act_dim);
  TRL_REQUIRE(smem_bytes <= 227 * 1024, "trl_synth_env_step: obs_dim %d act_dim %d need %.0f B of shared memory "
              "(> 227 KB)", obs_dim, act_dim, smem_bytes);
  const int smem = static_cast<int>(smem_bytes);
  // Both shared-memory limits, 48 KB without the opt-in and 227 KB with it, cover dynamic plus static shared memory.
  // The kernel's static size is read once and the opt-in set once per size increase (outside of any stream capture:
  // the first call is eager).
  static int s_static_smem = -1, s_attr_smem = 0;
  if (s_static_smem < 0) {
    cudaFuncAttributes fa;
    const cudaError_t e = cudaFuncGetAttributes(&fa, synth_env_step_kernel);
    if (e != cudaSuccess) { set_error("cudaFuncGetAttributes: %s", cudaGetErrorString(e)); return (int)e; }
    s_static_smem = static_cast<int>(fa.sharedSizeBytes);
  }
  TRL_REQUIRE(smem + s_static_smem <= 227 * 1024,
              "trl_synth_env_step: obs_dim %d act_dim %d need %d B of shared memory + %d B static (> 227 KB)", obs_dim,
              act_dim, smem, s_static_smem);
  if (smem + s_static_smem > 48 * 1024 && smem > s_attr_smem) {
    const cudaError_t e =
        cudaFuncSetAttribute(synth_env_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
    s_attr_smem = smem;
  }
  synth_env_step_kernel<<<trl_synth_env_num_ctas(N), kEnvThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("synth_env_step_kernel");
}

TRL_API int trl_synth_env_reset(float* state, int* elapsed, unsigned* episode, const unsigned* seeds,
                                const uint8_t* mask, int64_t N, int obs_dim, double init_scale, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && obs_dim >= 1, "trl_synth_env_reset: bad sizes");
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(state && elapsed && episode && seeds, "trl_synth_env_reset: null pointer");
  ResetParams p{state, elapsed, episode, seeds, mask, N, obs_dim, init_scale};
  const int threads = 256;
  const long long blocks = ceil_div<long long>(N * 32, threads);
  synth_env_reset_kernel<<<static_cast<unsigned>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("synth_env_reset_kernel");
}

TRL_API int trl_synth_env_seed(unsigned* seeds, unsigned* episode, int64_t N, unsigned seed, unsigned n_total,
                               unsigned first_env, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0, "trl_synth_env_seed: bad size");
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(seeds && episode, "trl_synth_env_seed: null pointer");
  synth_env_seed_kernel<<<static_cast<unsigned>(ceil_div<long long>(N, 256)), 256, 0,
                          static_cast<cudaStream_t>(stream)>>>(seeds, episode, N, seed, n_total, first_env);
  return check_launch("synth_env_seed_kernel");
}
