// categorical.cu -- the categorical action distribution of the discrete on-policy path: sampling, log-probabilities
// of stored actions and the fused PPO / A2C actor loss with its gradient wrt the logits.
//
// Replaces, on the device,
//   CategoricalDisPolicy.forward / explore / update   /root/reference/torchrl/policies/discrete_policies.py:123-160
//   (softmax, torch.distributions.Categorical(probs).sample / log_prob / entropy)
//   the actor half of PPO.update_actor                 /root/reference/torchrl/algo/on_policy/ppo.py:41-91
//   and of A2C.update                                  /root/reference/torchrl/algo/on_policy/a2c.py:45-112
// The distribution is torch's Categorical(probs=softmax(x)): p = softmax(x) (maximum subtracted, then renormalised as
// Categorical does), l_j = log(clamp(p_j, eps, 1-eps)) (probs_to_logits, NOT log_softmax), log_prob(a) = l_a,
// entropy = -sum_j p_j l_j.  Gradients wrt x, with m_j = 1 where the clamp passes (eps <= p_j <= 1-eps):
//   d l_a / d x_k = m_a (delta_ak - p_k)
//   d ent / d x_k = -p_k (l_k + m_k) + p_k sum_j p_j (l_j + m_j)
// One thread per row; a row's (<= 32) logits live in registers.  The actor loss's reductions are two-level and
// deterministic (reduce.cuh: block_partials per CTA, then last_cta; the last CTA folds in a fixed order).
#include "reduce.cuh"

namespace trl {

constexpr int kCatMaxA = 32;
constexpr int kCatThreads = 256;
constexpr float kCatEps = 1.1920928955078125e-07f;  // torch.finfo(torch.float32).eps = 2^-23
// per-CTA partials of the actor loss: [0] sum L_b [1] sum logp [2] sum logp^2 [3] sum ent [4] sum (old - new logp)
// [5] max logp [6] max -logp [7] max ratio [8] max -ratio
constexpr int kCatPartials = 9;

// p, l and the clamp mask of one row; returns false if any logit is not finite
__device__ __forceinline__ bool cat_row(const float* __restrict__ x, int A, float (&p)[kCatMaxA], float (&l)[kCatMaxA],
                                        unsigned& pass) {
  float mx = -INFINITY;
  bool finite = true;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      const float v = x[j];
      finite &= isfinite(v);
      p[j] = v;
      mx = fmaxf(mx, v);
    }
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      p[j] = expf(p[j] - mx);
      s += p[j];
    }
  }
  const float inv = 1.0f / s;
  float s2 = 0.f;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      p[j] *= inv;
      s2 += p[j];
    }
  }
  const float inv2 = 1.0f / s2;  // Categorical(probs) renormalises the softmax output once more
  pass = 0u;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      p[j] *= inv2;
      const bool ok = p[j] >= kCatEps && p[j] <= 1.0f - kCatEps;
      l[j] = logf(fminf(fmaxf(p[j], kCatEps), 1.0f - kCatEps));
      pass |= ok ? (1u << j) : 0u;
    }
  }
  return finite;
}

// the action index stored as float; -1 if it is not an integer in [0, A)
__device__ __forceinline__ int cat_action(float a, int A) {
  const int i = static_cast<int>(a);
  return (a == static_cast<float>(i) && i >= 0 && i < A) ? i : -1;
}

__device__ __forceinline__ float cat_pick(const float (&l)[kCatMaxA], int A, int i) {
  float r = NAN;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j)
    if (j < A && j == i) r = l[j];
  return r;
}

// ------------------------------------------------------------------------------------ sampling
__global__ void __launch_bounds__(128) categorical_sample_kernel(const float* __restrict__ logits,
                                                                 const float* __restrict__ u,
                                                                 unsigned long long seed,
                                                                 const unsigned long long* __restrict__ rng_counter,
                                                                 long long M, int A, float* __restrict__ action,
                                                                 float* __restrict__ log_prob,
                                                                 int* __restrict__ nan_flag) {
  const long long m = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float p[kCatMaxA], l[kCatMaxA];
  unsigned pass;
  const bool finite = cat_row(logits + m * A, A, p, l, pass);
  float uu;
  if (u) {
    uu = u[m];
  } else {
    uint32_t r[4];
    const unsigned long long ctr = rng_counter ? *rng_counter : 0ull;
    Philox::gen(seed, ctr * 0x100000000ull + static_cast<unsigned long long>(m), 0u, r);
    uu = static_cast<float>(r[0] >> 8) * (1.0f / 16777216.0f);  // [0, 1)
  }
  // inverse CDF: the first j with u < p_0 + ... + p_j; rounding can leave the total just below u, then the last
  // action of non-zero probability is taken
  int pick = -1, last = 0;
  float c = 0.f;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      c += p[j];
      if (pick < 0 && uu < c) pick = j;
      if (p[j] > 0.f) last = j;
    }
  }
  if (pick < 0) pick = last;
  if (!finite) {
    pick = 0;
    if (nan_flag) atomicOr(nan_flag, 1);
  }
  action[m] = static_cast<float>(pick);
  if (log_prob) log_prob[m] = finite ? cat_pick(l, A, pick) : NAN;
}

__global__ void categorical_logprob_kernel(const float* __restrict__ logits, const float* __restrict__ actions,
                                           long long M, int A, float* __restrict__ logp) {
  const long long m = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float p[kCatMaxA], l[kCatMaxA];
  unsigned pass;
  cat_row(logits + m * A, A, p, l, pass);
  logp[m] = cat_pick(l, A, cat_action(actions[m], A));
}

// ------------------------------------------------------------------------------------ actor loss
struct CatLossParams {
  const float* __restrict__ logits;     // (B,A)
  const float* __restrict__ actions;    // (B) index as float
  const float* __restrict__ old_logp;   // (B) or nullptr (A2C: plain policy gradient)
  const float* __restrict__ advs;       // (B) raw advantages
  const float* __restrict__ adv_stats;  // rows of [mean, std, max, min] or nullptr (no normalisation)
  const int* __restrict__ stats_pos;    // device scalar: row of adv_stats (nullptr: row 0)
  float* __restrict__ g_logits;         // (B,A)
  float* __restrict__ logp_out;         // (B) or nullptr
  float* __restrict__ info;             // (16)
  double* __restrict__ partial;         // (grid, kCatPartials)
  unsigned* __restrict__ ticket;
  long long B;
  int A;
  float clip, ent_coef;
};

__global__ void __launch_bounds__(kCatThreads) ppo_categorical_actor_loss_kernel(const CatLossParams p) {
  __shared__ double sh_d[kCatThreads / 32][5];
  __shared__ float sh_f[kCatThreads / 32][4];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool ok = b < p.B;
  const int A = p.A;
  const float invB = 1.0f / static_cast<float>(p.B);
  float Lb = 0.f, logp = 0.f, ratio = 1.f, dkl = 0.f, ent = 0.f;
  if (ok) {
    float pr[kCatMaxA], l[kCatMaxA];
    unsigned pass;
    cat_row(p.logits + b * A, A, pr, l, pass);
    const int ai = cat_action(p.actions[b], A);
    logp = cat_pick(l, A, ai);
    float sm = 0.f;
#pragma unroll
    for (int j = 0; j < kCatMaxA; ++j) {
      if (j < A) {
        ent -= pr[j] * l[j];
        sm += pr[j] * (l[j] + ((pass >> j) & 1u ? 1.f : 0.f));
      }
    }
    float adv = p.advs[b];
    if (p.adv_stats) {
      const float* st = p.adv_stats + (p.stats_pos ? 4LL * (*p.stats_pos) : 0LL);
      adv = (adv - st[0]) / (st[1] + 1e-5f);
    }
    float coef;  // dL/dlogp_b
    if (p.old_logp) {
      // clipped surrogate and torch's tie rule, as in ppo_actor_loss_kernel
      const float oldlp = p.old_logp[b];
      ratio = expf(logp - oldlp);
      dkl = oldlp - logp;
      const float lo = 1.0f - p.clip, hi = 1.0f + p.clip;
      const float s1 = ratio * adv;
      const float s2 = fminf(fmaxf(ratio, lo), hi) * adv;
      Lb = -fminf(s2, s1);
      const bool in_range = (ratio >= lo) && (ratio <= hi);
      float dLdr;
      if (s1 < s2) dLdr = -adv;
      else if (s2 < s1) dLdr = in_range ? -adv : 0.f;
      else dLdr = -0.5f * adv - (in_range ? 0.5f * adv : 0.f);
      coef = dLdr * ratio * invB;
    } else {
      Lb = -logp * adv;
      coef = -adv * invB;
    }
    const float ca = (ai >= 0 && ((pass >> ai) & 1u)) ? coef : 0.f;  // m_a
    const float ce = p.ent_coef * invB;
#pragma unroll
    for (int j = 0; j < kCatMaxA; ++j) {
      if (j < A) {
        const float mj = (pass >> j) & 1u ? 1.f : 0.f;
        const float dlp = (j == ai ? ca : 0.f) - ca * pr[j];
        const float dent = pr[j] * (sm - l[j] - mj);
        p.g_logits[b * A + j] = dlp - ce * dent;
      }
    }
    if (p.logp_out) p.logp_out[b] = logp;
  }

  // per-CTA partials with one barrier (warp shuffles, a per-warp table in shared memory, then one thread per quantity)
  const double sums[5] = {static_cast<double>(Lb), ok ? static_cast<double>(logp) : 0.0,
                          ok ? static_cast<double>(logp) * logp : 0.0, static_cast<double>(ent),
                          static_cast<double>(dkl)};
  const float maxs[4] = {ok ? logp : -INFINITY, ok ? -logp : -INFINITY, ok ? ratio : -INFINITY,
                         ok ? -ratio : -INFINITY};
  block_partials<kCatThreads / 32>(sums, maxs, sh_d, sh_f, p.partial + static_cast<long long>(blockIdx.x) * kCatPartials);
  if (!last_cta(p.ticket, gridDim.x)) return;
  // last CTA: warp w folds quantities w and w + 8; lane l takes partials l, l+32, ... then a fixed shuffle tree
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __shared__ double tot[kCatPartials];
  for (int k = wid; k < kCatPartials; k += kCatThreads / 32) {
    const bool is_max = k >= 5;
    double acc = is_max ? -INFINITY : 0.0;
    for (unsigned i = lane; i < gridDim.x; i += 32) {
      const double v = __ldcg(p.partial + static_cast<long long>(i) * kCatPartials + k);
      acc = is_max ? fmax(acc, v) : acc + v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double w = __shfl_xor_sync(0xffffffffu, acc, o);
      acc = is_max ? fmax(acc, w) : acc + w;
    }
    if (lane == 0) tot[k] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double Bn = static_cast<double>(p.B);
    const double ent_mean = tot[3] / Bn;
    const double lp_mean = tot[1] / Bn;
    const double lp_var = (tot[2] - tot[1] * lp_mean) / (Bn - 1.0);
    p.info[0] = static_cast<float>(tot[0] / Bn - p.ent_coef * ent_mean);  // policy_loss
    p.info[1] = static_cast<float>(lp_mean);
    p.info[2] = static_cast<float>(sqrt(lp_var > 0.0 ? lp_var : 0.0));
    p.info[3] = static_cast<float>(tot[5]);
    p.info[4] = static_cast<float>(-tot[6]);
    p.info[5] = static_cast<float>(tot[7]);
    p.info[6] = static_cast<float>(-tot[8]);
    for (int k = 7; k < 11; ++k) p.info[k] = 0.f;  // the log-std slots of the Gaussian kernel
    p.info[11] = static_cast<float>(ent_mean);
    p.info[12] = static_cast<float>(tot[4] / Bn);
  }
}

}  // namespace trl

TRL_API int trl_categorical_sample(const float* logits, const float* u, uint64_t seed, const uint64_t* rng_counter,
                                   int64_t M, int num_actions, float* action, float* log_prob, int* nan_flag,
                                   void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && num_actions >= 1 && num_actions <= kCatMaxA,
              "trl_categorical_sample: bad sizes M=%lld A=%d (1 <= A <= %d)", (long long)M, num_actions, kCatMaxA);
  TRL_REQUIRE(logits && action, "trl_categorical_sample: null pointer");
  TRL_REQUIRE(u || rng_counter, "trl_categorical_sample: null pointer: needs u or rng_counter");
  if (M == 0) return TRL_OK;
  categorical_sample_kernel<<<static_cast<unsigned>(ceil_div<long long>(M, 128)), 128, 0,
                              static_cast<cudaStream_t>(stream)>>>(
      logits, u, seed, reinterpret_cast<const unsigned long long*>(rng_counter), M, num_actions, action, log_prob,
      nan_flag);
  return check_launch("categorical_sample_kernel");
}

TRL_API int trl_categorical_log_prob(const float* logits, const float* actions, int64_t M, int num_actions,
                                     float* logp, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && num_actions >= 1 && num_actions <= kCatMaxA,
              "trl_categorical_log_prob: bad sizes M=%lld A=%d (1 <= A <= %d)", (long long)M, num_actions, kCatMaxA);
  TRL_REQUIRE(logits && actions && logp, "trl_categorical_log_prob: null pointer");
  if (M == 0) return TRL_OK;
  categorical_logprob_kernel<<<static_cast<unsigned>(ceil_div<long long>(M, 256)), 256, 0,
                               static_cast<cudaStream_t>(stream)>>>(logits, actions, M, num_actions, logp);
  return check_launch("categorical_logprob_kernel");
}

TRL_API int64_t trl_ppo_categorical_actor_scratch_doubles(int64_t B) {
  return trl::ceil_div<long long>(B, trl::kCatThreads) * trl::kCatPartials;
}

TRL_API int trl_ppo_categorical_actor_loss(const float* logits, const float* actions, const float* old_logp,
                                           const float* advs, const float* adv_stats, const int* adv_stats_pos,
                                           int64_t B, int num_actions, float clip_para, float entropy_coeff,
                                           float* g_logits, float* logp_out, float* info16, double* scratch,
                                           unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1 && num_actions >= 1 && num_actions <= kCatMaxA,
              "trl_ppo_categorical_actor_loss: bad sizes B=%lld A=%d (1 <= A <= %d)", (long long)B, num_actions,
              kCatMaxA);
  TRL_REQUIRE(logits && actions && advs && g_logits && info16 && scratch && ticket,
              "trl_ppo_categorical_actor_loss: null pointer");
  CatLossParams p{logits, actions, old_logp, advs, adv_stats, adv_stats_pos, g_logits, logp_out, info16, scratch,
                  ticket, B, num_actions, clip_para, entropy_coeff};
  ppo_categorical_actor_loss_kernel<<<static_cast<unsigned>(ceil_div<long long>(B, kCatThreads)), kCatThreads, 0,
                                      static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("ppo_categorical_actor_loss_kernel");
}
