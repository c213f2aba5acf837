// categorical.cu -- the categorical action distribution of the discrete on-policy path: sampling, log-probabilities
// of stored actions and the fused PPO / A2C actor loss with its gradient wrt the logits.
//
// Replaces, on the device,
//   CategoricalDisPolicy.forward / explore / update   /root/reference/torchrl/policies/discrete_policies.py:123-160
//   (softmax, torch.distributions.Categorical(probs).sample / log_prob / entropy)
//   the actor half of PPO.update_actor                 /root/reference/torchrl/algo/on_policy/ppo.py:41-91
//   and of A2C.update                                  /root/reference/torchrl/algo/on_policy/a2c.py:45-112
//   VMPO.update_actor for this policy (top-half selection, loss, dual gradients)
//                                                      /root/reference/torchrl/algo/on_policy/v_mpo.py:57-133
//   TRPO's Fisher-vector product, the bias / activation step of its tangent pass and its line-search score
//                                                      /root/reference/torchrl/algo/on_policy/trpo.py:29-151
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
// The last CTA's fold of the per-CTA partials (NP quantities per CTA, the first NS sums, the rest maxima) into tot:
// warp w folds quantities w, w + 8, ...; lane l takes partials l, l+32, ... then a fixed shuffle tree.  Ends with a
// barrier, after which tot is valid in every thread.
template <int NP, int NS>
__device__ __forceinline__ void cat_fold_partials(const double* __restrict__ partial, double* tot) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int k = wid; k < NP; k += kCatThreads / 32) {
    const bool is_max = k >= NS;
    double acc = is_max ? -INFINITY : 0.0;
    for (unsigned i = lane; i < gridDim.x; i += 32) {
      const double v = __ldcg(partial + static_cast<long long>(i) * NP + k);
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
}

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
  __shared__ double tot[kCatPartials];
  cat_fold_partials<kCatPartials, 5>(p.partial, tot);
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

// ------------------------------------------------------------------------------------ V-MPO
// Top-half selection (v_mpo.py:65-67): of a minibatch's B normalised advantages keep the k = B - B/2 largest, ties to
// the lower position (torch.sort(stable=True) then chunk(2)[0]).  One CTA per minibatch: an MSB-first radix select
// over a descending-order key (4 passes of 8-bit histograms in shared memory) finds the key of the k-th largest value
// and how many of the values equal to it are kept; one ordered pass then writes the kept positions in ascending order
// with block-wide ballot scans.  Every pass reads the same values, so the counts are consistent whatever they are (NaN
// included) and the kernel always finishes.
constexpr int kSelThreads = 1024;

// minibatch position q of group u: time row perm[u*b + q / n] (row q / n if perm is null), env q % n -- the order of
// gather_rows -- normalised exactly as the loss normalises it
// (B < 2^31: 32-bit division, which compiles inline)
__device__ __forceinline__ float vmpo_advn(const float* __restrict__ advs, const long long* __restrict__ perm,
                                           long long base, unsigned n, unsigned q, float mean, float den) {
  const unsigned t = q / n;
  const long long r = perm ? perm[base + t] : static_cast<long long>(t);
  return (advs[r * n + (q - t * n)] - mean) / den;
}

// key(a) < key(b) iff a > b as floats; -0 and +0 share a key (they compare equal in torch.sort)
__device__ __forceinline__ unsigned vmpo_desc_key(float v) {
  if (v == 0.f) v = 0.f;
  const unsigned x = __float_as_uint(v);
  return (x & 0x80000000u) ? x : ~(x | 0x80000000u);
}

__global__ void __launch_bounds__(kSelThreads) vmpo_select_kernel(const float* __restrict__ advs,
                                                                  const long long* __restrict__ perm, int b,
                                                                  unsigned n, const float* __restrict__ stats,
                                                                  long long* __restrict__ sel, unsigned k) {
  __shared__ unsigned hist[256];
  __shared__ unsigned s_prefix, s_need;
  __shared__ unsigned s_cnt[2][kSelThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned B = static_cast<unsigned>(b) * n;
  const long long base = static_cast<long long>(blockIdx.x) * b;
  const float mean = stats[4LL * blockIdx.x], den = stats[4LL * blockIdx.x + 1] + 1e-5f;
  unsigned prefix = 0u, need = k;  // need: 1-based rank of the k-th key among those matching
  if (tid == 0) { s_prefix = 0u; s_need = need; }
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kSelThreads) hist[i] = 0u;
    __syncthreads();
    const unsigned hi = shift == 24 ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (unsigned q = tid; q < B; q += kSelThreads) {
      const unsigned key = vmpo_desc_key(vmpo_advn(advs, perm, base, n, q, mean, den));
      if ((key & hi) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (wid == 0) {  // lane l owns bins 8l .. 8l+7: a warp scan finds the bin holding rank `need`
      unsigned c[8], s = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[lane * 8 + j]; s += c[j]; }
      unsigned incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const unsigned ball = __ballot_sync(0xffffffffu, incl >= need);
      if (ball != 0u && lane == __ffs(ball) - 1) {
        unsigned acc = incl - s;
        int jb = 7;
#pragma unroll
        for (int j = 7; j >= 0; --j) {  // the first bin whose running count reaches `need`, in registers
          unsigned before = acc;
#pragma unroll
          for (int m = 0; m < j; ++m) before += c[m];
          if (before + c[j] >= need) jb = j;
        }
#pragma unroll
        for (int m = 0; m < 8; ++m) acc += m < jb ? c[m] : 0u;
        s_prefix = prefix | (static_cast<unsigned>(lane * 8 + jb) << shift);
        s_need = need - acc;
      }
    }
    __syncthreads();
    prefix = s_prefix;
    need = s_need;
  }
  // keep key < prefix, and the first `need` positions with key == prefix
  const unsigned lt_mask = (1u << lane) - 1u;
  unsigned eq_base = 0u, out_base = 0u;
  for (unsigned q0 = 0; q0 < B && out_base < k; q0 += kSelThreads) {
    const unsigned q = q0 + tid;
    bool lt = false, eq = false;
    if (q < B) {
      const unsigned key = vmpo_desc_key(vmpo_advn(advs, perm, base, n, q, mean, den));
      lt = key < prefix;
      eq = key == prefix;
    }
    const unsigned be = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) s_cnt[0][wid] = __popc(be);
    __syncthreads();
    unsigned eq_before = eq_base + __popc(be & lt_mask), eq_tot = 0u;
    for (int w = 0; w < kSelThreads / 32; ++w) {
      eq_before += w < wid ? s_cnt[0][w] : 0u;
      eq_tot += s_cnt[0][w];
    }
    const bool take = lt || (eq && eq_before < need);
    const unsigned bt = __ballot_sync(0xffffffffu, take);
    if (lane == 0) s_cnt[1][wid] = __popc(bt);
    __syncthreads();
    unsigned pos = out_base + __popc(bt & lt_mask), t_tot = 0u;
    for (int w = 0; w < kSelThreads / 32; ++w) {
      pos += w < wid ? s_cnt[1][w] : 0u;
      t_tot += s_cnt[1][w];
    }
    if (take && pos < k) sel[static_cast<long long>(blockIdx.x) * k + pos] = q;
    eq_base += eq_tot;
    out_base += t_tot;
    __syncthreads();  // s_cnt is rewritten by the next chunk
  }
}

// The categorical V-MPO actor loss on the k selected rows (v_mpo.py:69-99 with CategoricalDisPolicy.update,
// discrete_policies.py:156-167), value and gradient in one launch.  phi = softmax(advn / eta) needs the maximum and
// the sum of exp over all k rows before any row's gradient: every CTA computes both itself from the k advantages (the
// same block reductions in the same order, so every CTA holds the same values), which saves a second launch.
// KL_i = sum_j p_j (l_j - lq_j) as torch's _kl_categorical_categorical: a term with q_j == 0 is +inf (no gradient), a
// term with p_j == 0 is 0.  With g_j = l_j - lq_j + m_j on the live terms (0 elsewhere),
//   dKL_i / dz_k = p_k (g_k - sum_j p_j g_j),   dL/dz_i = -(phi_i / k) m_a (delta_a - p) + c dKL_i/dz_i,
// c = alpha (the reference's summed KL, reference_quirks) or alpha / k (per-row KL).
// per-CTA partials: [0] sum phi logp [1] sum logp [2] sum logp^2 [3] sum KL [4] sum KL^2 [5] sum phi advn
// [6] max logp [7] max -logp [8] max KL [9] max -KL
constexpr int kVmpoPartials = 10;

struct VmpoLossParams {
  const float* __restrict__ logits;     // (k,A)
  const float* __restrict__ tlogits;    // (k,A) target policy
  const float* __restrict__ actions;    // (k)
  const float* __restrict__ advs;       // (k) raw advantages of the selected rows
  const float* __restrict__ adv_stats;  // rows of [mean, std, max, min]
  const int* __restrict__ stats_pos;    // device scalar: row of adv_stats (nullptr: row 0)
  const float* __restrict__ dual;       // [eta, alpha]
  float* __restrict__ g_logits;         // (k,A)
  float* __restrict__ g_dual;           // (2)
  float* __restrict__ info;             // (12)
  double* __restrict__ partial;         // (grid, kVmpoPartials)
  unsigned* __restrict__ ticket;
  long long k;
  int A;
  float eta_eps, alpha_eps;
  int per_row;
};

__global__ void __launch_bounds__(kCatThreads) vmpo_categorical_loss_kernel(const VmpoLossParams p) {
  __shared__ double sh_d[kCatThreads / 32][6];
  __shared__ float sh_f[kCatThreads / 32][4];
  __shared__ double sh_sum[32];
  __shared__ float sh_max[32];
  __shared__ double s_norm[2];
  const int A = p.A;
  const float* st = p.adv_stats + (p.stats_pos ? 4LL * (*p.stats_pos) : 0LL);
  const float mean = st[0], den = st[1] + 1e-5f;
  const float eta = p.dual[0], alpha = p.dual[1];
  // phi's normaliser over all k rows: M = max advn / eta, S = sum exp(advn / eta - M)
  float mx = -INFINITY;
  for (long long i = threadIdx.x; i < p.k; i += kCatThreads) mx = fmaxf(mx, ((p.advs[i] - mean) / den) / eta);
  mx = block_reduce_max(mx, sh_max);
  if (threadIdx.x == 0) s_norm[0] = mx;
  __syncthreads();
  mx = static_cast<float>(s_norm[0]);
  double se = 0.0;
  for (long long i = threadIdx.x; i < p.k; i += kCatThreads)
    se += static_cast<double>(expf(((p.advs[i] - mean) / den) / eta - mx));
  se = block_reduce_sum(se, sh_sum);
  if (threadIdx.x == 0) s_norm[1] = se;
  __syncthreads();
  se = s_norm[1];

  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool ok = i < p.k;
  const float invk = 1.0f / static_cast<float>(p.k);
  float logp = 0.f, kl = 0.f, phi = 0.f, advn = 0.f;
  if (ok) {
    // target row first, kept as lq and a bit mask of its zero probabilities
    float pr[kCatMaxA], l[kCatMaxA], lq[kCatMaxA];
    unsigned pass, qzero = 0u;
    cat_row(p.tlogits + i * A, A, pr, lq, pass);
#pragma unroll
    for (int j = 0; j < kCatMaxA; ++j)
      if (j < A && pr[j] == 0.f) qzero |= 1u << j;
    cat_row(p.logits + i * A, A, pr, l, pass);
    const int ai = cat_action(p.actions[i], A);
    logp = cat_pick(l, A, ai);
    advn = (p.advs[i] - mean) / den;
    phi = static_cast<float>(static_cast<double>(expf(advn / eta - mx)) / se);
    bool inf_term = false;
    float spg = 0.f;
#pragma unroll
    for (int j = 0; j < kCatMaxA; ++j) {
      if (j < A) {
        const bool pz = pr[j] == 0.f, qz = (qzero >> j) & 1u;
        inf_term |= qz && !pz;
        const bool live = !pz && !qz;
        l[j] -= lq[j];  // from here l holds l - lq
        kl += live ? pr[j] * l[j] : 0.f;
        spg += live ? pr[j] * (l[j] + ((pass >> j) & 1u ? 1.f : 0.f)) : 0.f;
      }
    }
    if (inf_term) kl = INFINITY;
    const float ca = (ai >= 0 && ((pass >> ai) & 1u)) ? -phi * invk : 0.f;  // dL/dlogp_i, times m_a
    const float c = p.per_row ? alpha * invk : alpha;
#pragma unroll
    for (int j = 0; j < kCatMaxA; ++j) {
      if (j < A) {
        const bool live = pr[j] != 0.f && !((qzero >> j) & 1u);
        const float gj = live ? l[j] + ((pass >> j) & 1u ? 1.f : 0.f) : 0.f;
        p.g_logits[i * A + j] = ((j == ai ? ca : 0.f) - ca * pr[j]) + c * (pr[j] * (gj - spg));
      }
    }
  }

  const double sums[6] = {static_cast<double>(phi) * logp, static_cast<double>(logp),
                          static_cast<double>(logp) * logp, static_cast<double>(kl), static_cast<double>(kl) * kl,
                          static_cast<double>(phi) * advn};
  const float maxs[4] = {ok ? logp : -INFINITY, ok ? -logp : -INFINITY, ok ? kl : -INFINITY, ok ? -kl : -INFINITY};
  block_partials<kCatThreads / 32>(sums, maxs, sh_d, sh_f, p.partial + static_cast<long long>(blockIdx.x) * kVmpoPartials);
  if (!last_cta(p.ticket, gridDim.x)) return;
  __shared__ double tot[kVmpoPartials];
  cat_fold_partials<kVmpoPartials, 6>(p.partial, tot);
  if (threadIdx.x == 0) {
    const double kn = static_cast<double>(p.k);
    const double K = p.per_row ? tot[3] / kn : tot[3];  // what multiplies alpha
    p.info[0] = static_cast<float>(-tot[0] / kn + static_cast<double>(alpha) * K);    // policy_loss
    p.info[1] = static_cast<float>(static_cast<double>(alpha) * p.alpha_eps - static_cast<double>(alpha) * K);
    stats_from_moments(tot[1], tot[2], tot[6], -tot[7], kn, p.info + 4);               // logprob/*
    if (p.per_row) {
      stats_from_moments(tot[3], tot[4], tot[8], -tot[9], kn, p.info + 8);            // KL/*
    } else {  // the KL is one summed value: its std is torch's std of one element
      p.info[8] = p.info[10] = p.info[11] = static_cast<float>(tot[3]);
      p.info[9] = NAN;
    }
    const double lme = static_cast<double>(mx) + log(se / kn);  // log(mean(exp(advn / eta))), maximum subtracted
    p.g_dual[0] = static_cast<float>(p.eta_eps + lme - tot[5] / eta);
    p.g_dual[1] = static_cast<float>(p.alpha_eps - K);
  }
}

// ------------------------------------------------------------------------------------ TRPO
// The Fisher-vector product in logit space (trpo.py:29-86 with the KL over probs, trpo.py:53-61): at theta0 the
// Hessian of sum_a p_a log(p_a / (p_a.detach() + 1e-8)) wrt the logits z is diag(p) - p p^T up to O(1e-8) terms
// (DESIGN §6 deviation 20), so with t = J v the row's product is g = scale * (p * t - p <p, t>).  One thread per row;
// p is a max-subtracted softmax of the row's logits.
__global__ void __launch_bounds__(kCatThreads) categorical_fisher_vp_kernel(const float* __restrict__ logits,
                                                                            const float* __restrict__ tangent,
                                                                            long long M, int A, float scale,
                                                                            float* __restrict__ g) {
  const long long m = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* x = logits + m * A;
  const float* t = tangent + m * A;
  float p[kCatMaxA];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      p[j] = x[j];
      mx = fmaxf(mx, p[j]);
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
  float pt = 0.f;
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j) {
    if (j < A) {
      p[j] *= inv;
      pt += p[j] * t[j];
    }
  }
#pragma unroll
  for (int j = 0; j < kCatMaxA; ++j)
    if (j < A) g[m * A + j] = scale * (p[j] * (t[j] - pt));
}

// The bias and activation step of the tangent forward pass, in place: t <- (t + db[c]) * act'(y) over (M, C, S)
// (NCHW conv outputs with S = H * W, or (M, H) linear outputs with S = 1), with act'(y) from the cached output y:
// 1 - y*y (tanh, act 1), y > 0 (ReLU, act 2), 1 (no activation, act 0: the output layer, y unused).  Every operation
// is rounded on its own, so the result is bit for bit torch's (t + db) * (1 - y * y) / (t + db) * (y > 0).  VEC
// elements per thread (float4 loads when the caller checked alignment); the channel of the first element costs one
// division and one remainder, the others step from it.
template <int VEC, typename Idx>
__global__ void __launch_bounds__(256) tangent_bias_act_kernel(float* __restrict__ t, const float* __restrict__ db,
                                                               const float* __restrict__ y, Idx n, Idx C, Idx S,
                                                               int act) {
  const Idx stride = static_cast<Idx>(gridDim.x) * blockDim.x * VEC;
  for (Idx i = (static_cast<Idx>(blockIdx.x) * blockDim.x + threadIdx.x) * VEC; i < n; i += stride) {
    float tv[VEC], yv[VEC];
    if constexpr (VEC == 4) {
      const float4 a = *reinterpret_cast<const float4*>(t + i);
      tv[0] = a.x; tv[1] = a.y; tv[2] = a.z; tv[3] = a.w;
      if (act != 0) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(y + i));
        yv[0] = b.x; yv[1] = b.y; yv[2] = b.z; yv[3] = b.w;
      }
    } else {
      tv[0] = t[i];
      if (act != 0) yv[0] = __ldg(y + i);
    }
    const Idx q = i / S;
    Idx s = i - q * S, c = q % C;
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      float v = __fadd_rn(tv[k], __ldg(db + c));
      if (act == 1) v = __fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(yv[k], yv[k])));
      else if (act == 2) v = __fmul_rn(v, yv[k] > 0.f ? 1.0f : 0.0f);
      tv[k] = v;
      if (++s == S) {
        s = 0;
        c = c + 1 == C ? 0 : c + 1;
      }
    }
    if constexpr (VEC == 4) {
      *reinterpret_cast<float4*>(t + i) = make_float4(tv[0], tv[1], tv[2], tv[3]);
    } else {
      t[i] = tv[0];
    }
  }
}

// The line search's score of one candidate (trpo.py:113-129): -mean(exp(logp - logp_old) * advn) with logp the
// clamped log-probability of trl_categorical_log_prob.  Each row's term in fp32 as torch forms it, the sum in fp64:
// per-CTA block sums, then the last CTA folds them in a fixed order (cat_fold_partials) -- deterministic, one launch.
__global__ void __launch_bounds__(kCatThreads) categorical_surrogate_kernel(const float* __restrict__ logits,
                                                                            const float* __restrict__ actions,
                                                                            const float* __restrict__ logp_old,
                                                                            const float* __restrict__ advn,
                                                                            long long M, int A,
                                                                            float* __restrict__ out,
                                                                            double* __restrict__ partial,
                                                                            unsigned* __restrict__ ticket) {
  __shared__ double sh[32];
  const long long m = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  double term = 0.0;
  if (m < M) {
    float p[kCatMaxA], l[kCatMaxA];
    unsigned pass;
    cat_row(logits + m * A, A, p, l, pass);
    const float logp = cat_pick(l, A, cat_action(actions[m], A));
    term = static_cast<double>(__fmul_rn(expf(__fsub_rn(logp, logp_old[m])), advn[m]));
  }
  term = block_reduce_sum<false>(term, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = term;
  if (!last_cta(ticket, gridDim.x)) return;
  __shared__ double tot[1];
  cat_fold_partials<1, 1>(partial, tot);
  if (threadIdx.x == 0) out[0] = static_cast<float>(-tot[0] / static_cast<double>(M));
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

TRL_API int trl_vmpo_select(const float* advs, const int64_t* perm, int groups, int b, int64_t row_elems,
                            const float* stats4, int64_t* sel, void* stream) {
  using namespace trl;
  TRL_REQUIRE(groups >= 1 && b >= 1 && row_elems >= 1 && static_cast<long long>(b) * row_elems < (1LL << 31),
              "trl_vmpo_select: bad sizes groups=%d b=%d row_elems=%lld (B = b * row_elems >= 1, < 2^31)", groups, b,
              (long long)row_elems);
  TRL_REQUIRE(advs && stats4 && sel, "trl_vmpo_select: null pointer");
  const long long B = static_cast<long long>(b) * row_elems;
  vmpo_select_kernel<<<static_cast<unsigned>(groups), kSelThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      advs, reinterpret_cast<const long long*>(perm), b, static_cast<unsigned>(row_elems), stats4,
      reinterpret_cast<long long*>(sel), static_cast<unsigned>(B - B / 2));
  return check_launch("vmpo_select_kernel");
}

TRL_API int64_t trl_vmpo_categorical_scratch_doubles(int64_t k) {
  return trl::ceil_div<long long>(k, trl::kCatThreads) * trl::kVmpoPartials;
}

TRL_API int trl_vmpo_categorical_loss(const float* logits, const float* target_logits, const float* actions,
                                      const float* advs, const float* adv_stats, const int* adv_stats_pos,
                                      const float* dual, int64_t k, int num_actions, float eta_eps, float alpha_eps,
                                      int per_row_kl, float* g_logits, float* g_dual, float* info12, double* scratch,
                                      unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(k >= 1 && num_actions >= 1 && num_actions <= kCatMaxA,
              "trl_vmpo_categorical_loss: bad sizes k=%lld A=%d (1 <= A <= %d)", (long long)k, num_actions, kCatMaxA);
  TRL_REQUIRE(logits && target_logits && actions && advs && adv_stats && dual && g_logits && g_dual && info12 &&
                  scratch && ticket,
              "trl_vmpo_categorical_loss: null pointer");
  VmpoLossParams p{logits, target_logits, actions, advs, adv_stats, adv_stats_pos, dual, g_logits, g_dual, info12,
                   scratch, ticket, k, num_actions, eta_eps, alpha_eps, per_row_kl ? 1 : 0};
  vmpo_categorical_loss_kernel<<<static_cast<unsigned>(ceil_div<long long>(k, kCatThreads)), kCatThreads, 0,
                                 static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("vmpo_categorical_loss_kernel");
}

TRL_API int trl_categorical_fisher_vp(const float* logits, const float* tangent, int64_t M, int num_actions,
                                      float scale, float* g_logits, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && num_actions >= 1 && num_actions <= kCatMaxA,
              "trl_categorical_fisher_vp: bad sizes M=%lld A=%d (1 <= A <= %d)", (long long)M, num_actions, kCatMaxA);
  TRL_REQUIRE(logits && tangent && g_logits, "trl_categorical_fisher_vp: null pointer");
  if (M == 0) return TRL_OK;
  categorical_fisher_vp_kernel<<<static_cast<unsigned>(ceil_div<long long>(M, kCatThreads)), kCatThreads, 0,
                                 static_cast<cudaStream_t>(stream)>>>(logits, tangent, M, num_actions, scale, g_logits);
  return check_launch("categorical_fisher_vp_kernel");
}

TRL_API int trl_tangent_bias_act(float* t, const float* bias_tangent, const float* y, int64_t M, int C, int64_t S,
                                 int act, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && C >= 1 && S >= 1 && act >= 0 && act <= 2,
              "trl_tangent_bias_act: bad sizes M=%lld C=%d S=%lld act=%d (act 0 none, 1 tanh, 2 relu)", (long long)M,
              C, (long long)S, act);
  TRL_REQUIRE(t && bias_tangent && (y || act == 0), "trl_tangent_bias_act: null pointer");
  const long long n = M * C * S;
  if (n == 0) return TRL_OK;
  const bool vec = n % 4 == 0 && reinterpret_cast<uintptr_t>(t) % 16 == 0 &&
                   (act == 0 || reinterpret_cast<uintptr_t>(y) % 16 == 0);
  const int V = vec ? 4 : 1;
  const long long blocks = ceil_div<long long>(n, 256LL * V);
  const unsigned grid = static_cast<unsigned>(blocks < 132LL * 16 ? blocks : 132LL * 16);  // grid-stride beyond
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n < (1LL << 31)) {
    const unsigned nn = static_cast<unsigned>(n), cc = static_cast<unsigned>(C), ss = static_cast<unsigned>(S);
    if (vec) tangent_bias_act_kernel<4, unsigned><<<grid, 256, 0, st>>>(t, bias_tangent, y, nn, cc, ss, act);
    else tangent_bias_act_kernel<1, unsigned><<<grid, 256, 0, st>>>(t, bias_tangent, y, nn, cc, ss, act);
  } else {
    const unsigned long long nn = n, cc = C, ss = S;
    if (vec) tangent_bias_act_kernel<4, unsigned long long><<<grid, 256, 0, st>>>(t, bias_tangent, y, nn, cc, ss, act);
    else tangent_bias_act_kernel<1, unsigned long long><<<grid, 256, 0, st>>>(t, bias_tangent, y, nn, cc, ss, act);
  }
  return check_launch("tangent_bias_act_kernel");
}

TRL_API int trl_categorical_surrogate(const float* logits, const float* actions, const float* logp_old,
                                      const float* advn, int64_t M, int num_actions, float* out, double* scratch,
                                      unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && num_actions >= 1 && num_actions <= kCatMaxA,
              "trl_categorical_surrogate: bad sizes M=%lld A=%d (1 <= A <= %d)", (long long)M, num_actions, kCatMaxA);
  TRL_REQUIRE(logits && actions && logp_old && advn && out && scratch && ticket,
              "trl_categorical_surrogate: null pointer");
  categorical_surrogate_kernel<<<static_cast<unsigned>(ceil_div<long long>(M, kCatThreads)), kCatThreads, 0,
                                 static_cast<cudaStream_t>(stream)>>>(logits, actions, logp_old, advn, M, num_actions,
                                                                     out, scratch, ticket);
  return check_launch("categorical_surrogate_kernel");
}
