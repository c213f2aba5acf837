// ppo_loss.cu -- K8: fused PPO actor / critic loss, forward value AND gradient wrt the net outputs.
//
// Replaces the op-by-op torch graph (and its .item() syncs) of
//   PPO.update_actor   /root/reference/torchrl/algo/on_policy/ppo.py:41-91
//   PPO.update_critic  /root/reference/torchrl/algo/on_policy/ppo.py:93-122
//   advantage normalisation                              ppo.py:147
//   GuassianContPolicyBase.update   /root/reference/torchrl/policies/continuous_policy.py:134-153
//   TanhNormal.log_prob (atanh recomputed from the action)  /root/reference/torchrl/policies/distribution.py:33-45
// One launch produces the scalar loss, dL/d(mean), dL/d(log_std) and the logged statistics;
// the caller seeds torch.autograd.backward at the MLP outputs with these gradients, so no
// intermediate (B,a) tensors ever round-trip through HBM and nothing syncs with the host.
// Reductions are two-level and deterministic (reduce.cuh: per-CTA partials, then last_cta; each kernel's last CTA folds
// the partials in its own fixed order).
#include "reduce.cuh"

namespace trl {

constexpr float kHalfLog2Pi = 0.9189385332046727f;
constexpr int kLossThreads = 256;
constexpr int kMaxAct = 32;

// ---- partial layout of the actor kernel -------------------------------------------------
// [0] sum L_b  [1] sum logp  [2] sum logp^2  [3] max logp  [4] min logp  [5] max ratio  [6] min ratio
// [7] sum ls   [8] sum ls^2  [9] max ls      [10] min ls   [11] sum (old-new logp) (approx KL)
// [12 .. 12+a) sum_b dL/dls_j (shared log_std only)
constexpr int kActorFixed = 12;

struct ActorParams {
  const float* __restrict__ mean;       // (B,a)
  const float* __restrict__ log_std;    // (a) or (B,a)
  const float* __restrict__ actions;    // (B,a)
  const float* __restrict__ old_logp;   // (B)
  const float* __restrict__ advs;       // (B) raw advantages
  const float* __restrict__ adv_stats;  // [mean, std, ..] rows of 4 floats, or nullptr (no normalisation)
  const int* __restrict__ stats_pos;    // device scalar: which row of adv_stats (nullptr: row 0)
  float* __restrict__ g_mean;           // (B,a)
  float* __restrict__ g_log_std;        // (a) or (B,a)
  float* __restrict__ logp_out;         // (B) or nullptr
  float* __restrict__ info;             // (16) outputs, see trl_ppo_actor_loss
  double* __restrict__ partial;         // (grid, 12+a)
  unsigned* __restrict__ ticket;
  long long B;
  int a, ls_stride, tanh_action;
  float clip, ent_coef;
  float ls_min, ls_max;                 // log_std is clamped to [ls_min, ls_max] first (ls_min > ls_max: no clamp)
};

// torch.clamp(log_std, lo, hi) folded into the loss (GuassianContPolicyBasicBias.forward,
// /root/reference/torchrl/policies/continuous_policy.py:173-188): value, and whether the gradient passes
// (clamp's backward lets it through for lo <= x <= hi)
__device__ __forceinline__ float clamped_ls(const ActorParams& p, float raw, bool* pass) {
  if (p.ls_min > p.ls_max) { *pass = true; return raw; }
  *pass = (raw >= p.ls_min) && (raw <= p.ls_max);
  return fminf(fmaxf(raw, p.ls_min), p.ls_max);
}

__global__ void __launch_bounds__(kLossThreads) ppo_actor_loss_kernel(const ActorParams p) {
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool ok = b < p.B;
  const int a = p.a;
  const float invB = 1.0f / static_cast<float>(p.B);
  float Lb = 0.f, logp = 0.f, ratio = 1.f, dkl = 0.f, coef = 0.f;
  float ls_s = 0.f, ls_q = 0.f, ls_mx = -INFINITY, ls_mn = INFINITY;

  if (ok) {
    for (int j = 0; j < a; ++j) {
      const float act = p.actions[b * a + j];
      const float mu = p.mean[b * a + j];
      bool pass;
      const float ls = clamped_ls(p, p.log_std[(p.ls_stride ? b * p.ls_stride : 0) + j], &pass);
      const float sd = expf(ls);
      // pre-tanh value recovered exactly as the reference does: log((1+a)/(1-a))/2
      const float z = p.tanh_action ? 0.5f * logf((1.0f + act) / (1.0f - act)) : act;
      const float d = (z - mu) / sd;
      float l = -0.5f * d * d - ls - kHalfLog2Pi;
      if (p.tanh_action) l -= logf(1.0f - act * act + 1e-6f);
      logp += l;
      if (p.ls_stride) { ls_s += ls; ls_q += ls * ls; ls_mx = fmaxf(ls_mx, ls); ls_mn = fminf(ls_mn, ls); }
    }
    float adv = p.advs[b];
    if (p.adv_stats) {
      const float* st = p.adv_stats + (p.stats_pos ? 4LL * (*p.stats_pos) : 0LL);
      adv = (adv - st[0]) / (st[1] + 1e-5f);
    }
    if (p.old_logp) {
      const float oldlp = p.old_logp[b];
      ratio = expf(logp - oldlp);
      dkl = oldlp - logp;
      const float lo = 1.0f - p.clip, hi = 1.0f + p.clip;
      const float s1 = ratio * adv;
      const float s2 = fminf(fmaxf(ratio, lo), hi) * adv;
      Lb = -fminf(s2, s1);
      // d(-min(s2,s1))/d ratio with torch's tie rule (equal -> split evenly)
      const bool in_range = (ratio >= lo) && (ratio <= hi);
      float dLdr;
      if (s1 < s2) dLdr = -adv;
      else if (s2 < s1) dLdr = in_range ? -adv : 0.f;
      else dLdr = -0.5f * adv - (in_range ? 0.5f * adv : 0.f);
      coef = dLdr * ratio * invB;  // dL/dlogp
    } else {
      // plain policy gradient (A2C, /root/reference/torchrl/algo/on_policy/a2c.py:66-70): L_b = -logp_b * adv_b
      Lb = -logp * adv;
      coef = -adv * invB;
    }
    if (p.logp_out) p.logp_out[b] = logp;
  }

  double* pp = p.partial + static_cast<long long>(blockIdx.x) * (kActorFixed + a);
  // One block-wide reduction for everything: warp shuffles, per-warp results in shared memory, ONE barrier,
  // then thread k folds the warps' values of quantity k (previously 18 separate two-barrier reductions).
  __shared__ double sh_sum[kLossThreads / 32][6 + kMaxAct];
  __shared__ float sh_max[kLossThreads / 32][6];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  constexpr int NW = kLossThreads / 32;
  // ---- gradients: second pass over the action dims (values re-read from L1) -------------
  for (int j = 0; j < a; ++j) {
    float gl = 0.f;
    if (ok) {
      const float act = p.actions[b * a + j];
      const float mu = p.mean[b * a + j];
      bool pass;
      const float ls = clamped_ls(p, p.log_std[(p.ls_stride ? b * p.ls_stride : 0) + j], &pass);
      const float sd = expf(ls);
      const float z = p.tanh_action ? 0.5f * logf((1.0f + act) / (1.0f - act)) : act;
      const float d = (z - mu) / sd;
      p.g_mean[b * a + j] = coef * (d / sd);          // dlogp/dmu = (z-mu)/sd^2
      gl = coef * (d * d - 1.0f);                     // dlogp/dls = (z-mu)^2/sd^2 - 1
      if (p.ls_stride) p.g_log_std[b * a + j] = pass ? gl - p.ent_coef * invB : 0.f;  // entropy: d ent_b/d ls = 1
    }
    if (!p.ls_stride) {
      const double w = warp_sum(static_cast<double>(gl));
      if (lane == 0) sh_sum[wid][6 + j] = w;
    }
  }
  {
    const double sums[6] = {static_cast<double>(Lb), ok ? static_cast<double>(logp) : 0.0,
                            ok ? static_cast<double>(logp) * logp : 0.0, static_cast<double>(ls_s),
                            static_cast<double>(ls_q), static_cast<double>(dkl)};
    const float maxs[6] = {ok ? logp : -INFINITY, ok ? -logp : -INFINITY, ok ? ratio : -INFINITY,
                           ok ? -ratio : -INFINITY, ls_mx, -ls_mn};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const double w = warp_sum(sums[k]);
      const float m = warp_max(maxs[k]);
      if (lane == 0) { sh_sum[wid][k] = w; sh_max[wid][k] = m; }
    }
  }
  __syncthreads();
  {
    const int k = threadIdx.x;
    const int nsum = 6 + (p.ls_stride ? 0 : a);
    if (k < nsum) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < NW; ++w) t += sh_sum[w][k];
      // partial slots: 0 L, 1 logp, 2 logp^2, 7 ls, 8 ls^2, 11 dkl, 12+j dL/dls_j
      const int slot = k == 0 ? 0 : k == 1 ? 1 : k == 2 ? 2 : k == 3 ? 7 : k == 4 ? 8 : k == 5 ? 11 : kActorFixed + (k - 6);
      pp[slot] = t;
    } else if (k >= 6 + kMaxAct && k < 12 + kMaxAct) {
      // threads of their own, past the largest nsum: with a shared log-std and a >= 27 the sum slots reach thread 32
      const int q = k - (6 + kMaxAct);
      float m = -INFINITY;
#pragma unroll
      for (int w = 0; w < NW; ++w) m = fmaxf(m, sh_max[w][q]);
      // 3 max logp, 4 min logp, 5 max ratio, 6 min ratio, 9 max ls, 10 min ls
      const int slot = q == 0 ? 3 : q == 1 ? 4 : q == 2 ? 5 : q == 3 ? 6 : q == 4 ? 9 : 10;
      pp[slot] = (q & 1) ? -static_cast<double>(m) : static_cast<double>(m);
    }
  }
  if (!last_cta(p.ticket, gridDim.x)) return;
  // ---- last CTA: fixed-order reduction of the partials ----------------------------------
  const int K = kActorFixed + a;   // <= 44
  const int nb = gridDim.x;
  // 4 chunks x 64 quantity slots: thread (chunk, k) folds partials i = chunk, chunk+4, ... ; fixed order
  __shared__ double sh_fin[4][64];
  {
    const int k = threadIdx.x & 63, chunk = threadIdx.x >> 6;
    const bool is_max = (k == 3 || k == 5 || k == 9), is_min = (k == 4 || k == 6 || k == 10);
    double acc = is_max ? -INFINITY : (is_min ? INFINITY : 0.0);
    if (k < K) {
      // eight partials are requested before the first is folded (same fold order as a plain loop; a dependent
      // load per partial made this tail ~nb/4 L2 round trips long)
      const double ident = acc;
      for (int i = chunk; i < nb; i += 32) {
        double v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          v[u] = (i + 4 * u < nb) ? __ldcg(p.partial + static_cast<long long>(i + 4 * u) * K + k) : ident;
#pragma unroll
        for (int u = 0; u < 8; ++u) acc = is_max ? fmax(acc, v[u]) : (is_min ? fmin(acc, v[u]) : acc + v[u]);
      }
    }
    sh_fin[chunk][k] = acc;
    __syncthreads();
    if (chunk == 0 && k < K) {
      for (int c = 1; c < 4; ++c) {
        const double v = sh_fin[c][k];
        acc = is_max ? fmax(acc, v) : (is_min ? fmin(acc, v) : acc + v);
      }
      p.partial[k] = acc;  // slot 0 now holds the totals (all other CTAs are done)
    }
  }
  __syncthreads();
  // the scalar outputs are independent of one another: a few threads compute them side by side (one thread doing all the
  // fp64 divisions and square roots in sequence was ~2 us of this kernel's serial tail)
  const double Bn = static_cast<double>(p.B);
  const double* t = p.partial;
  if (threadIdx.x == 0) {
    // entropy of the Normal: sum_j (0.5 + 0.5 log 2pi + ls_j), averaged over the batch
    double ent_mean, ls_mean, ls_std, ls_max, ls_min;
    if (p.ls_stride) {
      const double cnt = Bn * a;
      ls_mean = t[7] / cnt;
      double var = (t[8] - t[7] * ls_mean) / (cnt - 1.0);
      ls_std = sqrt(var > 0.0 ? var : 0.0);
      ls_max = t[9]; ls_min = t[10];
      ent_mean = a * (0.5 + static_cast<double>(kHalfLog2Pi)) + t[7] / Bn;
    } else {
      double s = 0.0, q = 0.0; ls_max = -INFINITY; ls_min = INFINITY;
      for (int j = 0; j < a; ++j) {
        bool pass;
        const double ls = clamped_ls(p, p.log_std[j], &pass);
        s += ls; q += ls * ls; ls_max = fmax(ls_max, ls); ls_min = fmin(ls_min, ls);
      }
      ls_mean = s / a;
      double var = a > 1 ? (q - s * ls_mean) / (a - 1.0) : NAN;
      ls_std = a > 1 ? sqrt(var > 0.0 ? var : 0.0) : NAN;
      ent_mean = a * (0.5 + static_cast<double>(kHalfLog2Pi)) + s;
    }
    p.info[0] = static_cast<float>(t[0] / Bn - p.ent_coef * ent_mean);  // policy_loss
    p.info[7] = static_cast<float>(ls_mean);
    p.info[8] = static_cast<float>(ls_std);
    p.info[9] = static_cast<float>(ls_max);
    p.info[10] = static_cast<float>(ls_min);
    p.info[11] = static_cast<float>(ent_mean);
  } else if (threadIdx.x == 32) {
    const double lp_mean = t[1] / Bn;
    const double lp_var = (t[2] - t[1] * lp_mean) / (Bn - 1.0);
    p.info[1] = static_cast<float>(lp_mean);
    p.info[2] = static_cast<float>(sqrt(lp_var > 0.0 ? lp_var : 0.0));
  } else if (threadIdx.x == 64) {
    p.info[3] = static_cast<float>(t[3]);
    p.info[4] = static_cast<float>(t[4]);
    p.info[5] = static_cast<float>(t[5]);
    p.info[6] = static_cast<float>(t[6]);
    p.info[12] = static_cast<float>(t[11] / Bn);
  } else if (threadIdx.x >= 96 && threadIdx.x < 96 + a && !p.ls_stride) {
    const int j = threadIdx.x - 96;
    bool pass;
    clamped_ls(p, p.log_std[j], &pass);
    p.g_log_std[j] = pass ? static_cast<float>(t[kActorFixed + j]) - p.ent_coef : 0.f;
  }
}

// ------------------------------------------------------------------------------------ critic
struct CriticParams {
  const float* __restrict__ values;      // (B) V(obs) from the value net
  const float* __restrict__ returns;     // (B) estimate_returns
  const float* __restrict__ old_values;  // (B) or nullptr
  float* __restrict__ g_values;          // (B) dL/dV
  float* __restrict__ info;              // [0] vf_loss
  double* __restrict__ partial;          // (grid)
  unsigned* __restrict__ ticket;
  long long B;
  float clip;
  int clipped;
};

__global__ void __launch_bounds__(kLossThreads) ppo_critic_loss_kernel(const CriticParams p) {
  __shared__ double shd[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const float invB = 1.0f / static_cast<float>(p.B);
  float L = 0.f;
  if (b < p.B) {
    const float v = p.values[b], ret = p.returns[b];
    const float d1 = v - ret;
    if (p.clipped) {
      // 0.5*mean(max((V-R)^2, (Vold + clamp(V-Vold,+-c) - R)^2))   ppo.py:100-107
      const float vo = p.old_values[b];
      const float dv = v - vo;
      const float dvc = fminf(fmaxf(dv, -p.clip), p.clip);
      const float d2 = vo + dvc - ret;
      const float l1 = d1 * d1, l2 = d2 * d2;
      L = 0.5f * fmaxf(l1, l2);
      const float g1 = d1;                                              // d(0.5*l1)/dV
      const float g2 = (dv >= -p.clip && dv <= p.clip) ? d2 : 0.f;      // d(0.5*l2)/dV
      float g = l1 > l2 ? g1 : (l2 > l1 ? g2 : 0.5f * (g1 + g2));
      p.g_values[b] = g * invB;
    } else {
      L = d1 * d1;                                                      // nn.MSELoss
      p.g_values[b] = 2.0f * d1 * invB;
    }
  }
  double r = block_reduce_sum(static_cast<double>(L), shd);
  if (threadIdx.x == 0) p.partial[blockIdx.x] = r;
  if (!last_cta(p.ticket, gridDim.x)) return;
  if (threadIdx.x < 32) {
    // lane l folds partials l, l+32, ... (independent loads), then a fixed shuffle tree: deterministic
    double acc = 0.0;
    for (unsigned i = threadIdx.x; i < gridDim.x; i += 32) acc += __ldcg(p.partial + i);
    acc = warp_sum(acc);
    if (threadIdx.x == 0) p.info[0] = static_cast<float>(acc / static_cast<double>(p.B));
  }
}

}  // namespace trl

TRL_API int64_t trl_ppo_actor_scratch_doubles(int64_t B, int act_dim) {
  return trl::ceil_div<long long>(B, trl::kLossThreads) * (trl::kActorFixed + act_dim);
}

TRL_API int trl_ppo_actor_loss(const float* mean, const float* log_std, int ls_stride, const float* actions,
                               const float* old_logp, const float* advs, const float* adv_stats,
                               const int* adv_stats_pos, int64_t B,
                               int act_dim, int tanh_action, float clip_para, float entropy_coeff, float ls_min,
                               float ls_max, float* g_mean,
                               float* g_log_std, float* logp_out, float* info16, double* scratch, unsigned* ticket,
                               void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1 && act_dim >= 1 && act_dim <= kMaxAct, "trl_ppo_actor_loss: bad sizes B=%lld a=%d (a<=%d)",
              (long long)B, act_dim, kMaxAct);
  TRL_REQUIRE(ls_stride == 0 || ls_stride == act_dim, "trl_ppo_actor_loss: ls_stride must be 0 or act_dim");
  TRL_REQUIRE(mean && log_std && actions && advs && g_mean && g_log_std && info16 && scratch && ticket,
              "trl_ppo_actor_loss: null pointer");
  ActorParams p{mean, log_std, actions, old_logp, advs, adv_stats, adv_stats_pos, g_mean, g_log_std, logp_out, info16, scratch,
                ticket, B, act_dim, ls_stride, tanh_action, clip_para, entropy_coeff, ls_min, ls_max};
  ppo_actor_loss_kernel<<<static_cast<unsigned>(ceil_div<long long>(B, kLossThreads)), kLossThreads, 0,
                          static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("ppo_actor_loss_kernel");
}

TRL_API int trl_ppo_critic_loss(const float* values, const float* returns, const float* old_values, int64_t B,
                                int clipped, float clip_para, float* g_values, float* info1, double* scratch,
                                unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_ppo_critic_loss: empty batch");
  TRL_REQUIRE(values && returns && g_values && info1 && scratch && ticket, "trl_ppo_critic_loss: null pointer");
  TRL_REQUIRE(!clipped || old_values, "trl_ppo_critic_loss: clipped loss needs old_values");
  CriticParams p{values, returns, old_values, g_values, info1, scratch, ticket, B, clip_para, clipped};
  ppo_critic_loss_kernel<<<static_cast<unsigned>(ceil_div<long long>(B, kLossThreads)), kLossThreads, 0,
                           static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("ppo_critic_loss_kernel");
}

// log pi(a|s) of STORED actions (the "old" log-probs, cached once per epoch): forward only.
namespace trl {
__global__ void gaussian_logprob_kernel(const float* __restrict__ mean, const float* __restrict__ log_std,
                                        int ls_stride, const float* __restrict__ actions, long long B, int a,
                                        int tanh_action, float* __restrict__ logp) {
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float lp = 0.f;
  for (int j = 0; j < a; ++j) {
    const float act = actions[b * a + j], mu = mean[b * a + j];
    const float ls = log_std[(ls_stride ? b * ls_stride : 0) + j];
    const float sd = expf(ls);
    const float z = tanh_action ? 0.5f * logf((1.0f + act) / (1.0f - act)) : act;
    const float d = (z - mu) / sd;
    float l = -0.5f * d * d - ls - kHalfLog2Pi;
    if (tanh_action) l -= logf(1.0f - act * act + 1e-6f);
    lp += l;
  }
  logp[b] = lp;
}
}  // namespace trl

TRL_API int trl_gaussian_log_prob(const float* mean, const float* log_std, int ls_stride, const float* actions,
                                  int64_t B, int act_dim, int tanh_action, float* logp, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 0 && act_dim >= 1, "trl_gaussian_log_prob: bad sizes");
  if (B == 0) return TRL_OK;
  TRL_REQUIRE(mean && log_std && actions && logp, "trl_gaussian_log_prob: null pointer");
  TRL_REQUIRE(ls_stride == 0 || ls_stride == act_dim, "trl_gaussian_log_prob: ls_stride must be 0 or act_dim");
  gaussian_logprob_kernel<<<static_cast<unsigned>(ceil_div<long long>(B, 256)), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(mean, log_std, ls_stride, actions, B, act_dim,
                                                                 tanh_action, logp);
  return check_launch("gaussian_logprob_kernel");
}
