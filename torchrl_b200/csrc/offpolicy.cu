// offpolicy.cu -- K10: TD-target assembly and loss reductions of the off-policy agents.
//
// Replaces the op-by-op torch graphs (and .item() syncs) of
//   TwinSACQ.update   /root/reference/torchrl/algo/off_policy/twin_sac_q.py:84-219
//       alpha loss :111-123, target :125-139, critic MSE :142-143, policy loss :145-160
//   SAC.update / TwinSAC.update   /root/reference/torchrl/algo/off_policy/sac.py:74-208, twin_sac.py:82-229
//       value target + value MSE + policy loss :128-144 / :138-156 (the rest reuses the kernels above)
//   TD3.update        /root/reference/torchrl/algo/off_policy/td3.py:57-154
//       target smoothing :75-84, target :86-90, actor loss :128-130
//   QRDQN.update      /root/reference/torchrl/algo/off_policy/qrdqn.py:22-74
//       + quantile_regression_loss / huber   /root/reference/torchrl/algo/utils.py:5-13
//   DQN.update        /root/reference/torchrl/algo/off_policy/dqn.py:38-74
// Every kernel returns the scalar loss (device), the gradient wrt the network outputs and the
// logged statistics; network forward/backward stays in PyTorch.  Reductions are two-level and
// deterministic (reduce.cuh: block_reduce_* per CTA, then the last CTA's thread 0 folds the partials
// serially in CTA order).  All HBM/latency-bound.
#include "reduce.cuh"

namespace trl {

constexpr int kOffThreads = 256;

// ---------------------------------------------------------------------------------------------
// y = r + (1-d)*gamma*(min(q1n,q2n) - alpha*logp_next)      (alpha = exp(*log_alpha); SAC)
// y = r + (1-d)*gamma* min(q1n,q2n)                          (log_alpha == nullptr;  TD3)
// also info[0] = mean(r)
struct TdTargetParams {
  const float* __restrict__ rewards;   // (B)
  const uint8_t* __restrict__ terminals;  // (B)
  const float* __restrict__ q1n;       // (B)
  const float* __restrict__ q2n;       // (B) or nullptr (single critic)
  const float* __restrict__ logp_next; // (B) or nullptr
  const float* __restrict__ log_alpha; // (1) or nullptr
  float* __restrict__ y;               // (B)
  float* __restrict__ info;            // [0] reward mean
  double* __restrict__ partial;
  unsigned* __restrict__ ticket;
  long long B;
  float gamma, fixed_alpha;
};

__global__ void __launch_bounds__(kOffThreads) td_target_kernel(const TdTargetParams p) {
  __shared__ double shd[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  float r = 0.f;
  if (b < p.B) {
    r = p.rewards[b];
    float v = p.q2n ? fminf(p.q1n[b], p.q2n[b]) : p.q1n[b];
    if (p.logp_next) {
      const float alpha = p.log_alpha ? expf(*p.log_alpha) : p.fixed_alpha;
      v -= alpha * p.logp_next[b];
    }
    const float nd = p.terminals[b] ? 0.f : 1.f;
    p.y[b] = r + nd * p.gamma * v;
  }
  const double s = block_reduce_sum(static_cast<double>(r), shd);
  if (threadIdx.x == 0) p.partial[blockIdx.x] = s;
  if (last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) {
    double acc = 0.0;
    for (unsigned i = 0; i < gridDim.x; ++i) acc += p.partial[i];
    p.info[0] = static_cast<float>(acc / static_cast<double>(p.B));
  }
}

// ---------------------------------------------------------------------------------------------
// TD3 target policy smoothing: a' = clamp(a + clamp(sigma*eps, -c, c), -1, 1)
__global__ void td3_smooth_kernel(const float* __restrict__ act, const float* __restrict__ eps, float sigma,
                                  float noise_clip, unsigned long long seed,
                                  const unsigned long long* __restrict__ rng_counter, long long n,
                                  float* __restrict__ out) {
  const long long i4 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  float z[4];
  if (eps) {
#pragma unroll
    for (int k = 0; k < 4; ++k) z[k] = (i4 + k < n) ? eps[i4 + k] : 0.f;
  } else {
    uint32_t r[4];
    Philox::gen(seed, (rng_counter ? *rng_counter : 0ull) * 0x100000000ull + static_cast<unsigned long long>(i4 >> 2),
                0x7D3u, r);
    box_muller(r[0], r[1], z[0], z[1]);
    box_muller(r[2], r[3], z[2], z[3]);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (i4 + k < n) {
      const float nz = fminf(fmaxf(sigma * z[k], -noise_clip), noise_clip);
      out[i4 + k] = fminf(fmaxf(act[i4 + k] + nz, -1.f), 1.f);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// SAC temperature: L_alpha = -mean(log_alpha * (logp + target_entropy)); one Adam step on log_alpha
// inside the kernel (torch.optim.Adam semantics, 1 parameter).  state = [exp_avg, exp_avg_sq, step].
struct AlphaParams {
  const float* __restrict__ logp;  // (B) log pi(a~|s), treated as a constant
  float* __restrict__ log_alpha;   // (1)
  float* __restrict__ state;       // (3)
  float* __restrict__ info;        // [0] alpha (post-step) [1] alpha_loss (pre-step log_alpha)
  double* __restrict__ partial;
  unsigned* __restrict__ ticket;
  long long B;
  float target_entropy, lr, beta1, beta2, eps;
};

__global__ void __launch_bounds__(kOffThreads) sac_alpha_step_kernel(const AlphaParams p) {
  __shared__ double shd[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const double v = (b < p.B) ? static_cast<double>(p.logp[b] + p.target_entropy) : 0.0;
  const double s = block_reduce_sum(v, shd);
  if (threadIdx.x == 0) p.partial[blockIdx.x] = s;
  if (last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) {
    double acc = 0.0;
    for (unsigned i = 0; i < gridDim.x; ++i) acc += p.partial[i];
    const float mean_term = static_cast<float>(acc / static_cast<double>(p.B));
    const float la = *p.log_alpha;
    const float g = -mean_term;                      // dL/dlog_alpha
    const float loss = -la * mean_term;
    const float step = p.state[2] + 1.f;
    const float m = p.beta1 * p.state[0] + (1.f - p.beta1) * g;
    const float vv = p.beta2 * p.state[1] + (1.f - p.beta2) * g * g;
    const double bc1 = 1.0 - pow_int(static_cast<double>(p.beta1), step);
    const double bc2 = 1.0 - pow_int(static_cast<double>(p.beta2), step);
    const float denom = sqrtf(vv) / static_cast<float>(sqrt(bc2)) + p.eps;
    const float la_new = la - (p.lr / static_cast<float>(bc1)) * (m / denom);
    p.state[0] = m; p.state[1] = vv; p.state[2] = step;
    *p.log_alpha = la_new;
    p.info[0] = expf(la_new);
    p.info[1] = loss;
  }
}

// ---------------------------------------------------------------------------------------------
// SAC policy loss: L = mean(alpha*logp - min(q1,q2)); gradients wrt logp, q1, q2 (torch.min tie: split).
// Also the statistics the reference logs for log_probs (mean/std/max/min).
struct SacPolicyParams {
  const float* __restrict__ logp;      // (B)
  const float* __restrict__ q1;        // (B)
  const float* __restrict__ q2;        // (B)
  const float* __restrict__ log_alpha; // (1) or nullptr (alpha = fixed_alpha)
  float* __restrict__ g_logp;          // (B)
  float* __restrict__ g_q1;            // (B)
  float* __restrict__ g_q2;            // (B)
  float* __restrict__ info;            // [0] policy_loss [1..4] logp mean/std/max/min
  double* __restrict__ partial;        // (grid, 5)
  unsigned* __restrict__ ticket;
  long long B;
  float fixed_alpha;
};

__global__ void __launch_bounds__(kOffThreads) sac_policy_loss_kernel(const SacPolicyParams p) {
  __shared__ double shd[32];
  __shared__ float shf[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool ok = b < p.B;
  const float alpha = p.log_alpha ? expf(*p.log_alpha) : p.fixed_alpha;
  const float invB = 1.0f / static_cast<float>(p.B);
  float L = 0.f, lp = 0.f;
  if (ok) {
    lp = p.logp[b];
    const float a = p.q1[b], c = p.q2[b];
    L = alpha * lp - fminf(a, c);
    p.g_logp[b] = alpha * invB;
    p.g_q1[b] = (a < c) ? -invB : (a > c ? 0.f : -0.5f * invB);
    p.g_q2[b] = (c < a) ? -invB : (c > a ? 0.f : -0.5f * invB);
  }
  double* pp = p.partial + static_cast<long long>(blockIdx.x) * 5;
  double r;
  float f;
  r = block_reduce_sum(static_cast<double>(L), shd);                      if (threadIdx.x == 0) pp[0] = r;
  r = block_reduce_sum(ok ? static_cast<double>(lp) : 0.0, shd);          if (threadIdx.x == 0) pp[1] = r;
  r = block_reduce_sum(ok ? static_cast<double>(lp) * lp : 0.0, shd);     if (threadIdx.x == 0) pp[2] = r;
  f = block_reduce_max(ok ? lp : -INFINITY, shf);                         if (threadIdx.x == 0) pp[3] = f;
  f = block_reduce_max(ok ? -lp : -INFINITY, shf);                        if (threadIdx.x == 0) pp[4] = -f;
  if (last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) {
    double t[5] = {0.0, 0.0, 0.0, -INFINITY, INFINITY};
    for (unsigned i = 0; i < gridDim.x; ++i) {
      const double* q = p.partial + static_cast<long long>(i) * 5;
      t[0] += q[0]; t[1] += q[1]; t[2] += q[2]; t[3] = fmax(t[3], q[3]); t[4] = fmin(t[4], q[4]);
    }
    const double Bn = static_cast<double>(p.B);
    const double mean = t[1] / Bn;
    const double var = (t[2] - t[1] * mean) / (Bn - 1.0);
    p.info[0] = static_cast<float>(t[0] / Bn);
    p.info[1] = static_cast<float>(mean);
    p.info[2] = static_cast<float>(sqrt(var > 0.0 ? var : 0.0));
    p.info[3] = static_cast<float>(t[3]);
    p.info[4] = static_cast<float>(t[4]);
  }
}

// ---------------------------------------------------------------------------------------------
// SAC / TwinSAC with a state-value network (sac.py:128-144, twin_sac.py:138-156):
//   m = min(qn1, qn2) (or qn1),  t = m - alpha*logp  (detached)
//   vf_loss = mean((v - t)^2),                 g_v    = 2(v - t)/B
//   reparameterised: L = mean(alpha*logp - m),  g_logp = alpha/B, g_qn per torch.min's backward (tie: split)
//   otherwise:       c = alpha*logp - (m - v) (detached), L = mean(logp*c), g_logp = c/B, g_qn = 0
// plus the log_probs mean/std/max/min the reference logs.
struct SacVParams {
  const float* __restrict__ logp;      // (B)
  const float* __restrict__ qn1;       // (B)
  const float* __restrict__ qn2;       // (B) or nullptr (single critic)
  const float* __restrict__ v;         // (B) V(s)
  const float* __restrict__ log_alpha; // (1) or nullptr (alpha = fixed_alpha)
  float* __restrict__ g_logp;          // (B)
  float* __restrict__ g_qn1;           // (B)
  float* __restrict__ g_qn2;           // (B) or nullptr (with qn2)
  float* __restrict__ g_v;             // (B)
  float* __restrict__ info;            // [0] policy_loss [1] vf_loss [2..5] logp mean/std/max/min
  double* __restrict__ partial;        // (grid, 5): 4 sums, then max/min packed as two floats
  unsigned* __restrict__ ticket;
  long long B;
  float fixed_alpha;
  int reparam;
};

__global__ void __launch_bounds__(kOffThreads) sac_v_loss_kernel(const SacVParams p) {
  __shared__ double shd[32];
  __shared__ float shf[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool ok = b < p.B;
  const float alpha = p.log_alpha ? expf(*p.log_alpha) : p.fixed_alpha;
  const float invB = 1.0f / static_cast<float>(p.B);
  float L = 0.f, Lv = 0.f, lp = 0.f;
  if (ok) {
    lp = p.logp[b];
    const float a = p.qn1[b];
    const float c = p.qn2 ? p.qn2[b] : a;
    const float m = p.qn2 ? fminf(a, c) : a;
    const float v = p.v[b];
    const float dv = v - (m - alpha * lp);
    Lv = dv * dv;
    p.g_v[b] = 2.f * dv * invB;
    if (p.reparam) {
      L = alpha * lp - m;
      p.g_logp[b] = alpha * invB;
      if (p.qn2) {
        p.g_qn1[b] = (a < c) ? -invB : (a > c ? 0.f : -0.5f * invB);
        p.g_qn2[b] = (c < a) ? -invB : (c > a ? 0.f : -0.5f * invB);
      } else {
        p.g_qn1[b] = -invB;
      }
    } else {
      const float cc = alpha * lp - (m - v);
      L = lp * cc;
      p.g_logp[b] = cc * invB;
      p.g_qn1[b] = 0.f;
      if (p.qn2) p.g_qn2[b] = 0.f;
    }
  }
  double* pp = p.partial + static_cast<long long>(blockIdx.x) * 5;
  double r;
  float f;
  r = block_reduce_sum(static_cast<double>(L), shd);                      if (threadIdx.x == 0) pp[0] = r;
  r = block_reduce_sum(static_cast<double>(Lv), shd);                     if (threadIdx.x == 0) pp[1] = r;
  r = block_reduce_sum(ok ? static_cast<double>(lp) : 0.0, shd);          if (threadIdx.x == 0) pp[2] = r;
  r = block_reduce_sum(ok ? static_cast<double>(lp) * lp : 0.0, shd);     if (threadIdx.x == 0) pp[3] = r;
  float2* mm = reinterpret_cast<float2*>(pp + 4);
  f = block_reduce_max(ok ? lp : -INFINITY, shf);                         if (threadIdx.x == 0) mm->x = f;
  f = block_reduce_max(ok ? -lp : -INFINITY, shf);                        if (threadIdx.x == 0) mm->y = -f;
  if (last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) {
    double t[4] = {0.0, 0.0, 0.0, 0.0};
    float mx = -INFINITY, mn = INFINITY;
    for (unsigned i = 0; i < gridDim.x; ++i) {
      const double* q = p.partial + static_cast<long long>(i) * 5;
      t[0] += q[0]; t[1] += q[1]; t[2] += q[2]; t[3] += q[3];
      const float2 e = *reinterpret_cast<const float2*>(q + 4);
      mx = fmaxf(mx, e.x); mn = fminf(mn, e.y);
    }
    const double Bn = static_cast<double>(p.B);
    const double mean = t[2] / Bn;
    const double var = (t[3] - t[2] * mean) / (Bn - 1.0);   // B == 1: 0/0 = NaN, torch's std of one element
    p.info[0] = static_cast<float>(t[0] / Bn);
    p.info[1] = static_cast<float>(t[1] / Bn);
    p.info[2] = static_cast<float>(mean);
    p.info[3] = static_cast<float>(p.B > 1 ? sqrt(var > 0.0 ? var : 0.0) : NAN);
    p.info[4] = mx;
    p.info[5] = mn;
  }
}

// ---------------------------------------------------------------------------------------------
// MSE(pred, target) for two critics at once: loss_k = mean((q_k - y)^2), g_k = 2(q_k - y)/B.
// kWeighted (prioritised replay): loss_k = mean(w_b (q_k - y)^2), g_k = ((2(q_k - y)) w_b) / B, td_out (B, critics) =
// the unweighted |q_k - y|; weights and td_out may each be null.  w_b = 1 gives the unweighted bits.
struct TwinMseParams {
  const float* __restrict__ q1;
  const float* __restrict__ q2;   // or nullptr
  const float* __restrict__ y;
  float* __restrict__ g1;
  float* __restrict__ g2;
  float* __restrict__ info;       // [0] loss1 [1] loss2
  double* __restrict__ partial;   // (grid, 2)
  unsigned* __restrict__ ticket;
  long long B;
  const float* __restrict__ weights;  // (B) importance weights or nullptr (kWeighted only)
  float* __restrict__ td_out;         // (B, 1 or 2) or nullptr (kWeighted only)
};

template <bool kWeighted>
__global__ void __launch_bounds__(kOffThreads) twin_mse_kernel(const TwinMseParams p) {
  __shared__ double shd[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const float invB = 1.0f / static_cast<float>(p.B);
  float l1 = 0.f, l2 = 0.f;
  if (b < p.B) {
    const float y = p.y[b];
    const float w = kWeighted && p.weights ? p.weights[b] : 1.f;
    const int nc = p.q2 ? 2 : 1;
    const float d1 = p.q1[b] - y;
    l1 = kWeighted ? d1 * d1 * w : d1 * d1;
    p.g1[b] = kWeighted ? 2.f * d1 * w * invB : 2.f * d1 * invB;
    if (kWeighted && p.td_out) p.td_out[b * nc] = fabsf(d1);
    if (p.q2) {
      const float d2 = p.q2[b] - y;
      l2 = kWeighted ? d2 * d2 * w : d2 * d2;
      p.g2[b] = kWeighted ? 2.f * d2 * w * invB : 2.f * d2 * invB;
      if (kWeighted && p.td_out) p.td_out[b * nc + 1] = fabsf(d2);
    }
  }
  double r = block_reduce_sum(static_cast<double>(l1), shd);
  if (threadIdx.x == 0) p.partial[2 * blockIdx.x] = r;
  r = block_reduce_sum(static_cast<double>(l2), shd);
  if (threadIdx.x == 0) p.partial[2 * blockIdx.x + 1] = r;
  if (last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) {
    double a = 0.0, c = 0.0;
    for (unsigned i = 0; i < gridDim.x; ++i) { a += p.partial[2 * i]; c += p.partial[2 * i + 1]; }
    p.info[0] = static_cast<float>(a / static_cast<double>(p.B));
    p.info[1] = static_cast<float>(c / static_cast<double>(p.B));
  }
}

// ---------------------------------------------------------------------------------------------
// QR-DQN (one CTA per sample):
//   theta_i  = pred[b, act_b, i]                                  (qrdqn.py:38-44)
//   a*       = argmax_a mean_j next[b, a, j]                      (qrdqn.py:46-50)
//   y_j      = r_b + gamma*(1-d_b)*next[b, a*, j]                 (qrdqn.py:52-55)
//   loss     = mean_{b,j,i} huber(y_j - theta_i) * |tau_i - 1[y_j - theta_i < 0]|   (utils.py:5-9)
//   grad[b, act_b, i] = d loss / d theta_i ; zero elsewhere.
// DQN is the Q == 1 special case with a plain squared error (dqn.py:53-60): handled by `mse`.
struct QrParams {
  const float* __restrict__ pred;       // (B, A, Q)
  const float* __restrict__ next;       // (B, A, Q) target network on next_obs
  const float* __restrict__ actions;    // (B) action index stored as float
  const float* __restrict__ rewards;    // (B)
  const uint8_t* __restrict__ terminals;// (B)
  const float* __restrict__ weights;    // (B) importance weights (prioritised replay) or nullptr
  float* __restrict__ td_out;           // (B) per-sample loss magnitude (new priority signal) or nullptr
  float* __restrict__ grad;             // (B, A, Q)
  float* __restrict__ info;             // [0] loss [1] mean q_s_a [2] mean reward
  double* __restrict__ partial;         // (B, 3)
  unsigned* __restrict__ ticket;
  int B, A, Q;
  float gamma, kappa;
  int mse;                              // 1: DQN -- (theta - y)^2 with y from max_a next (Q must be 1)
};

// dynamic smem: theta[Q], y[Q], amean[A]
__global__ void __launch_bounds__(kOffThreads) qr_loss_kernel(const QrParams p) {
  extern __shared__ float sm[];
  __shared__ double shd[32];
  __shared__ int s_astar;
  float* s_theta = sm;
  float* s_y = sm + p.Q;
  float* s_am = sm + 2 * p.Q;
  const int b = blockIdx.x, A = p.A, Q = p.Q, tid = threadIdx.x, nthr = blockDim.x;
  const float* nb = p.next + static_cast<long long>(b) * A * Q;
  const float* pb = p.pred + static_cast<long long>(b) * A * Q;
  float* gb = p.grad + static_cast<long long>(b) * A * Q;
  // per-action mean of the target quantiles (warp per action)
  const int lane = tid & 31, wid = tid >> 5, nw = nthr >> 5;
  for (int a = wid; a < A; a += nw) {
    float s = 0.f;
    for (int j = lane; j < Q; j += 32) s += nb[a * Q + j];
    s = warp_sum(s);
    if (lane == 0) s_am[a] = s / static_cast<float>(Q);
  }
  for (int i = tid; i < A * Q; i += nthr) gb[i] = 0.f;
  __syncthreads();
  if (tid == 0) {
    int best = 0;
    float bv = s_am[0];
    for (int a = 1; a < A; ++a) if (s_am[a] > bv) { bv = s_am[a]; best = a; }  // first max, like torch.max
    s_astar = best;
  }
  __syncthreads();
  const int act = static_cast<int>(p.actions[b]);
  const float r = p.rewards[b];
  const float nd = p.terminals[b] ? 0.f : 1.f;
  for (int j = tid; j < Q; j += nthr) {
    s_theta[j] = pb[act * Q + j];
    s_y[j] = r + p.gamma * nd * nb[s_astar * Q + j];
  }
  __syncthreads();
  double lsum = 0.0, qsum = 0.0;
  const float wb = p.weights ? p.weights[b] : 1.0f;       // importance weight of this sample
  const float scale = wb / (static_cast<float>(p.B) * static_cast<float>(Q) * static_cast<float>(Q));
  for (int i = tid; i < Q; i += nthr) {
    const float th = s_theta[i];
    qsum += th;
    float g = 0.f;
    if (p.mse) {
      const float d = th - s_y[0];
      lsum += static_cast<double>(d) * d;
      g = 2.f * d * wb / static_cast<float>(p.B);
    } else {
      const float tau = (2.f * i + 1.f) / (2.f * Q);
      float acc_l = 0.f, acc_g = 0.f;
      for (int j = 0; j < Q; ++j) {
        const float u = s_y[j] - th;
        const float au = fabsf(u);
        const float w = fabsf(tau - (u < 0.f ? 1.f : 0.f));
        const float hub = au < p.kappa ? 0.5f * u * u : p.kappa * (au - 0.5f * p.kappa);
        const float dh = au < p.kappa ? u : (u > 0.f ? p.kappa : -p.kappa);   // d huber / du
        acc_l += hub * w;
        acc_g -= dh * w;                                                      // du/dtheta = -1
      }
      lsum += acc_l;
      g = acc_g * scale;
    }
    gb[act * Q + i] = g;
  }
  double v = block_reduce_sum(lsum, shd);
  if (tid == 0) {
    p.partial[3 * b] = v * wb;
    // un-weighted per-sample loss magnitude: |TD| for DQN, mean quantile-Huber loss for QR-DQN
    if (p.td_out) p.td_out[b] = p.mse ? sqrtf(static_cast<float>(v)) : static_cast<float>(v / (static_cast<double>(Q) * Q));
  }
  v = block_reduce_sum(qsum, shd);
  if (tid == 0) { p.partial[3 * b + 1] = v; p.partial[3 * b + 2] = r; }
  if (last_cta(p.ticket, gridDim.x) && tid == 0) {
    double l = 0.0, q = 0.0, rr = 0.0;
    for (int i = 0; i < p.B; ++i) { l += p.partial[3 * i]; q += p.partial[3 * i + 1]; rr += p.partial[3 * i + 2]; }
    const double nB = static_cast<double>(p.B);
    p.info[0] = static_cast<float>(p.mse ? l / nB : l / (nB * Q * Q));
    p.info[1] = static_cast<float>(q / (nB * Q));
    p.info[2] = static_cast<float>(rr / nB);
  }
}

}  // namespace trl

static inline unsigned off_blocks(long long B) { return static_cast<unsigned>(trl::ceil_div<long long>(B, trl::kOffThreads)); }

TRL_API int64_t trl_offpolicy_scratch_doubles(int64_t B) {
  const int64_t per_cta = 5 * static_cast<int64_t>(trl::ceil_div<long long>(B, trl::kOffThreads));
  const int64_t per_sample = 3 * B;
  return per_cta > per_sample ? per_cta : per_sample;
}

TRL_API int trl_td_target(const float* rewards, const uint8_t* terminals, const float* q1_next, const float* q2_next,
                          const float* logp_next, const float* log_alpha, float fixed_alpha, float gamma, int64_t B,
                          float* y, float* info1, double* scratch, unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_td_target: empty batch");
  TRL_REQUIRE(rewards && terminals && q1_next && y && info1 && scratch && ticket, "trl_td_target: null pointer");
  TdTargetParams p{rewards, terminals, q1_next, q2_next, logp_next, log_alpha, y, info1, scratch, ticket, B, gamma,
                   fixed_alpha};
  td_target_kernel<<<off_blocks(B), kOffThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("td_target_kernel");
}

TRL_API int trl_td3_smooth_action(const float* action, const float* eps, float sigma, float noise_clip, uint64_t seed,
                                  const uint64_t* rng_counter, int64_t n, float* out, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 0, "trl_td3_smooth_action: negative size");
  if (n == 0) return TRL_OK;
  TRL_REQUIRE(action && out, "trl_td3_smooth_action: null pointer");
  td3_smooth_kernel<<<static_cast<unsigned>(ceil_div<long long>(ceil_div<long long>(n, 4), 256)), 256, 0,
                      static_cast<cudaStream_t>(stream)>>>(action, eps, sigma, noise_clip, seed,
                                                           reinterpret_cast<const unsigned long long*>(rng_counter),
                                                           n, out);
  return check_launch("td3_smooth_kernel");
}

TRL_API int trl_sac_alpha_step(const float* logp, float target_entropy, float* log_alpha, float* adam_state3, float lr,
                               float beta1, float beta2, float eps, int64_t B, float* info2, double* scratch,
                               unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_sac_alpha_step: empty batch");
  TRL_REQUIRE(logp && log_alpha && adam_state3 && info2 && scratch && ticket, "trl_sac_alpha_step: null pointer");
  AlphaParams p{logp, log_alpha, adam_state3, info2, scratch, ticket, B, target_entropy, lr, beta1, beta2, eps};
  sac_alpha_step_kernel<<<off_blocks(B), kOffThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("sac_alpha_step_kernel");
}

TRL_API int trl_sac_policy_loss(const float* logp, const float* q1, const float* q2, const float* log_alpha,
                                float fixed_alpha, int64_t B, float* g_logp, float* g_q1, float* g_q2, float* info5,
                                double* scratch, unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_sac_policy_loss: empty batch");
  TRL_REQUIRE(logp && q1 && q2 && g_logp && g_q1 && g_q2 && info5 && scratch && ticket,
              "trl_sac_policy_loss: null pointer");
  SacPolicyParams p{logp, q1, q2, log_alpha, g_logp, g_q1, g_q2, info5, scratch, ticket, B, fixed_alpha};
  sac_policy_loss_kernel<<<off_blocks(B), kOffThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("sac_policy_loss_kernel");
}

TRL_API int trl_sac_v_loss(const float* logp, const float* qn1, const float* qn2, const float* v_pred,
                           const float* log_alpha, float fixed_alpha, int reparameterization, int64_t B, float* g_logp,
                           float* g_qn1, float* g_qn2, float* g_v, float* info6, double* scratch, unsigned* ticket,
                           void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_sac_v_loss: empty batch");
  TRL_REQUIRE(logp && qn1 && v_pred && g_logp && g_qn1 && g_v && info6 && scratch && ticket,
              "trl_sac_v_loss: null pointer");
  TRL_REQUIRE(!qn2 || g_qn2, "trl_sac_v_loss: qn2 given without g_qn2");
  SacVParams p{logp, qn1, qn2, v_pred, log_alpha, g_logp, g_qn1, qn2 ? g_qn2 : nullptr, g_v, info6, scratch, ticket,
               B, fixed_alpha, reparameterization ? 1 : 0};
  sac_v_loss_kernel<<<off_blocks(B), kOffThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("sac_v_loss_kernel");
}

TRL_API int trl_twin_mse_loss(const float* q1, const float* q2, const float* y, int64_t B, float* g1, float* g2,
                              float* info2, double* scratch, unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_twin_mse_loss: empty batch");
  TRL_REQUIRE(q1 && y && g1 && info2 && scratch && ticket, "trl_twin_mse_loss: null pointer");
  TRL_REQUIRE(!q2 || g2, "trl_twin_mse_loss: q2 given without g2");
  TwinMseParams p{q1, q2, y, g1, g2, info2, scratch, ticket, B, nullptr, nullptr};
  twin_mse_kernel<false><<<off_blocks(B), kOffThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("twin_mse_kernel");
}

TRL_API int trl_twin_mse_loss_weighted(const float* q1, const float* q2, const float* y, const float* weights, int64_t B,
                                       float* g1, float* g2, float* td_out, float* info2, double* scratch,
                                       unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1, "trl_twin_mse_loss_weighted: empty batch");
  TRL_REQUIRE(q1 && y && g1 && info2 && scratch && ticket, "trl_twin_mse_loss_weighted: null pointer");
  TRL_REQUIRE(!q2 || g2, "trl_twin_mse_loss_weighted: q2 given without g2");
  TwinMseParams p{q1, q2, y, g1, g2, info2, scratch, ticket, B, weights, td_out};
  twin_mse_kernel<true><<<off_blocks(B), kOffThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("twin_mse_kernel");
}

TRL_API int trl_qr_dqn_loss(const float* pred, const float* next, const float* actions, const float* rewards,
                            const uint8_t* terminals, const float* weights, int B, int n_actions, int n_quantiles,
                            float gamma, float kappa, int mse, float* grad, float* td_out, float* info3,
                            double* scratch, unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1 && n_actions >= 1 && n_quantiles >= 1, "trl_qr_dqn_loss: bad sizes");
  TRL_REQUIRE(!mse || n_quantiles == 1, "trl_qr_dqn_loss: the DQN (mse) form needs n_quantiles == 1");
  TRL_REQUIRE(pred && next && actions && rewards && terminals && grad && info3 && scratch && ticket,
              "trl_qr_dqn_loss: null pointer");
  QrParams p{pred, next, actions, rewards, terminals, weights, td_out, grad, info3, scratch, ticket, B, n_actions, n_quantiles, gamma,
             kappa, mse};
  const size_t smem = sizeof(float) * (2 * n_quantiles + n_actions);
  TRL_REQUIRE(smem <= 48 * 1024, "trl_qr_dqn_loss: %d quantiles x %d actions exceed shared memory", n_quantiles,
              n_actions);
  qr_loss_kernel<<<B, kOffThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("qr_loss_kernel");
}
