// bootstrapped.cu -- Bootstrapped DQN: the masked multi-head TD loss and the pixel collector's per-env head / bootstrap
// mask decision.
//
// Replaces, on the device,
//   BootstrappedDQN.update           /root/reference/torchrl/algo/off_policy/bootstrapped_dqn.py:66-113
//       per head h: y_h = r + gamma*(1-d)*max_a' Q'_h(s', a')  (its own target head, no double-DQN)
//       loss = mean_b sum_h m_bh (Q_h(s,a) - y_h)^2 / H          (divided by H, not by the number of active heads)
//   BootstrappedDQN.take_actions / start_episode and BootstrappedDQNDiscretePolicy.sample_head / explore
//       (bootstrapped_dqn.py:22-62, policies/discrete_policies.py:92-115), vectorised over N envs: a head drawn
//       uniformly at the first step of every episode, the greedy action of that head, and one Bernoulli(p) mask row
//       over the H heads stored with every transition.
// The loss's reductions are two-level and deterministic (reduce.cuh: block_reduce_sum per CTA, then the last CTA's
// thread 0 folds the fp64 partials serially in CTA order), as in offpolicy.cu.
#include "reduce.cuh"

namespace trl {

constexpr int kBootThreads = 256;
constexpr uint32_t kBootStream = 0xB0075u;   // Philox stream id of the head / mask draws

// ---------------------------------------------------------------------------------------------
// One thread per sample b, looping over the heads in order.  pred / next / grad are (H, B, A): for a fixed head the
// threads of a warp touch 32 consecutive rows.
struct BootLossParams {
  const float* __restrict__ pred;        // (H, B, A) Q_h(s, .)
  const float* __restrict__ next;        // (H, B, A) target network Q'_h(s', .)
  const float* __restrict__ actions;     // (B) action index stored as float
  const float* __restrict__ rewards;     // (B)
  const uint8_t* __restrict__ terminals; // (B)
  const uint8_t* __restrict__ masks;     // (B, H) 0 / non-zero
  float* __restrict__ grad;              // (H, B, A), every element written
  float* __restrict__ info;              // [0] loss [1] mean over (b, h) of Q_h(s, a) [2] mean reward
  double* __restrict__ partial;          // (grid, 3)
  unsigned* __restrict__ ticket;
  long long B;
  int H, A;
  float gamma;
};

__global__ void __launch_bounds__(kBootThreads) bootstrapped_dqn_loss_kernel(const BootLossParams p) {
  __shared__ double shd[32];
  const long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int H = p.H, A = p.A;
  double lsum = 0.0, qsum = 0.0;
  float r = 0.f;
  if (b < p.B) {
    const int act = static_cast<int>(p.actions[b]);
    r = p.rewards[b];
    const float nd = p.terminals[b] ? 0.f : 1.f;
    // d loss / d Q_h(s, a) = 2 m (Q - y) / (H B); autograd's chain: mean (1/B), / H, * m, then 2 (Q - y)
    const float coef = (1.0f / static_cast<float>(p.B)) / static_cast<float>(H);
    for (int h = 0; h < H; ++h) {
      const long long row = (static_cast<long long>(h) * p.B + b) * A;
      const float* nr = p.next + row;
      float mx = nr[0];
      for (int a = 1; a < A; ++a) mx = fmaxf(mx, nr[a]);
      const float y = r + p.gamma * nd * mx;
      const float q = p.pred[row + act];
      const float d = q - y;
      const bool on = p.masks[b * H + h] != 0;
      if (on) lsum += static_cast<double>(d) * d;
      qsum += q;
      const float g = on ? 2.f * d * coef : 0.f;
      float* gr = p.grad + row;
      for (int a = 0; a < A; ++a) gr[a] = (a == act) ? g : 0.f;
    }
  }
  double v = block_reduce_sum(lsum, shd);
  if (threadIdx.x == 0) p.partial[3 * blockIdx.x] = v;
  v = block_reduce_sum(qsum, shd);
  if (threadIdx.x == 0) p.partial[3 * blockIdx.x + 1] = v;
  v = block_reduce_sum(static_cast<double>(r), shd);
  if (threadIdx.x == 0) p.partial[3 * blockIdx.x + 2] = v;
  if (last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) {
    double l = 0.0, q = 0.0, rr = 0.0;
    for (unsigned i = 0; i < gridDim.x; ++i) {
      l += p.partial[3 * i];
      q += p.partial[3 * i + 1];
      rr += p.partial[3 * i + 2];
    }
    const double nB = static_cast<double>(p.B);
    p.info[0] = static_cast<float>(l / (nB * H));
    p.info[1] = static_cast<float>(q / (nB * H));
    p.info[2] = static_cast<float>(rr / nB);
  }
}

// ---------------------------------------------------------------------------------------------
// One thread per env n.  Uniforms: u_head (N) and u_mask (N, H) given, or Philox4x32-10 keyed by
// (seed, (*rng_counter << 32) + n, kBootStream + k / 4), element k % 4, with k = 0 the head draw and k = 1 + j the
// mask draw of head j; the last CTA then advances *rng_counter by one.
struct BootActParams {
  const float* __restrict__ q;           // (H, N, A) all heads on the current observations
  const int* __restrict__ current_step;  // (N) the collector's per-env step counter; 0 = first step of an episode
  int* __restrict__ head;                // (N) per-env head, redrawn where current_step == 0
  float* __restrict__ action;            // (N) greedy action of the env's head, as float
  uint8_t* __restrict__ masks;           // (T, N, H) ring; row *top is written
  const int* __restrict__ top;           // device scalar: this transition's ring row
  const float* __restrict__ u_head;      // (N) or nullptr
  const float* __restrict__ u_mask;      // (N, H) or nullptr
  unsigned long long seed;
  unsigned long long* __restrict__ rng_counter;
  unsigned* __restrict__ ticket;
  long long N;
  int H, A;
  float p;
};

__device__ __forceinline__ float boot_uniform(const BootActParams& p, unsigned long long ctr, long long n, int k) {
  uint32_t r[4];
  Philox::gen(p.seed, ctr * 0x100000000ull + static_cast<unsigned long long>(n), kBootStream + k / 4, r);
  return static_cast<float>(r[k & 3] >> 8) * (1.0f / 16777216.0f);   // [0, 1)
}

__global__ void __launch_bounds__(kBootThreads) bootstrapped_act_kernel(const BootActParams p) {
  const long long n = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool philox = p.u_head == nullptr;
  if (n < p.N) {
    const int H = p.H, A = p.A;
    const unsigned long long ctr = philox ? *p.rng_counter : 0ull;
    int h;
    if (p.current_step[n] == 0) {
      const float u = philox ? boot_uniform(p, ctr, n, 0) : p.u_head[n];
      h = min(static_cast<int>(u * static_cast<float>(H)), H - 1);
      p.head[n] = h;
    } else {
      h = p.head[n];
    }
    const float* qr = p.q + (static_cast<long long>(h) * p.N + n) * A;
    int best = 0;
    float bv = qr[0];
    for (int a = 1; a < A; ++a) {
      const float v = qr[a];
      if (v > bv) { bv = v; best = a; }   // first maximum, like torch.max on the CPU
    }
    p.action[n] = static_cast<float>(best);
    uint8_t* mrow = p.masks + (static_cast<long long>(*p.top) * p.N + n) * H;
    for (int j = 0; j < H; ++j) {
      const float u = philox ? boot_uniform(p, ctr, n, 1 + j) : p.u_mask[n * H + j];
      mrow[j] = u < p.p ? 1 : 0;
    }
  }
  if (philox && last_cta(p.ticket, gridDim.x) && threadIdx.x == 0) *p.rng_counter += 1ull;
}

}  // namespace trl

TRL_API int trl_bootstrapped_dqn_loss(const float* pred, const float* next, const float* actions, const float* rewards,
                                      const uint8_t* terminals, const uint8_t* masks, int64_t B, int num_heads,
                                      int num_actions, float gamma, float* grad, float* info3, double* scratch,
                                      unsigned* ticket, void* stream) {
  using namespace trl;
  TRL_REQUIRE(B >= 1 && num_heads >= 1 && num_actions >= 2,
              "trl_bootstrapped_dqn_loss: bad sizes B=%lld H=%d A=%d (B >= 1, H >= 1, A >= 2)", (long long)B,
              num_heads, num_actions);
  TRL_REQUIRE(pred && next && actions && rewards && terminals && masks && grad && info3 && scratch && ticket,
              "trl_bootstrapped_dqn_loss: null pointer");
  BootLossParams p{pred, next, actions, rewards, terminals, masks, grad, info3, scratch, ticket, B, num_heads,
                   num_actions, gamma};
  bootstrapped_dqn_loss_kernel<<<static_cast<unsigned>(ceil_div<long long>(B, kBootThreads)), kBootThreads, 0,
                                 static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("bootstrapped_dqn_loss_kernel");
}

TRL_API int trl_bootstrapped_act(const float* q_all, const int* current_step, int* head, float* action,
                                 uint8_t* masks_ring, const int* top, const float* u_head, const float* u_mask,
                                 uint64_t seed, uint64_t* rng_counter, unsigned* ticket, int64_t N, int num_heads,
                                 int num_actions, float bernoulli_p, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && num_heads >= 1 && num_actions >= 1,
              "trl_bootstrapped_act: bad sizes N=%lld H=%d A=%d (N >= 0, H >= 1, A >= 1)", (long long)N, num_heads,
              num_actions);
  TRL_REQUIRE(bernoulli_p >= 0.f && bernoulli_p <= 1.f, "trl_bootstrapped_act: bernoulli_p=%g outside [0, 1]",
              (double)bernoulli_p);
  TRL_REQUIRE(q_all && current_step && head && action && masks_ring && top, "trl_bootstrapped_act: null pointer");
  TRL_REQUIRE((u_head == nullptr) == (u_mask == nullptr), "trl_bootstrapped_act: give both u_head and u_mask or neither");
  TRL_REQUIRE(u_head || (rng_counter && ticket), "trl_bootstrapped_act: null pointer: needs u_head/u_mask or "
              "rng_counter and ticket");
  if (N == 0) return TRL_OK;
  BootActParams p{q_all, current_step, head, action, masks_ring, top, u_head, u_mask, seed,
                  reinterpret_cast<unsigned long long*>(rng_counter), ticket, N, num_heads, num_actions, bernoulli_p};
  bootstrapped_act_kernel<<<static_cast<unsigned>(ceil_div<long long>(N, kBootThreads)), kBootThreads, 0,
                            static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("bootstrapped_act_kernel");
}
