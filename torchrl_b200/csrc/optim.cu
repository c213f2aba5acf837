// optim.cu -- K11: multi-tensor gradient-norm clip + Adam, and Polyak target update, on FLAT buffers.
//
// Replaces the per-parameter Python loops / many tiny kernels of
//   torch.nn.utils.clip_grad_norm_ call sites   /root/reference/torchrl/algo/on_policy/ppo.py:72,117,
//                                               /root/reference/torchrl/algo/off_policy/twin_sac_q.py:169-184
//   optimizer.step() (torch.optim.Adam)         ppo.py:74,119 ; a2c.py:29-39 (eps=1e-5)
//   soft_update_from_to                         /root/reference/torchrl/algo/utils.py:16-20
//   copy_model_params_from_to                   /root/reference/torchrl/algo/utils.py:23-25
// All parameters of all networks of an agent live in ONE contiguous fp32 buffer (and their
// gradients / Adam moments in three more); a "segment" is one network = one optimizer of the
// reference, with its own lr, max-norm and step count.  Two launches per update:
//   trl_grad_sumsq  : per-segment sum of squares (two-level, deterministic), bumps step counts
//   trl_adam_step   : clip coefficient + Adam + zero the gradient, one pass over the buffers
// The same flat gradient buffer is what NCCL all-reduces in the multi-GPU path (K12).
// HBM-bound: 4 reads + 4 writes of 4 B per parameter.
#include "reduce.cuh"

namespace trl {

constexpr int kMaxSeg = 8;
constexpr int kOptThreads = 256;

struct SegTable {
  long long begin[kMaxSeg + 1];  // element offsets into the flat buffer
  int nseg;
};

struct SumsqParams {
  const float* __restrict__ g;
  SegTable seg;
  double* __restrict__ partial;   // (grid)
  int* __restrict__ blk_seg;      // unused (segments are derived from offsets)
  double* __restrict__ out;       // (nseg) sum of squares, then (2*nseg) bias corrections [1-b1^t, sqrt(1-b2^t)]
  double beta1, beta2;
  int* __restrict__ step;         // (nseg) Adam step counts, incremented here for active segments
  unsigned* __restrict__ ticket;
  unsigned active_mask;           // which segments take part in this update
  int blocks_per_seg;
};

// grid = nseg * blocks_per_seg
__global__ void __launch_bounds__(kOptThreads) grad_sumsq_kernel(const SumsqParams p) {
  __shared__ double sh[32];
  const int s = blockIdx.x / p.blocks_per_seg, bi = blockIdx.x % p.blocks_per_seg;
  double acc = 0.0;
  if ((p.active_mask >> s) & 1u) {
    const long long lo = p.seg.begin[s], hi = p.seg.begin[s + 1];
    for (long long i = lo + static_cast<long long>(bi) * blockDim.x + threadIdx.x; i < hi;
         i += static_cast<long long>(p.blocks_per_seg) * blockDim.x) {
      const float v = p.g[i];
      acc += static_cast<double>(v) * v;
    }
  }
  acc = block_reduce_sum</*kReuse=*/false>(acc, sh);
  if (threadIdx.x == 0) p.partial[blockIdx.x] = acc;
  if (!last_cta(p.ticket, gridDim.x)) return;
  const int k = threadIdx.x;
  if (k < p.seg.nseg && ((p.active_mask >> k) & 1u))
    sumsq_segment_tail(p.partial + k * p.blocks_per_seg, p.blocks_per_seg, 1, k, p.seg.nseg, p.out, p.step, p.beta1,
                       p.beta2);
}

struct AdamParams {
  float* __restrict__ w;
  float* __restrict__ g;
  float* __restrict__ m;
  float* __restrict__ v;
  SegTable seg;
  const double* __restrict__ sumsq;   // (3*nseg) from grad_sumsq_kernel: sumsq, then bias corrections
  const float* __restrict__ lr;       // (nseg) device (LR schedules update it without re-capturing graphs)
  float max_norm[kMaxSeg];            // <= 0: no clipping
  float beta1, beta2, eps[kMaxSeg];
  unsigned active_mask;
  int zero_grad;
  float grad_scale;                   // multiplies g before everything (1/world_size after an all-reduce SUM)
  float* __restrict__ w_hi;           // optional TF32 planes of the updated weights for csrc/gemm_pair.cu:
  float* __restrict__ w_lo;           //   hi = tf32(w), lo = w - hi (both NULL: not maintained)
};

__device__ __forceinline__ void split_tf32_store(float w, float* __restrict__ hi, float* __restrict__ lo, long long i) {
  unsigned u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(w));
  const float h = __uint_as_float(u);
  hi[i] = h;
  lo[i] = w - h;
}

__device__ __forceinline__ void adam_element(const AdamParams& p, long long i, int s, float norm_s, float bc1,
                                             float bc2_sqrt) {
  float g = p.g[i] * p.grad_scale;
  if (p.max_norm[s] > 0.f) {
    // clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), applied only when < 1
    const float total_norm = norm_s * fabsf(p.grad_scale);
    const float coef = p.max_norm[s] / (total_norm + 1e-6f);
    if (coef < 1.0f) g *= coef;
  }
  const float m = p.beta1 * p.m[i] + (1.0f - p.beta1) * g;
  const float v = p.beta2 * p.v[i] + (1.0f - p.beta2) * g * g;
  p.m[i] = m;
  p.v[i] = v;
  const float denom = sqrtf(v) / bc2_sqrt + p.eps[s];
  const float w = p.w[i] - (p.lr[s] / bc1) * (m / denom);
  p.w[i] = w;
  if (p.w_hi) split_tf32_store(w, p.w_hi, p.w_lo, i);
  if (p.zero_grad) p.g[i] = 0.f;
}

__global__ void __launch_bounds__(kOptThreads) adam_step_kernel(const AdamParams p) {
  const long long total = p.seg.begin[p.seg.nseg];
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    int s = 0;
#pragma unroll
    for (int k = 1; k < kMaxSeg; ++k) s += (k < p.seg.nseg && i >= p.seg.begin[k]) ? 1 : 0;
    if (!((p.active_mask >> s) & 1u)) continue;
    adam_element(p, i, s, static_cast<float>(sqrt(p.sumsq[s])), static_cast<float>(p.sumsq[p.seg.nseg + 2 * s]),
                 static_cast<float>(p.sumsq[p.seg.nseg + 2 * s + 1]));
  }
}

__global__ void polyak_kernel(float* __restrict__ target, const float* __restrict__ source, long long n, float tau,
                              float* __restrict__ t_hi, float* __restrict__ t_lo) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // target * (1 - tau) + source * tau with every operation rounded on its own, as torch evaluates the soft update
    // (no contraction into an FFMA): the target and its TF32 planes equal torch's bit for bit
    const float w = __fadd_rn(__fmul_rn(target[i], __fsub_rn(1.0f, tau)), __fmul_rn(source[i], tau));
    target[i] = w;
    if (t_hi) split_tf32_store(w, t_hi, t_lo, i);
  }
}

static bool fill_segs(SegTable& t, const int64_t* seg_begin, int nseg) {
  if (nseg < 1 || nseg > kMaxSeg) return false;
  for (int i = 0; i <= nseg; ++i) t.begin[i] = seg_begin[i];
  for (int i = nseg + 1; i <= kMaxSeg; ++i) t.begin[i] = seg_begin[nseg];
  for (int i = 0; i < nseg; ++i) if (t.begin[i + 1] < t.begin[i]) return false;
  t.nseg = nseg;
  return true;
}

}  // namespace trl

TRL_API int trl_grad_sumsq_blocks(int nseg) { return nseg * 16; }

// seg_begin_host: (nseg+1) element offsets (host memory).  scratch: trl_grad_sumsq_blocks(nseg) doubles.
// sumsq3_out: (3*nseg) doubles = [sum of squares per segment | (1-b1^t, sqrt(1-b2^t)) per segment]
TRL_API int trl_grad_sumsq(const float* grad, const int64_t* seg_begin_host, int nseg, unsigned active_mask,
                           double* sumsq3_out, int* step_counts, double beta1, double beta2, double* scratch,
                           unsigned* ticket, void* stream) {
  using namespace trl;
  SumsqParams p;
  TRL_REQUIRE(seg_begin_host && fill_segs(p.seg, seg_begin_host, nseg), "trl_grad_sumsq: bad segment table");
  TRL_REQUIRE(grad && sumsq3_out && scratch && ticket, "trl_grad_sumsq: null pointer");
  p.g = grad; p.partial = scratch; p.blk_seg = nullptr; p.out = sumsq3_out; p.step = step_counts; p.beta1 = beta1; p.beta2 = beta2; p.ticket = ticket;
  p.active_mask = active_mask; p.blocks_per_seg = 16;
  grad_sumsq_kernel<<<nseg * 16, kOptThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("grad_sumsq_kernel");
}

TRL_API int trl_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, const int64_t* seg_begin_host,
                          int nseg, unsigned active_mask, const double* sumsq3, const float* lr_dev, const float* max_norm_host, const float* eps_host, float beta1,
                          float beta2, float grad_scale, int zero_grad, float* param_hi, float* param_lo, void* stream) {
  using namespace trl;
  AdamParams p;
  TRL_REQUIRE(seg_begin_host && fill_segs(p.seg, seg_begin_host, nseg), "trl_adam_step: bad segment table");
  TRL_REQUIRE(param && grad && exp_avg && exp_avg_sq && sumsq3 && lr_dev && max_norm_host && eps_host,
              "trl_adam_step: null pointer");
  p.w = param; p.g = grad; p.m = exp_avg; p.v = exp_avg_sq; p.sumsq = sumsq3; p.lr = lr_dev;
  for (int i = 0; i < kMaxSeg; ++i) {
    p.max_norm[i] = i < nseg ? max_norm_host[i] : 0.f;
    p.eps[i] = i < nseg ? eps_host[i] : 1e-8f;
  }
  TRL_REQUIRE((param_hi == nullptr) == (param_lo == nullptr), "trl_adam_step: param_hi / param_lo must be given together");
  p.beta1 = beta1; p.beta2 = beta2; p.active_mask = active_mask; p.zero_grad = zero_grad; p.grad_scale = grad_scale;
  p.w_hi = param_hi; p.w_lo = param_lo;
  const long long total = p.seg.begin[nseg];
  if (total == 0) return TRL_OK;
  long long blocks = ceil_div<long long>(total, kOptThreads);
  if (blocks > 4LL * kNumSM) blocks = 4LL * kNumSM;
  adam_step_kernel<<<static_cast<unsigned>(blocks), kOptThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("adam_step_kernel");
}

TRL_API int trl_polyak_update(float* target, const float* source, int64_t n, float tau, float* target_hi,
                              float* target_lo, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 0, "trl_polyak_update: negative size");
  if (n == 0) return TRL_OK;
  TRL_REQUIRE(target && source, "trl_polyak_update: null pointer");
  TRL_REQUIRE((target_hi == nullptr) == (target_lo == nullptr), "trl_polyak_update: target_hi / target_lo must be given together");
  long long blocks = ceil_div<long long>(n, 256);
  if (blocks > 4LL * kNumSM) blocks = 4LL * kNumSM;
  polyak_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(target, source, n, tau,
                                                                                          target_hi, target_lo);
  return check_launch("polyak_kernel");
}
