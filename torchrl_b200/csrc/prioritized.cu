// prioritized.cu -- K9 (prioritised variant): proportional prioritised sampling of replay TIME ROWS.
//
// PARITY UNPINNED: the reference has no prioritised replay anywhere (SURVEY.md fact 7; grep for
// priorit|sumtree|segment finds nothing) although BASELINE.json config 4 asks for one.  The definition
// is this build's, restated on the CPU in oracle/ref_numpy.py (per_sample / per_update):
//   * granularity is the time row, like BaseReplayBuffer.random_batch
//     (/root/reference/torchrl/replay_buffers/base.py:39-51): one priority per stored row,
//     p_row = (mean_n |TD_{row,n}| + eps)^alpha, new rows enter with the running maximum priority;
//   * stratified proportional sampling (Schaul et al. 2016): segment k of b draws
//     target = (k + u_k)/b * sum(p), u_k ~ U[0,1) supplied by the caller (host np.random),
//     idx_k = first row whose inclusive prefix sum > target; a target that rounds up to the total (k = b-1, u_k
//     within 2^-53 of 1) draws the last row with a positive priority -- a zero-priority row is never drawn;
//   * importance weights w_k = (size * p_idx/sum)^-beta / max_w, max_w from the minimum positive priority;
//   * at least one of the `size` priorities must be positive (all zero: the sum is 0 and the weights are NaN;
//     the oracle refuses the case).
// One CTA: block-wide inclusive scan of <= 4096 priorities in shared memory (fp64 accumulation), then one
// binary search per drawn row.  The scan adds in its own order (per-thread runs, a warp scan, a scan across
// warps), not np.cumsum's sequential one.  The two prefixes are equal -- and the indices bit-exact vs the
// oracle -- whenever every partial sum is exact in fp64, e.g. when all priorities are integer multiples
// of one 2^-q and their total is below 2^(53-q).  Otherwise (priorities over a wide exponent range) the
// prefixes may differ in the last bits, and a drawn row may differ from the oracle's when its target lies
// within that rounding of a row boundary.
#include "common.cuh"

namespace trl {

constexpr int kPerThreads = 1024;
constexpr int kPerMaxRows = 4096;   // 32 KB of fp64 prefix in static shared memory

struct PerSampleParams {
  const float* __restrict__ prio;    // (rows) priorities (already ^alpha)
  const double* __restrict__ u;      // (b) uniforms in [0,1)
  long long* __restrict__ idx;       // (b) sampled rows
  float* __restrict__ weights;       // (b) importance weights (normalised by the max weight)
  int size, b;
  float beta;
};

__global__ void __launch_bounds__(kPerThreads) per_sample_kernel(const PerSampleParams p) {
  __shared__ double pre[kPerMaxRows];
  __shared__ double warp_tot[32];
  __shared__ float s_min[32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (p.size + kPerThreads - 1) / kPerThreads;   // consecutive rows per thread
  const int lo = tid * per, hi = min(lo + per, p.size);
  double local = 0.0;
  float mn = INFINITY;
  for (int i = lo; i < hi; ++i) {
    const float v = p.prio[i];
    local += static_cast<double>(v);
    pre[i] = local;                                            // thread-local inclusive prefix
    if (v > 0.f) mn = fminf(mn, v);                            // zero rows are never drawn: no weight to normalise
  }
  // exclusive scan of the per-thread totals: warp shuffle, then across warps
  double incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[wid] = incl;
  mn = warp_min(mn);
  if (lane == 0) s_min[wid] = mn;
  __syncthreads();
  if (wid == 0) {
    double w = warp_tot[lane];
    double wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    warp_tot[lane] = wi - w;                                   // exclusive prefix of warp totals
    float m = s_min[lane];
    m = warp_min(m);
    if (lane == 0) s_min[0] = m;
  }
  __syncthreads();
  const double offset = warp_tot[wid] + (incl - local);
  for (int i = lo; i < hi; ++i) pre[i] += offset;
  __syncthreads();
  const double total = pre[p.size - 1];
  const double max_w = pow(static_cast<double>(p.size) * static_cast<double>(s_min[0]) / total,
                           -static_cast<double>(p.beta));
  for (int k = tid; k < p.b; k += kPerThreads) {
    const double target = (static_cast<double>(k) + p.u[k]) / static_cast<double>(p.b) * total;
    int a = 0, c = p.size - 1;                                 // first i with pre[i] > target
    while (a < c) {
      const int m = (a + c) >> 1;
      if (pre[m] > target) c = m; else a = m + 1;
    }
    // a zero-priority row here is a target at (or rounded past) a boundary: the search fell through to size-1
    // (target == total), or the scan's rounding stepped up at a zero row starting a thread's run.  Take the next
    // row with a positive priority, else the last one before it.
    while (a < p.size - 1 && !(p.prio[a] > 0.f)) ++a;
    while (a > 0 && !(p.prio[a] > 0.f)) --a;
    p.idx[k] = a;
    const double prob = static_cast<double>(p.prio[a]) / total;
    p.weights[k] = static_cast<float>(pow(static_cast<double>(p.size) * prob, -static_cast<double>(p.beta)) / max_w);
  }
}

// prio[idx_k] = (mean_n |td[k][n]| + eps)^alpha ; *max_prio = max(*max_prio, new priorities)
__global__ void __launch_bounds__(256) per_update_kernel(float* __restrict__ prio, const long long* __restrict__ idx,
                                                        const float* __restrict__ td, int b, int n, float alpha,
                                                        float eps, float* __restrict__ max_prio) {
  __shared__ double sh[32];
  const int k = blockIdx.x;
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += fabs(static_cast<double>(td[static_cast<long long>(k) * n + i]));
  s = warp_sum(s);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) sh[wid] = s;
  __syncthreads();
  if (wid == 0) {
    s = lane < (blockDim.x >> 5) ? sh[lane] : 0.0;
    s = warp_sum(s);
    if (lane == 0) {
      const float pr = powf(static_cast<float>(s / n) + eps, alpha);
      prio[idx[k]] = pr;                  // duplicate rows in a batch: last writer wins (same as the oracle's loop
      atomic_max_float(max_prio, pr);     // order only if the values are equal; documented as unordered)
    }
  }
}

// priority of the row just written by the collector <- running max
__global__ void per_insert_kernel(float* prio, const int* row_ptr, const float* max_prio) {
  if (threadIdx.x == 0 && blockIdx.x == 0) prio[*row_ptr] = *max_prio;
}

}  // namespace trl

TRL_API int trl_per_sample(const float* prio, int size, const double* u, int b, float beta, int64_t* idx,
                           float* weights, void* stream) {
  using namespace trl;
  TRL_REQUIRE(size >= 1 && size <= kPerMaxRows, "trl_per_sample: size %d not in 1..%d rows", size, kPerMaxRows);
  TRL_REQUIRE(b >= 1, "trl_per_sample: empty batch");
  TRL_REQUIRE(prio && u && idx && weights, "trl_per_sample: null pointer");
  PerSampleParams p{prio, u, reinterpret_cast<long long*>(idx), weights, size, b, beta};
  per_sample_kernel<<<1, kPerThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("per_sample_kernel");
}

TRL_API int trl_per_update(float* prio, const int64_t* idx, const float* td, int b, int n, float alpha, float eps,
                           float* max_prio, void* stream) {
  using namespace trl;
  TRL_REQUIRE(b >= 1 && n >= 1, "trl_per_update: bad sizes");
  TRL_REQUIRE(prio && idx && td && max_prio, "trl_per_update: null pointer");
  per_update_kernel<<<b, 256, 0, static_cast<cudaStream_t>(stream)>>>(prio, reinterpret_cast<const long long*>(idx), td,
                                                                     b, n, alpha, eps, max_prio);
  return check_launch("per_update_kernel");
}

TRL_API int trl_per_insert(float* prio, const int* row_ptr, const float* max_prio, void* stream) {
  using namespace trl;
  TRL_REQUIRE(prio && row_ptr && max_prio, "trl_per_insert: null pointer");
  per_insert_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(prio, row_ptr, max_prio);
  return check_launch("per_insert_kernel");
}
