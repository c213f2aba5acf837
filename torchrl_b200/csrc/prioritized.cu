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
// trl_per_sample: one CTA, a block-wide inclusive scan of <= 4096 priorities in shared memory (fp64 accumulation), then
// one binary search per drawn row.  The scan adds in its own order (per-thread runs, a warp scan, a scan across warps),
// not np.cumsum's sequential one.  The two prefixes are equal -- and the indices bit-exact vs the oracle -- whenever
// every partial sum is exact in fp64, e.g. when all priorities are integer multiples of one 2^-q and their total is
// below 2^(53-q).  Otherwise (priorities over a wide exponent range) the prefixes may differ in the last bits, and a
// drawn row may differ from the oracle's when its target lies within that rounding of a row boundary.
// trl_per_sample_rows: rings of up to 2^24 rows in two launches, the live size and the draw position read on the device
// (graph-safe).  Pass 1 runs the same block scan on each chunk of 4096 rows; pass 2 scans the chunk totals with it and
// resolves the draws on the two-level prefix fl(chunk offset + in-chunk prefix).  With one chunk the offset is 0.0 and
// the scan order is trl_per_sample's, so for size <= 4096 both return the same bits.
#include <climits>

#include "common.cuh"

namespace trl {

constexpr int kPerThreads = 1024;
constexpr int kPerMaxRows = 4096;   // rows one CTA scans: 32 KB of fp64 prefix in static shared memory
constexpr int kPerMaxChunks = 4096; // chunks of kPerMaxRows rows the draw pass scans: rings of up to 2^24 rows
constexpr int kPerChunkFields = 5;  // per chunk in the scratch: total, min positive, first / last positive row, offset

struct PerSampleParams {
  const float* __restrict__ prio;    // (rows) priorities (already ^alpha)
  const double* __restrict__ u;      // (b) uniforms in [0,1)
  long long* __restrict__ idx;       // (b) sampled rows
  float* __restrict__ weights;       // (b) importance weights (normalised by the max weight)
  int size, b;
  float beta;
};

// ---- the pieces both samplers are made of (one CTA of kPerThreads threads) ----------------------------------------
// Inclusive prefix of v[0..n), n <= kPerMaxRows, into pre[] (shared): each thread adds a run of consecutive elements in
// fp64, a warp scan of the run totals, then a scan across warps.  Every thread must call it; it ends with a barrier.
template <typename T>
__device__ __forceinline__ void block_prefix(const T* __restrict__ v, int n, double* pre, double* warp_tot) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (n + kPerThreads - 1) / kPerThreads;       // consecutive elements per thread
  const int lo = tid * per, hi = min(lo + per, n);
  double local = 0.0;
  for (int i = lo; i < hi; ++i) {
    local += static_cast<double>(v[i]);
    pre[i] = local;                                            // thread-local inclusive prefix
  }
  // exclusive scan of the per-thread totals: warp shuffle, then across warps
  double incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const double w = warp_tot[lane];
    double wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    warp_tot[lane] = wi - w;                                   // exclusive prefix of warp totals
  }
  __syncthreads();
  const double offset = warp_tot[wid] + (incl - local);
  for (int i = lo; i < hi; ++i) pre[i] += offset;
  __syncthreads();
}

// Running maximum of v[0..n) in place, n <= kPerMaxChunks, in the same thread runs as block_prefix.  Ends with a barrier.
__device__ __forceinline__ void block_running_max(double* v, int n, double* warp_max_buf) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int per = (n + kPerThreads - 1) / kPerThreads;
  const int lo = tid * per, hi = min(lo + per, n);
  double run = -INFINITY;
  for (int i = lo; i < hi; ++i) {
    run = fmax(run, v[i]);
    v[i] = run;
  }
  double incl = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = fmax(incl, t);
  }
  double before = __shfl_up_sync(0xffffffffu, incl, 1);       // maximum over the earlier lanes of this warp
  if (lane == 0) before = -INFINITY;
  if (lane == 31) warp_max_buf[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    double wi = warp_max_buf[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi = fmax(wi, t);
    }
    const double prev = __shfl_up_sync(0xffffffffu, wi, 1);
    warp_max_buf[lane] = lane ? prev : -INFINITY;             // maximum over the earlier warps
  }
  __syncthreads();
  before = fmax(before, warp_max_buf[wid]);
  for (int i = lo; i < hi; ++i) v[i] = fmax(v[i], before);
  __syncthreads();
}

// Over rows v[0..n): the minimum positive priority (INFINITY if none) and the first / last row with a positive
// priority (-1 if none), valid in every thread.  The minimum is exact in any order.  Ends with a barrier.
struct PositiveRows {
  float min;
  int first, last;
};

__device__ __forceinline__ PositiveRows block_positive_rows(const float* __restrict__ v, int n, float* s_min,
                                                            int* s_first, int* s_last) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float mn = INFINITY;
  int first = INT_MAX, last = -1;
  for (int i = tid; i < n; i += kPerThreads) {
    const float x = v[i];
    if (x > 0.f) {                                             // zero rows are never drawn: no weight to normalise
      mn = fminf(mn, x);
      first = min(first, i);
      last = i;
    }
  }
  mn = warp_min(mn);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  }
  if (lane == 0) { s_min[wid] = mn; s_first[wid] = first; s_last[wid] = last; }
  __syncthreads();
  PositiveRows r{INFINITY, INT_MAX, -1};
  for (int w = 0; w < kPerThreads / 32; ++w) {
    r.min = fminf(r.min, s_min[w]);
    r.first = min(r.first, s_first[w]);
    r.last = max(r.last, s_last[w]);
  }
  if (r.first == INT_MAX) r.first = -1;
  __syncthreads();
  return r;
}

// First i in [0, n) with prefix(i) > target, or n - 1 if there is none; prefix is non-decreasing.
template <typename Prefix>
__device__ __forceinline__ int first_above(const Prefix& prefix, int n, double target) {
  int a = 0, c = n - 1;
  while (a < c) {
    const int m = (a + c) >> 1;
    if (prefix(m) > target) c = m; else a = m + 1;
  }
  return a;
}

// The first row in [a, end) with a positive priority, or end.  A zero-priority row found by the search is a target at
// (or rounded past) a boundary: the scan's rounding stepped up at a zero row that starts a thread's run or a chunk.
__device__ __forceinline__ long long next_positive(const float* __restrict__ prio, long long a, long long end) {
  while (a < end && !(prio[a] > 0.f)) ++a;
  return a;
}

__device__ __forceinline__ double stratum_target(int k, double u, int b, double total) {
  return (static_cast<double>(k) + u) / static_cast<double>(b) * total;
}

__device__ __forceinline__ double max_weight(int size, float min_positive, double total, float beta) {
  return pow(static_cast<double>(size) * static_cast<double>(min_positive) / total, -static_cast<double>(beta));
}

__device__ __forceinline__ float draw_weight(float p, int size, double total, double max_w, float beta) {
  const double prob = static_cast<double>(p) / total;
  return static_cast<float>(pow(static_cast<double>(size) * prob, -static_cast<double>(beta)) / max_w);
}

// ---- one CTA, size <= kPerMaxRows ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPerThreads) per_sample_kernel(const PerSampleParams p) {
  __shared__ double pre[kPerMaxRows];
  __shared__ double warp_tot[32];
  __shared__ float s_min[32];
  __shared__ int s_first[32], s_last[32];
  block_prefix(p.prio, p.size, pre, warp_tot);
  const PositiveRows pos = block_positive_rows(p.prio, p.size, s_min, s_first, s_last);
  const double total = pre[p.size - 1];
  const double max_w = max_weight(p.size, pos.min, total, p.beta);
  const auto prefix = [&](int i) { return pre[i]; };
  for (int k = threadIdx.x; k < p.b; k += kPerThreads) {
    const double target = stratum_target(k, p.u[k], p.b, total);
    long long a = next_positive(p.prio, first_above(prefix, p.size, target), p.size);
    if (a == p.size) a = max(pos.last, 0);                     // none at or after it: the last positive row
    p.idx[k] = a;
    p.weights[k] = draw_weight(p.prio[a], p.size, total, max_w, p.beta);
  }
}

// ---- two passes, rings of up to kPerMaxChunks * kPerMaxRows rows -----------------------------------------------------
// scratch (doubles): [capacity) the in-chunk inclusive prefix of every live row, then kPerChunkFields arrays of one
// value per chunk: total, minimum positive priority, first and last positive row (global ids, -1: none), and the
// chunk's offset (the exclusive prefix of the chunk totals).
struct PerRowsParams {
  const float* __restrict__ prio;
  const int* __restrict__ size_ptr;  // live rows (device): the ring's size
  const double* __restrict__ u;      // uniforms; this draw reads u[*pos_ptr * b ..][0..b)
  const int* __restrict__ pos_ptr;
  long long* __restrict__ idx;
  float* __restrict__ weights;
  double* __restrict__ scratch;
  int capacity, chunks, b;
  float beta;
};

__device__ __forceinline__ int live_rows(const PerRowsParams& p) { return min(max(*p.size_ptr, 1), p.capacity); }

// One CTA per chunk of kPerMaxRows rows; chunks at or beyond the live size only mark themselves empty.
__global__ void __launch_bounds__(kPerThreads) per_chunk_kernel(const PerRowsParams p) {
  __shared__ double pre[kPerMaxRows];
  __shared__ double warp_tot[32];
  __shared__ float s_min[32];
  __shared__ int s_first[32], s_last[32];
  const int size = live_rows(p);
  const int c = blockIdx.x;
  const int start = c * kPerMaxRows;
  double* summary = p.scratch + p.capacity;
  if (start >= size) {
    if (threadIdx.x == 0) {
      summary[c] = 0.0;
      summary[p.chunks + c] = INFINITY;
      summary[2 * p.chunks + c] = -1.0;
      summary[3 * p.chunks + c] = -1.0;
    }
    return;
  }
  const int n = min(kPerMaxRows, size - start);
  const float* v = p.prio + start;
  block_prefix(v, n, pre, warp_tot);
  const PositiveRows pos = block_positive_rows(v, n, s_min, s_first, s_last);
  double* out = p.scratch + start;
  for (int i = threadIdx.x; i < n; i += kPerThreads) out[i] = pre[i];
  if (threadIdx.x == 0) {
    summary[c] = pre[n - 1];
    summary[p.chunks + c] = pos.min;
    summary[2 * p.chunks + c] = pos.first < 0 ? -1.0 : static_cast<double>(start + pos.first);
    summary[3 * p.chunks + c] = pos.last < 0 ? -1.0 : static_cast<double>(start + pos.last);
  }
}

// One CTA: scan the live chunks' totals, then resolve every draw.  The global prefix of row i of chunk c is
// fl(offset_c + in-chunk prefix_i).  The chunk is the first whose last row's prefix exceeds the target, found by a
// binary search over the running maximum of those last-row prefixes (the scan's rounding may lift one chunk's last
// prefix above the next chunk's offset); the row is trl_per_sample's binary search inside that chunk (the last chunk
// and its last row if nothing exceeds the target).  Where the prefix is exact (see above) it rises with the row, and
// the answer is the first row whose prefix exceeds the target, the oracle's searchsorted.  Over a wide exponent range
// the block scan's thread offsets round, so its prefix may dip by an ulp of the total; the searches then return a row
// within that rounding of the target, as trl_per_sample does, and with one chunk they are trl_per_sample's.
__global__ void __launch_bounds__(kPerThreads) per_draw_kernel(const PerRowsParams p) {
  __shared__ double pre[kPerMaxChunks];
  __shared__ double warp_tot[32];
  __shared__ float s_min[32];
  __shared__ int s_last[32];
  const int size = live_rows(p);
  const int live = (size + kPerMaxRows - 1) / kPerMaxRows;
  const double* totals = p.scratch + p.capacity;
  const double* mins = totals + p.chunks;
  const double* firsts = totals + 2 * p.chunks;
  const double* lasts = totals + 3 * p.chunks;
  double* offsets = p.scratch + p.capacity + 4 * p.chunks;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  block_prefix(totals, live, pre, warp_tot);
  // minimum positive priority and last positive row over the live chunks
  float mn = INFINITY;
  int last = -1;
  for (int c = tid; c < live; c += kPerThreads) {
    mn = fminf(mn, static_cast<float>(mins[c]));
    last = max(last, static_cast<int>(lasts[c]));
  }
  mn = warp_min(mn);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  if (lane == 0) { s_min[wid] = mn; s_last[wid] = last; }
  const double total = pre[live - 1];
  // the chunks' offsets, and the global prefix of each chunk's last row in place of the chunk prefix
  const int per = (live + kPerThreads - 1) / kPerThreads;     // <= 4
  double ends[kPerMaxChunks / kPerThreads];
  const int lo = tid * per;
#pragma unroll
  for (int j = 0; j < kPerMaxChunks / kPerThreads; ++j) {
    const int c = lo + j;
    if (j < per && c < live) {
      const double off = c ? pre[c - 1] : 0.0;
      offsets[c] = off;
      ends[j] = off + totals[c];
    }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kPerMaxChunks / kPerThreads; ++j)
    if (j < per && lo + j < live) pre[lo + j] = ends[j];
  for (int w = 0; w < kPerThreads / 32; ++w) {
    mn = fminf(mn, s_min[w]);
    last = max(last, s_last[w]);
  }
  __syncthreads();
  block_running_max(pre, live, warp_tot);
  const double max_w = max_weight(size, mn, total, p.beta);
  const double* u = p.u + static_cast<long long>(*p.pos_ptr) * p.b;
  const auto chunk_end = [&](int c) { return pre[c]; };
  for (int k = tid; k < p.b; k += kPerThreads) {
    const double target = stratum_target(k, u[k], p.b, total);
    const int c = first_above(chunk_end, live, target);      // live - 1 if no chunk's end exceeds the target
    const int start = c * kPerMaxRows, n = min(kPerMaxRows, size - start);
    const double off = offsets[c];
    const double* in_chunk = p.scratch + start;
    const auto prefix = [&](int i) { return off + in_chunk[i]; };
    long long a = next_positive(p.prio, start + first_above(prefix, n, target), start + n);
    if (a == start + n) {                                      // no positive row left in this chunk: the next one's
      a = -1;
      for (int d = c + 1; d < live && a < 0; ++d) a = static_cast<long long>(firsts[d]);
    }
    if (a < 0) a = max(last, 0);                               // none at or after it: the last positive row
    p.idx[k] = a;
    p.weights[k] = draw_weight(p.prio[a], size, total, max_w, p.beta);
  }
}

// prio[idx_k] = (mean_n |td[k][n]| + eps)^alpha ; *max_prio = max(*max_prio, new priorities).  A row drawn more than
// once takes the value of its last draw in batch order (the oracle's prio[idx] = new): a block writes only when no
// later draw holds its row, so the stored priorities do not depend on the order the blocks run in.
__global__ void __launch_bounds__(256) per_update_kernel(float* __restrict__ prio, const long long* __restrict__ idx,
                                                        const float* __restrict__ td, int b, int n, float alpha,
                                                        float eps, float* __restrict__ max_prio) {
  __shared__ double sh[32];
  const int k = blockIdx.x;
  const long long row = idx[k];
  int later = 0;
  for (int j = k + 1 + threadIdx.x; j < b; j += blockDim.x) later |= (idx[j] == row);
  later = __syncthreads_or(later);
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
      if (!later) prio[row] = pr;
      atomic_max_float(max_prio, pr);     // the running max takes every new value, duplicates included
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

TRL_API int trl_per_scratch_doubles(int capacity) {
  using namespace trl;
  if (capacity < 1 || capacity > kPerMaxChunks * kPerMaxRows) return -1;
  const int chunks = (capacity + kPerMaxRows - 1) / kPerMaxRows;
  return capacity + kPerChunkFields * chunks;
}

TRL_API int trl_per_sample_rows(const float* prio, int capacity, const int* size_ptr, const double* u, const int* pos_ptr,
                                int b, float beta, int64_t* idx, float* weights, double* scratch, void* stream) {
  using namespace trl;
  TRL_REQUIRE(capacity >= 1 && capacity <= kPerMaxChunks * kPerMaxRows, "trl_per_sample_rows: capacity %d not in 1..%d rows",
              capacity, kPerMaxChunks * kPerMaxRows);
  TRL_REQUIRE(b >= 1, "trl_per_sample_rows: empty batch");
  TRL_REQUIRE(prio && size_ptr && u && pos_ptr && idx && weights && scratch, "trl_per_sample_rows: null pointer");
  const int chunks = (capacity + kPerMaxRows - 1) / kPerMaxRows;
  PerRowsParams p{prio, size_ptr, u, pos_ptr, reinterpret_cast<long long*>(idx), weights, scratch, capacity, chunks, b,
                  beta};
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  per_chunk_kernel<<<chunks, kPerThreads, 0, s>>>(p);
  const int rc = check_launch("per_chunk_kernel");
  if (rc != TRL_OK) return rc;
  per_draw_kernel<<<1, kPerThreads, 0, s>>>(p);
  return check_launch("per_draw_kernel");
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
