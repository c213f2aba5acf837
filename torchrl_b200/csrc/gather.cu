// gather.cu -- K7 / K9 / K4: time-row gather (minibatch assembly), ring write, advantage statistics.
//
// Replaces
//   OnPolicyReplayBufferBase.one_iteration  /root/reference/torchrl/replay_buffers/on_policy.py:72-91
//   BaseReplayBuffer.random_batch           /root/reference/torchrl/replay_buffers/base.py:39-51
//   BaseReplayBuffer.add_sample/_advance    /root/reference/torchrl/replay_buffers/base.py:19-37
//   advantage statistics / normalisation    /root/reference/torchrl/algo/on_policy/ppo.py:141-147
// Sampling granularity is the TIME ROW (SURVEY.md fact 5): a sampled index selects one
// contiguous (N, D) slab, so "gather" is b contiguous memcpys per key; all keys of a
// minibatch are moved by ONE launch (grid.y = key).  The row indices themselves are produced
// by the host with the reference's own NumPy calls (bit-exact replay indexing) and uploaded.
// HBM-bound: 2 x row_bytes per (row, key).
#include "reduce.cuh"

namespace trl {

constexpr int kMaxKeys = 8;

struct RowCopyParams {
  const char* src[kMaxKeys];
  char* dst[kMaxKeys];
  long long row_bytes[kMaxKeys];   // N * D * elemsize
  int nkeys;
  const long long* idx;            // row indices (device) or nullptr
  const int* pos_ptr;              // optional device scalar: use idx[(*pos_ptr)*rows + k]
  const int* row_ptr;              // optional device scalar: single row index (ring write at *row_ptr)
  int rows;                        // number of rows moved
  int scatter;                     // 0: dst[k] = src[idx[k]] ; 1: dst[idx[k]] = src[k]
  long long src_rows;              // rows in the gather source (bounds check), 0 = unchecked
  // ring write + advance in one launch: the last CTA to finish bumps the row index it has just been used with
  int* adv_ptr;                    // nullptr: plain copy; else *adv_ptr = (*adv_ptr + 1) % adv_T after ALL copies
  int adv_T;
  int* adv_size;                   // optional ring fill count, saturating at adv_T
  unsigned* ticket;                // zero between launches (with adv_ptr)
};

template <typename V>
__device__ __forceinline__ void copy_units(const char* s, char* d, long long nbytes, int tid, int nthr) {
  const V* sv = reinterpret_cast<const V*>(s);
  V* dv = reinterpret_cast<V*>(d);
  const long long n = nbytes / static_cast<long long>(sizeof(V));
  for (long long i = tid; i < n; i += nthr) dv[i] = sv[i];
}

// grid = (chunks_per_row, min(rows, 65535), nkeys); each CTA copies one chunk of rows blockIdx.y, blockIdx.y +
// gridDim.y, ... of one key (grid y is limited to 65535, a batch of rows is not)
__global__ void __launch_bounds__(256) row_copy_kernel(const RowCopyParams p) {
  const int key = blockIdx.z;
  const long long rb = p.row_bytes[key];
  // chunking: split the row over gridDim.x CTAs in 16B-aligned pieces
  long long per = ceil_div<long long>(rb, gridDim.x);
  per = (per + 15) & ~15LL;
  const long long lo = per * blockIdx.x;
  for (long long k = blockIdx.y; k < p.rows; k += gridDim.y) {
    long long r;
    if (p.row_ptr) r = *p.row_ptr;
    else if (p.idx) r = p.idx[(p.pos_ptr ? static_cast<long long>(*p.pos_ptr) * p.rows : 0) + k];
    else r = k;
    const long long srow = p.scatter ? k : r, drow = p.scatter ? r : k;
    if (lo < rb) {
      const long long len = min(per, rb - lo);
      const char* s = p.src[key] + srow * rb + lo;
      char* d = p.dst[key] + drow * rb + lo;
      const uintptr_t al = reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d) | static_cast<uintptr_t>(len);
      if ((al & 15) == 0) copy_units<uint4>(s, d, len, threadIdx.x, blockDim.x);
      else if ((al & 3) == 0) copy_units<unsigned>(s, d, len, threadIdx.x, blockDim.x);
      else copy_units<unsigned char>(s, d, len, threadIdx.x, blockDim.x);
    }
  }
  if (p.adv_ptr) {
    // every CTA has read *row_ptr by now; the last one to arrive advances it (one launch instead of copy + advance)
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (draw_ticket(p.ticket, gridDim.x * gridDim.y * gridDim.z)) {
        *p.adv_ptr = (*p.adv_ptr + 1) % p.adv_T;
        if (p.adv_size && *p.adv_size < p.adv_T) *p.adv_size += 1;
      }
    }
  }
}

// the raw moments (sum, sum of squares, max, min) of x[0..n) over the block (fp64 accumulation); true in thread 0,
// which holds them
__device__ __forceinline__ bool vec_block_moments(const float* __restrict__ x, long long n, double& s, double& q,
                                                  float& mx, float& mn) {
  s = 0.0; q = 0.0; mx = -INFINITY; mn = INFINITY;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = x[i];
    s += v; q += static_cast<double>(v) * v;
    mx = fmaxf(mx, v); mn = fminf(mn, v);
  }
  return block_moments(s, q, mx, mn);
}

// stats[0..3] = mean, unbiased std, max, min of x[0..n)   (one CTA; fp64 accumulation)
__global__ void __launch_bounds__(1024) vec_stats_kernel(const float* __restrict__ x, long long n,
                                                        float* __restrict__ stats) {
  double s, q;
  float mx, mn;
  if (vec_block_moments(x, n, s, q, mx, mn)) stats_from_moments(s, q, mx, mn, static_cast<double>(n), stats);
}

// raw moments of x[0..n): m[0..3] = sum, sum of squares, max, -min (fp64) -- the local half of a
// cross-rank statistic (K12: advantage normalisation over all ranks' envs, ppo.py:147)
__global__ void __launch_bounds__(1024) vec_moments_kernel(const float* __restrict__ x, long long n,
                                                          double* __restrict__ m) {
  double s, q;
  float mx, mn;
  if (vec_block_moments(x, n, s, q, mx, mn)) { m[0] = s; m[1] = q; m[2] = mx; m[3] = -static_cast<double>(mn); }
}

// [mean, unbiased std, max, min] from W ranks' raw moments g[r * stride ..][0..3] (sum, sum of squares, max, -min),
// combined in rank order
__device__ __forceinline__ void stats_from_rank_moments(const double* __restrict__ g, int W, long long stride,
                                                        double n_total, float* __restrict__ stats) {
  double s = 0.0, q = 0.0, mx = -INFINITY, nmn = -INFINITY;
  for (int r = 0; r < W; ++r) {
    const double* m = g + r * stride;
    s += m[0]; q += m[1];
    mx = fmax(mx, m[2]); nmn = fmax(nmn, m[3]);
  }
  stats_from_moments(s, q, mx, -nmn, n_total, stats);
}

// combine W ranks' raw moments (W x 4 doubles, rank order) into [mean, unbiased std, max, min]
__global__ void vec_stats_from_moments_kernel(const double* __restrict__ g, int W, double n_total,
                                              float* __restrict__ stats) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  stats_from_rank_moments(g, W, 4, n_total, stats);
}

// raw moments of every minibatch of an epoch in ONE launch: CTA u reduces the b time rows idx[u*b .. (u+1)*b) of x
// (rows of n floats) to out[4u ..] = sum, sum of squares, max, -min (fp64, fixed order) -- the minibatch membership is
// known as soon as the epoch's row permutations are drawn (ppo.py:27-39, on_policy.py:72-91), so the advantage
// statistics of ppo.py:141-147 need not be recomputed (nor all-reduced) per minibatch
__global__ void __launch_bounds__(1024) row_group_moments_kernel(const float* __restrict__ x, const long long* __restrict__ idx,
                                                                int b, long long n, double* __restrict__ out) {
  double s = 0.0, q = 0.0;
  float mx = -INFINITY, mn = INFINITY;
  for (int k = 0; k < b; ++k) {
    const float* row = x + idx[static_cast<long long>(blockIdx.x) * b + k] * n;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      const float v = row[i];
      s += v; q += static_cast<double>(v) * v;
      mx = fmaxf(mx, v); mn = fminf(mn, v);
    }
  }
  if (block_moments(s, q, mx, mn)) {
    double* o = out + 4LL * blockIdx.x;
    o[0] = s; o[1] = q; o[2] = mx; o[3] = -static_cast<double>(mn);
  }
}

// stats[4u ..] = mean, unbiased std, max, min of group u from W ranks' raw moments g (W, U, 4), rank order
__global__ void group_stats_from_moments_kernel(const double* __restrict__ g, int W, int U, double n_total,
                                                float* __restrict__ stats) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= U) return;
  stats_from_rank_moments(g + 4LL * u, W, 4LL * U, n_total, stats + 4 * u);
}

}  // namespace trl

static int launch_row_copy(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                           const int64_t* idx, const int* pos_ptr, const int* row_ptr, int rows, int scatter,
                           void* stream, const char* who, int* adv_ptr = nullptr, int adv_T = 1, int* adv_size = nullptr,
                           unsigned* ticket = nullptr) {
  using namespace trl;
  TRL_REQUIRE(nkeys >= 1 && nkeys <= kMaxKeys, "%s: nkeys %d not in 1..%d", who, nkeys, kMaxKeys);
  TRL_REQUIRE(rows >= 0, "%s: negative row count", who);
  if (rows == 0) return TRL_OK;
  TRL_REQUIRE(src && dst && row_bytes, "%s: null key table", who);
  RowCopyParams p;
  long long max_rb = 0;
  for (int i = 0; i < nkeys; ++i) {
    TRL_REQUIRE(src[i] && dst[i] && row_bytes[i] > 0, "%s: key %d has a null pointer or empty row", who, i);
    p.src[i] = static_cast<const char*>(src[i]);
    p.dst[i] = static_cast<char*>(dst[i]);
    p.row_bytes[i] = row_bytes[i];
    max_rb = max_rb > row_bytes[i] ? max_rb : row_bytes[i];
  }
  p.nkeys = nkeys;
  p.idx = reinterpret_cast<const long long*>(idx);
  p.pos_ptr = pos_ptr;
  p.row_ptr = row_ptr;
  p.rows = rows;
  p.scatter = scatter;
  p.src_rows = 0;
  p.adv_ptr = adv_ptr; p.adv_T = adv_T; p.adv_size = adv_size; p.ticket = ticket;
  // ~16 KB per CTA, but never more CTAs than ~8 waves of the chip
  long long chunks = ceil_div<long long>(max_rb, 16384);
  const long long cap = ceil_div<long long>(8LL * kNumSM, static_cast<long long>(rows) * nkeys);
  if (chunks > cap) chunks = cap < 1 ? 1 : cap;
  const unsigned grid_rows = rows < 65535 ? static_cast<unsigned>(rows) : 65535u;
  row_copy_kernel<<<dim3(static_cast<unsigned>(chunks), grid_rows, nkeys), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("row_copy_kernel");
}

TRL_API int trl_row_gather(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                           const int64_t* idx, const int* pos_ptr, int rows, void* stream) {
  TRL_REQUIRE(idx, "trl_row_gather: null index pointer");
  return launch_row_copy(nkeys, src, dst, row_bytes, idx, pos_ptr, nullptr, rows, 0, stream, "trl_row_gather");
}

TRL_API int trl_ring_write(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                           const int* row_ptr, void* stream) {
  TRL_REQUIRE(row_ptr, "trl_ring_write: null row pointer");
  return launch_row_copy(nkeys, src, dst, row_bytes, nullptr, nullptr, row_ptr, 1, 1, stream, "trl_ring_write");
}

// trl_ring_write followed by trl_step_advance(row_ptr, T, size_ptr) in ONE launch: every key's row is written at
// *row_ptr, then (after all copies) *row_ptr = (*row_ptr + 1) % T and, if given, *size_ptr = min(*size_ptr + 1, T).
// ticket: one unsigned, zero-initialised once by the caller.
TRL_API int trl_ring_write_advance(int nkeys, const void* const* src, void* const* dst, const int64_t* row_bytes,
                                   int* row_ptr, int T, int* size_ptr, unsigned* ticket, void* stream) {
  TRL_REQUIRE(row_ptr && ticket && T >= 1, "trl_ring_write_advance: null pointer or T < 1");
  return launch_row_copy(nkeys, src, dst, row_bytes, nullptr, nullptr, row_ptr, 1, 1, stream, "trl_ring_write_advance",
                         row_ptr, T, size_ptr, ticket);
}

TRL_API int trl_vec_stats(const float* x, int64_t n, float* stats4, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 1, "trl_vec_stats: need at least one element");
  TRL_REQUIRE(x && stats4, "trl_vec_stats: null pointer");
  vec_stats_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(x, n, stats4);
  return check_launch("vec_stats_kernel");
}

TRL_API int trl_vec_moments(const float* x, int64_t n, double* moments4, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 1, "trl_vec_moments: need at least one element");
  TRL_REQUIRE(x && moments4, "trl_vec_moments: null pointer");
  vec_moments_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(x, n, moments4);
  return check_launch("vec_moments_kernel");
}

TRL_API int trl_vec_stats_from_moments(const double* gathered, int world, double n_total, float* stats4, void* stream) {
  using namespace trl;
  TRL_REQUIRE(world >= 1 && n_total >= 1, "trl_vec_stats_from_moments: bad sizes");
  TRL_REQUIRE(gathered && stats4, "trl_vec_stats_from_moments: null pointer");
  vec_stats_from_moments_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(gathered, world, n_total, stats4);
  return check_launch("vec_stats_from_moments_kernel");
}

// moments4 (groups, 4) doubles: raw moments of x's rows idx[u*b .. (u+1)*b), one CTA per group
TRL_API int trl_row_group_moments(const float* x, const int64_t* idx, int groups, int b, int64_t row_elems,
                                  double* moments4, void* stream) {
  using namespace trl;
  TRL_REQUIRE(groups >= 1 && b >= 1 && row_elems >= 1, "trl_row_group_moments: bad sizes");
  TRL_REQUIRE(x && idx && moments4, "trl_row_group_moments: null pointer");
  row_group_moments_kernel<<<static_cast<unsigned>(groups), 1024, 0, static_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<const long long*>(idx), b, row_elems, moments4);
  return check_launch("row_group_moments_kernel");
}

// stats4 (groups, 4) floats = mean, unbiased std, max, min per group from `world` ranks' moments (world, groups, 4)
TRL_API int trl_group_stats_from_moments(const double* gathered, int world, int groups, double n_total, float* stats4,
                                         void* stream) {
  using namespace trl;
  TRL_REQUIRE(world >= 1 && groups >= 1 && n_total >= 1, "trl_group_stats_from_moments: bad sizes");
  TRL_REQUIRE(gathered && stats4, "trl_group_stats_from_moments: null pointer");
  group_stats_from_moments_kernel<<<static_cast<unsigned>(ceil_div(groups, 128)), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      gathered, world, groups, n_total, stats4);
  return check_launch("group_stats_from_moments_kernel");
}
