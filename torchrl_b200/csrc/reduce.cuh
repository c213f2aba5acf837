// reduce.cuh -- the deterministic reductions of this library: block reductions, the last-CTA ticket and the arithmetic
// that the reductions' tails share.
//
// Every reduction over more than one CTA is two-level: each CTA writes its partials, then takes a ticket (last_cta);
// the CTA that draws the last ticket sees every partial and folds them in a fixed order, so results do not depend on
// scheduling and no second launch is needed.  How the last CTA folds (serial, lane-strided, several loads in flight) is
// each kernel's own choice, because it fixes the summation order of that kernel's outputs.
#pragma once
#include "common.cuh"

namespace trl {

// ---- block reductions (blockDim.x a multiple of 32, <= 1024) -------------------------------------------------------
// One quantity: warp shuffles, one value per warp in sh[32], then warp 0 folds them with shuffles; the result is valid
// in warp 0.  The barrier before sh is written lets consecutive calls share sh; a kernel whose only block reduction
// this is may drop it (kReuse = false).
template <bool kReuse = true>
__device__ __forceinline__ double block_reduce_sum(double v, double* sh) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (kReuse) __syncthreads();
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  double r = 0.0;
  if (wid == 0) {
    r = lane < nw ? sh[lane] : 0.0;
    r = warp_sum(r);
  }
  return r;  // valid in warp 0
}
__device__ __forceinline__ float block_reduce_max(float v, float* sh) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  float r = -INFINITY;
  if (wid == 0) {
    r = lane < nw ? sh[lane] : -INFINITY;
    r = warp_max(r);
  }
  return r;
}

// Per-CTA partials of NS sums (fp64) and NM maxima in ONE barrier: every warp reduces each quantity with shuffles and
// lane 0 stores it in the per-warp tables sh_sum / sh_max; after the barrier thread k folds the warps' values of
// quantity k in warp order and writes out[k] (sums) or out[NS + k'] (maxima, as double).  Deterministic.
template <int NW, int NS, int NM>
__device__ __forceinline__ void block_partials(const double (&sums)[NS], const float (&maxs)[NM], double (*sh_sum)[NS],
                                               float (*sh_max)[NM], double* out) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NS; ++k) {
    const double w = warp_sum(sums[k]);
    if (lane == 0) sh_sum[wid][k] = w;
  }
#pragma unroll
  for (int k = 0; k < NM; ++k) {
    const float m = warp_max(maxs[k]);
    if (lane == 0) sh_max[wid][k] = m;
  }
  __syncthreads();
  const int k = threadIdx.x;
  if (k < NS) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) t += sh_sum[w][k];
    out[k] = t;
  } else if (k < NS + NM) {
    float m = -INFINITY;
#pragma unroll
    for (int w = 0; w < NW; ++w) m = fmaxf(m, sh_max[w][k - NS]);
    out[k] = static_cast<double>(m);
  }
}

// Raw moments (sum, sum of squares, max, min) of the threads' values, in place: warp shuffles, one barrier, then warp 0
// folds the per-warp values with shuffles.  Returns true in thread 0, which holds the results; the other warps leave
// at once.  The per-warp tables are this helper's own and are not guarded for reuse: one call per kernel.
__device__ __forceinline__ bool block_moments(double& s, double& q, float& mx, float& mn) {
  __shared__ double sh_s[32], sh_q[32];
  __shared__ float sh_mx[32], sh_mn[32];
  s = warp_sum(s); q = warp_sum(q); mx = warp_max(mx); mn = warp_min(mn);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) { sh_s[wid] = s; sh_q[wid] = q; sh_mx[wid] = mx; sh_mn[wid] = mn; }
  __syncthreads();
  if (wid != 0) return false;
  s = lane < nw ? sh_s[lane] : 0.0; q = lane < nw ? sh_q[lane] : 0.0;
  mx = lane < nw ? sh_mx[lane] : -INFINITY; mn = lane < nw ? sh_mn[lane] : INFINITY;
  s = warp_sum(s); q = warp_sum(q); mx = warp_max(mx); mn = warp_min(mn);
  return lane == 0;
}

// ---- the last-CTA ticket ---------------------------------------------------------------------------------------------
// `ticket` counts the arrivals of one launch; the caller zero-initialises it once.  Invariant: the winner -- the last of
// `arrivals` to draw -- resets it to zero before it exits (it does so as it draws: nobody is left to draw after it), so
// the next launch or graph replay starts from zero.  This is what keeps the kernels correct under graph replay.
//
// Thread-level half: for one thread whose CTA's writes are already published (__threadfence).  No barrier.
__device__ __forceinline__ bool draw_ticket(unsigned* ticket, unsigned arrivals) {
  const bool last = atomicAdd(ticket, 1u) == arrivals - 1;
  if (last) *ticket = 0u;
  return last;
}

// Called by every thread of a CTA once its partials are written; true in every thread of exactly one CTA, the last of
// `arrivals` to get here (gridDim.x for a whole 1-D grid), which then sees the partials of all the others.  The fence
// before the barrier publishes this CTA's partials; the winner's second fence orders its reads of the others' partials
// after its ticket.
__device__ __forceinline__ bool last_cta(unsigned* ticket, unsigned arrivals) {
  __shared__ unsigned s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = draw_ticket(ticket, arrivals) ? 1u : 0u;
  __syncthreads();
  if (s_last) __threadfence();
  return s_last != 0u;
}

// ---- shared tails ----------------------------------------------------------------------------------------------------
// stats[0..3] = mean, unbiased std (torch.std's default; n == 1 gives nan, as in torch), max, min from raw moments of n
// values.  max and min arrive as double; a float max / min converts to double and back exactly.
__device__ __forceinline__ void stats_from_moments(double s, double q, double mx, double mn, double n, float* stats) {
  const double mean = s / n;
  double var = (q - s * mean) / (n - 1.0);
  if (var < 0.0) var = 0.0;
  stats[0] = static_cast<float>(mean);
  stats[1] = static_cast<float>(sqrt(var));
  stats[2] = static_cast<float>(mx);
  stats[3] = static_cast<float>(mn);
}

// Segment k's tail of the gradient-norm reduction that feeds Adam: out[k] = the sum of the n partials part[i * stride],
// added in index order with 16 loads in flight (one L2 round trip per 16 instead of one per partial).  With step
// counts it also bumps step[k] to t and writes the bias corrections out[nseg + 2k] = 1 - beta1^t and
// out[nseg + 2k + 1] = sqrt(1 - beta2^t), in fp64 once per segment (torch computes them in Python floats).
__device__ __forceinline__ void sumsq_segment_tail(const double* part, int n, int stride, int k, int nseg, double* out,
                                                   int* step, double beta1, double beta2) {
  double t = 0.0;
  for (int i0 = 0; i0 < n; i0 += 16) {
    double v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) v[u] = (i0 + u < n) ? __ldcg(part + (i0 + u) * stride) : 0.0;
#pragma unroll
    for (int u = 0; u < 16; ++u) t += v[u];
  }
  out[k] = t;
  if (step) {
    const int st = step[k] + 1;
    step[k] = st;
    out[nseg + 2 * k] = 1.0 - pow_int(beta1, st);
    out[nseg + 2 * k + 1] = sqrt(1.0 - pow_int(beta2, st));
  }
}

// Chan et al.'s merge of a running (mean, var, count = cnt) with a batch of bn rows given by its sum s and sum of
// squares q (population variance), as the reference's update_mean_var_count does.  The caller adds bn to the count.
__device__ __forceinline__ void chan_merge(double s, double q, double bn, double cnt, double& mean, double& var) {
  const double bmean = s / bn;
  double bvar = q / bn - bmean * bmean;
  if (bvar < 0.0) bvar = 0.0;
  const double tot = cnt + bn;
  const double delta = bmean - mean;
  const double m2 = var * cnt + bvar * bn + delta * delta * cnt * bn / tot;
  mean = mean + delta * bn / tot;
  var = m2 / tot;
}

}  // namespace trl
