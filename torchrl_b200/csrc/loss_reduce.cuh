// loss_reduce.cuh -- block-level reductions shared by the fused loss kernels (ppo_loss.cu, categorical.cu).
// Both kernels reduce per-CTA partials that the last CTA to finish folds in a fixed order, so their results are
// deterministic; these helpers are the first level of that scheme (block_reduce_*: one quantity, two barriers;
// block_partials: several quantities, one barrier).
#pragma once
#include "common.cuh"

namespace trl {

__device__ __forceinline__ double block_reduce_sum(double v, double* sh) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
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

}  // namespace trl
