// skinny_common.cuh -- the slab geometry and the per-row arithmetic of the first-layer weight gradient
//   dW1 (H x K) = (G * act'(Y))^T X,   db1 (H) = colsum(G * act'(Y))
// shared by skinny_tn_kernel<K, true> (csrc/skinny.cu, G read from memory) and the dgrad GEMM whose epilogue forms the
// same slab partials (gemm3_wgmma_kernel with XK > 0, csrc/gemm_wgmma.cuh).  Both run these functions in the same order
// on the same values, so their partials are bit-identical: nvcc contracts a * b + c where it can (-fmad), and one copy
// of the code is what keeps the two contractions the same.
#pragma once
#include "common.cuh"

namespace trl {

constexpr int kSkMaxRows = 128;      // rows of the skinny operand staged per CTA (<= 12 KB of shared memory)
constexpr int kSkCtas = 2 * kNumSM;  // target grid: two resident CTAs per SM

// rows per slab (one CTA of the skinny kernels): this fixes the summation order of every slab partial
static inline int sk_rows_per_cta(long long M) {
  long long r = ceil_div<long long>(M, kSkCtas);
  if (r < 8) r = 8;
  if (r > kSkMaxRows) r = kSkMaxRows;
  return static_cast<int>(r);
}

// g * act'(.) with the derivative expressed through the activation's OUTPUT y (same convention as mlp_epilogue.cu)
__device__ __forceinline__ float4 sk_dact4(float4 g, float4 y, int act) {
  if (act == 1)
    return make_float4(g.x * fmaf(-y.x, y.x, 1.f), g.y * fmaf(-y.y, y.y, 1.f), g.z * fmaf(-y.z, y.z, 1.f),
                       g.w * fmaf(-y.w, y.w, 1.f));
  if (act == 2) return make_float4(y.x > 0.f ? g.x : 0.f, y.y > 0.f ? g.y : 0.f, y.z > 0.f ? g.z : 0.f, y.w > 0.f ? g.w : 0.f);
  return g;
}

// stage rows [row0, row0+nrows) of a row-major (M x K) matrix into shared memory as [nrows][KP], zero padded.  The slab
// is one contiguous run of nrows*K floats: it is read as such (fully coalesced); K is a compile-time constant, so the
// (row, column) split is a multiply-shift, not a division.
template <int K>
__device__ __forceinline__ void stage_rows(float* __restrict__ dst, const float* __restrict__ src, long long row0,
                                           int nrows, int tid, int nthr) {
  constexpr int KP = (K + 3) & ~3;
  const float* base = src + row0 * K;
  for (int j = tid; j < nrows * K; j += nthr) {
    const int r = j / K, k = j - r * K;
    dst[r * KP + k] = __ldg(base + j);
  }
  if (KP != K) {
    constexpr int PAD = KP - K > 0 ? KP - K : 1;
    for (int j = tid; j < nrows * PAD; j += nthr) {
      const int r = j / PAD, k = K + (j - r * PAD);
      dst[r * KP + k] = 0.f;
    }
  }
}

// acc[k][j] += a_j * brow[k] for the K real columns of a staged row (KP/4 broadcast LDS.128; the padding is never
// multiplied)
template <int K>
__device__ __forceinline__ void tn_fma_row(float (&acc)[(K + 3) & ~3][4], const float4 a, const float* __restrict__ brow) {
  constexpr int KP = (K + 3) & ~3;
  const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int q = 0; q < KP / 4; ++q) {
    const float4 b = reinterpret_cast<const float4*>(brow)[q];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (4 * q < K) acc[4 * q][j] = fmaf(av[j], b.x, acc[4 * q][j]);
      if (4 * q + 1 < K) acc[4 * q + 1][j] = fmaf(av[j], b.y, acc[4 * q + 1][j]);
      if (4 * q + 2 < K) acc[4 * q + 2][j] = fmaf(av[j], b.z, acc[4 * q + 2][j]);
      if (4 * q + 3 < K) acc[4 * q + 3][j] = fmaf(av[j], b.w, acc[4 * q + 3][j]);
    }
  }
}

// one row of the first-layer backward: gz = g * act'(y) (four columns), its column sums, and gz^T x into acc
template <int K>
__device__ __forceinline__ void act_wgrad_row(float (&acc)[(K + 3) & ~3][4], float4& asum, const float4 g, const float4 y,
                                              const float* __restrict__ xrow, int act) {
  const float4 a0 = sk_dact4(g, y, act);
  asum.x += a0.x; asum.y += a0.y; asum.z += a0.z; asum.w += a0.w;
  tn_fma_row<K>(acc, a0, xrow);
}

// The row-lane layout of a slab: a warp owns 32 columns, lane = (row lane rl = lane >> 3) x (column quad lane & 7);
// row lane rl runs the slab's rows rl, rl + 4, ... in increasing order.  tn_combine_lanes adds the 4 row lanes (lanes
// l, l^8, l^16, l^24 hold the same columns) in a fixed order; every lane ends with the sum.
__device__ __forceinline__ float tn_lane_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}
template <int K>
__device__ __forceinline__ void tn_combine_lanes(float (&acc)[(K + 3) & ~3][4]) {
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[k][j] = tn_lane_sum(acc[k][j]);
}
// the slab partial, k-major [K + 1][H]: row lane (k & 3) stores column quad k of acc, row K the column sums
template <int K>
__device__ __forceinline__ void tn_store_rows(float* __restrict__ pp, const float (&acc)[(K + 3) & ~3][4], int H, int c0,
                                              int rl) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if ((k & 3) == rl)
      *reinterpret_cast<float4*>(pp + static_cast<long long>(k) * H + c0) = make_float4(acc[k][0], acc[k][1], acc[k][2], acc[k][3]);
  }
}
template <int K>
__device__ __forceinline__ void act_wgrad_store(float* __restrict__ pp, float (&acc)[(K + 3) & ~3][4], float4 asum, int H,
                                                int c0, int rl) {
  tn_combine_lanes<K>(acc);
  tn_store_rows<K>(pp, acc, H, c0, rl);
  asum.x = tn_lane_sum(asum.x); asum.y = tn_lane_sum(asum.y); asum.z = tn_lane_sum(asum.z); asum.w = tn_lane_sum(asum.w);
  if (rl == (K & 3)) *reinterpret_cast<float4*>(pp + static_cast<long long>(K) * H + c0) = asum;
}

}  // namespace trl
