// gemm_tf32x3.cu -- entry points of the fp32-faithful 3xTF32 GEMM for the 256-wide MLP layers (K3/K8 support).
//
//   nt: C[M x 256] = act(A[M x K] . B[256 x K]^T + bias)      (A, B row-major with K contiguous = "K-major")
//   tn: C[M x 256] = A[K x M]^T . B[K x 256]                   (the weight-gradient shape, split-K)
//
// The policy / value / Q networks of the hot path are MLP(256,256)s (SURVEY.md section 8(a) K3, K8); their three big
// GEMM shapes -- forward (x W^T), dgrad (g W) and wgrad (g^T x) -- run on the tensor cores without giving up fp32
// accuracy through the warpgroup-MMA kernel of gemm_wgmma.cuh (every operand split into hi + lo, three tf32 products).
// These entry points take raw fp32 operands, apply tanh with libdevice tanhf and sum split-K slabs in a fixed order
// (splitk_reduce_kernel, deterministic); csrc/gemm_pair.cu serves the hot path with pre-split weights.
// Accuracy: the tensor core's fp32 accumulation truncates, so the error grows ~linearly with the reduction length
// accumulated by one CTA.  Callers keep K/splits <= 256 (the MLP layers here: K = 256; wgrad: 16384/64).
#include "gemm_wgmma.cuh"

namespace trl {

// C[m][n] = sum_s P[s][m][n]   (fixed order: 4 interleaved partial sums per element combined pairwise)
// CTA = 64 float4 outputs x 4 split groups; group g sums splits g, g+4, ...; groups combined through smem.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ P, float* __restrict__ C,
                                                           long long mn, int splits) {
  __shared__ float4 sh[4][64];
  const int o = threadIdx.x & 63, g = threadIdx.x >> 6;
  const long long i = (static_cast<long long>(blockIdx.x) * 64 + o) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < mn) {
#pragma unroll 4
    for (int s = g; s < splits; s += 4) {
      const float4 v = *reinterpret_cast<const float4*>(P + static_cast<long long>(s) * mn + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  sh[g][o] = acc;
  __syncthreads();
  if (g == 0 && i < mn) {
    const float4 a = sh[0][o], b = sh[1][o], c = sh[2][o], d = sh[3][o];
    *reinterpret_cast<float4*>(C + i) =
        make_float4((a.x + b.x) + (c.x + d.x), (a.y + b.y) + (c.y + d.y), (a.z + b.z) + (c.z + d.z), (a.w + b.w) + (c.w + d.w));
  }
}

// out (C x R) = in (R x C)^T, 32x32 tiles through shared memory
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, long long R, int C) {
  __shared__ float tile[32][33];
  const long long r0 = static_cast<long long>(blockIdx.y) * 32;
  const int c0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const long long r = r0 + j;
    const int c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < R && c < C) ? in[r * C + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j;
    const long long r = r0 + threadIdx.x;
    if (c < C && r < R) out[static_cast<long long>(c) * R + r] = tile[threadIdx.x][j];
  }
}

}  // namespace trl

// C (M x 256) = act(A (M x K) . B (256 x K)^T [+ bias]) with 3xTF32 tensor-core arithmetic (bias NULL: plain GEMM).
// splits > 1: K is divided into `splits` slabs; `workspace` must hold splits*M*256 floats and the slabs are
// summed into C in a fixed order.  Requirements: K % (32*splits) == 0, 16-byte aligned A/B/C, M >= 1.
TRL_API int trl_gemm_tf32x3_nt(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                               float* workspace, const float* bias, int act, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && K >= wg::kBK && splits >= 1, "trl_gemm_tf32x3_nt: bad sizes M=%lld K=%lld splits=%d", (long long)M,
              (long long)K, splits);
  TRL_REQUIRE(K % (static_cast<int64_t>(wg::kBK) * splits) == 0, "trl_gemm_tf32x3_nt: K=%lld must be a multiple of 32*splits",
              (long long)K);
  TRL_REQUIRE(A && B && C && (splits == 1 || workspace), "trl_gemm_tf32x3_nt: null pointer");
  TRL_REQUIRE(aligned16(A) && aligned16(B) && aligned16(C) && aligned16(workspace) && aligned16(bias),
              "trl_gemm_tf32x3_nt: pointers must be 16-byte aligned");
  TRL_REQUIRE(!(bias && splits > 1), "trl_gemm_tf32x3_nt: the bias/activation epilogue needs splits == 1");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_gemm_tf32x3_nt: unknown activation %d", act);
  using namespace trl::wg;
  CUtensorMap map_a, map_b;
  if (!make_map(&map_a, A, static_cast<uint64_t>(M), static_cast<uint64_t>(K), Box::kKMajor) ||
      !make_map(&map_b, B, static_cast<uint64_t>(kN), static_cast<uint64_t>(K), Box::kKMajor)) {
    set_error("trl_gemm_tf32x3_nt: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  Params p{bias, act, splits > 1 ? workspace : C, M, static_cast<int>(K / kBK / splits)};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = launch<false, false, false, false>(map_a, map_b, map_b, p, static_cast<unsigned>(splits), st,
                                              "gemm3_wgmma_kernel<nt>");
  if (rc != TRL_OK || splits == 1) return rc;
  const long long mn = M * kN;
  splitk_reduce_kernel<<<static_cast<unsigned>(ceil_div<long long>(mn / 4, 64)), 256, 0, st>>>(workspace, C, mn, splits);
  return check_launch("splitk_reduce_kernel");
}

// C (M x 256) = A (K x M)^T . B (K x 256): both operands with the reduction index as the ROW index (the
// weight-gradient shape dW = g^T x).  M % 128 == 0, K % (32*splits) == 0, split-K as above.
TRL_API int trl_gemm_tf32x3_tn(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                               float* workspace, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= wg::kBM && M % wg::kBM == 0 && K >= wg::kBK && splits >= 1, "trl_gemm_tf32x3_tn: bad sizes M=%lld K=%lld splits=%d",
              (long long)M, (long long)K, splits);
  TRL_REQUIRE(K % (static_cast<int64_t>(wg::kBK) * splits) == 0, "trl_gemm_tf32x3_tn: K=%lld must be a multiple of 32*splits",
              (long long)K);
  TRL_REQUIRE(A && B && C && (splits == 1 || workspace), "trl_gemm_tf32x3_tn: null pointer");
  TRL_REQUIRE(aligned16(A) && aligned16(B) && aligned16(C) && aligned16(workspace),
              "trl_gemm_tf32x3_tn: pointers must be 16-byte aligned");
  using namespace trl::wg;
  CUtensorMap map_a, map_b;
  // (K rows) x (M | 256 contiguous) matrices, consumed M/N-major
  if (!make_map(&map_a, A, static_cast<uint64_t>(K), static_cast<uint64_t>(M), Box::kMNMajorA) ||
      !make_map(&map_b, B, static_cast<uint64_t>(K), static_cast<uint64_t>(kN), Box::kMNMajor)) {
    set_error("trl_gemm_tf32x3_tn: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  Params p{nullptr, 0, splits > 1 ? workspace : C, M, static_cast<int>(K / kBK / splits)};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = launch<true, true, false, false>(map_a, map_b, map_b, p, static_cast<unsigned>(splits), st,
                                            "gemm3_wgmma_kernel<tn>");
  if (rc != TRL_OK || splits == 1) return rc;
  const long long mn = M * kN;
  splitk_reduce_kernel<<<static_cast<unsigned>(ceil_div<long long>(mn / 4, 64)), 256, 0, st>>>(workspace, C, mn, splits);
  return check_launch("splitk_reduce_kernel");
}

TRL_API int trl_transpose_f32(const float* in, float* out, int64_t rows, int cols, void* stream) {
  using namespace trl;
  TRL_REQUIRE(rows >= 1 && cols >= 1, "trl_transpose_f32: bad sizes");
  TRL_REQUIRE(in && out, "trl_transpose_f32: null pointer");
  // the row tiles run on grid.y (at most 65535 blocks)
  TRL_REQUIRE(ceil_div<long long>(rows, 32) <= 65535LL,
              "trl_transpose_f32: bad sizes rows=%lld (at most 65535 * 32 rows)", (long long)rows);
  const dim3 grid(static_cast<unsigned>(ceil_div(cols, 32)), static_cast<unsigned>(ceil_div<long long>(rows, 32)));
  transpose_kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(in, out, rows, cols);
  return check_launch("transpose_kernel");
}
