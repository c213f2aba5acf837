// gemm_pair.cu -- the hot path's fp32-faithful (3xTF32) tensor-core GEMMs for the 256-wide MLP layers (SURVEY.md
// section 8(a) K3/K8: the Linear layers in the rollout, the cached old-log-prob pass and the PPO / SAC minibatch
// update), on the warpgroup-MMA kernel of gemm_wgmma.cuh.  Unlike the csrc/gemm_tf32x3.cu entry points:
//   * B can arrive PRE-SPLIT (b_lo != NULL): the weights are split into hi = tf32(w), lo = w - hi once per optimizer
//     step (csrc/optim.cu writes both planes), TMA loads both planes and only the activation operand A is split;
//   * B may be N-major (b_nmajor): the dgrad shape dX = G . W reads W (K x 256, row-major) directly -- no per-
//     minibatch transpose of the weights;
//   * tanh = 1 - 2/(exp(2x)+1) on the MUFU unit (abs err < 2.5e-7, same as csrc/skinny.cu);
//   * split-K slabs are summed by an 8-way balanced tree (pair_splitk_reduce_kernel), or, in the same order, inside
//     the GEMM launch through thread-block clusters (trl_gemm3_pair_tn_cluster, the weight gradient's hot path).
// Shapes:
//   nt   : A (M x K) row-major, B (256 x K) row-major      forward  y = act(x W^T + b)
//   nn   : A (M x K) row-major, B (K x 256) row-major      dgrad    dX = G W
//   tn   : A (K x M) row-major, B (K x 256) row-major      wgrad    dW = G^T X (split-K, deterministic reduce)
#include "gemm_wgmma.cuh"

namespace trl {
namespace pair {

// C[i] = sum_s P[s][i]   (fixed order: 8 interleaved partial sums per element, combined as a balanced tree).  512
// threads = 64 float4 elements x 8 groups; a group's loads are independent, eight of them in flight.
__global__ void __launch_bounds__(512) pair_splitk_reduce_kernel(const float* __restrict__ P, float* __restrict__ C,
                                                                long long mn, int splits) {
  __shared__ float4 sh[8][64];
  const int o = threadIdx.x & 63, g = threadIdx.x >> 6;
  const long long i = (static_cast<long long>(blockIdx.x) * 64 + o) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < mn) {
    const float* pi = P + i;
    for (int s0 = g; s0 < splits; s0 += 64) {
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        v[u] = (s0 + 8 * u < splits) ? __ldcg(reinterpret_cast<const float4*>(pi + static_cast<long long>(s0 + 8 * u) * mn))
                                     : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 8; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
    }
  }
  sh[g][o] = acc;
  __syncthreads();
  if (g == 0 && i < mn) {
    float4 t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) t[u] = sh[u][o];
#define TRL_T3(c) (((t[0].c + t[1].c) + (t[2].c + t[3].c)) + ((t[4].c + t[5].c) + (t[6].c + t[7].c)))
    *reinterpret_cast<float4*>(C + i) = make_float4(TRL_T3(x), TRL_T3(y), TRL_T3(z), TRL_T3(w));
#undef TRL_T3
  }
}

}  // namespace pair
}  // namespace trl

// C (M x 256) = act(A (M x K) . B + bias) on the tensor cores.  B is the (256 x K) row-major matrix (b_nmajor == 0: C = A B^T,
// the Linear forward) or the (K x 256) row-major matrix (b_nmajor != 0: C = A B, the dgrad shape).  b_lo == NULL: b_hi is
// the raw fp32 matrix and is split in shared memory; b_lo != NULL: (b_hi, b_lo) are the pre-split planes of
// trl_split_tf32 / trl_adam_step.  K % 32 == 0, 16-byte aligned pointers, any M >= 1 (ragged tail rows are masked).
TRL_API int trl_gemm3_pair(const float* A, const float* b_hi, const float* b_lo, float* C, int64_t M, int64_t K,
                           int b_nmajor, const float* bias, int act, void* stream) {
  using namespace trl;
  using namespace trl::wg;
  TRL_REQUIRE(M >= 1 && K >= kBK && K % kBK == 0, "trl_gemm3_pair: bad sizes M=%lld K=%lld (K must be a multiple of 32)",
              (long long)M, (long long)K);
  TRL_REQUIRE(A && b_hi && C, "trl_gemm3_pair: null pointer");
  TRL_REQUIRE(aligned16(A) && aligned16(b_hi) && aligned16(b_lo) && aligned16(C) && aligned16(bias),
              "trl_gemm3_pair: pointers must be 16-byte aligned");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_gemm3_pair: unknown activation %d", act);
  CUtensorMap ma, mb, mb2;
  const uint64_t b_rows = b_nmajor ? static_cast<uint64_t>(K) : kN, b_cols = b_nmajor ? kN : static_cast<uint64_t>(K);
  const Box b_box = b_nmajor ? Box::kMNMajor : Box::kKMajor;
  if (!make_map(&ma, A, static_cast<uint64_t>(M), static_cast<uint64_t>(K), Box::kKMajor) ||
      !make_map(&mb, b_hi, b_rows, b_cols, b_box) || !make_map(&mb2, b_lo ? b_lo : b_hi, b_rows, b_cols, b_box)) {
    set_error("trl_gemm3_pair: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  Params p{bias, act, C, M, static_cast<int>(K / kBK)};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (b_nmajor) {
    if (b_lo) return launch<false, true, true, true>(ma, mb, mb2, p, 1, st, "gemm3_wgmma_kernel<nn,split>");
    return launch<false, true, false, true>(ma, mb, mb2, p, 1, st, "gemm3_wgmma_kernel<nn>");
  }
  if (b_lo) return launch<false, false, true, true>(ma, mb, mb2, p, 1, st, "gemm3_wgmma_kernel<nt,split>");
  return launch<false, false, false, true>(ma, mb, mb2, p, 1, st, "gemm3_wgmma_kernel<nt>");
}

// C (M x 256) = A (K x M)^T . B (K x 256): the weight-gradient shape dW = g^T x, both operands consumed M/N-major
// from their row-major storage.  M % 256 == 0, K % (32 * splits) == 0; splits > 1: `workspace` holds splits*M*256
// floats and the slabs are summed into C in a fixed order (deterministic).
TRL_API int trl_gemm3_pair_tn(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                              float* workspace, void* stream) {
  using namespace trl;
  using namespace trl::wg;
  TRL_REQUIRE(M >= kN && M % kN == 0 && K >= kBK && splits >= 1,
              "trl_gemm3_pair_tn: bad sizes M=%lld K=%lld splits=%d (M must be a multiple of 256)", (long long)M,
              (long long)K, splits);
  TRL_REQUIRE(K % (static_cast<int64_t>(kBK) * splits) == 0, "trl_gemm3_pair_tn: K=%lld must be a multiple of 32*splits",
              (long long)K);
  TRL_REQUIRE(A && B && C && (splits == 1 || workspace), "trl_gemm3_pair_tn: null pointer");
  TRL_REQUIRE(aligned16(A) && aligned16(B) && aligned16(C) && aligned16(workspace),
              "trl_gemm3_pair_tn: pointers must be 16-byte aligned");
  CUtensorMap ma, mb;
  if (!make_map(&ma, A, static_cast<uint64_t>(K), static_cast<uint64_t>(M), Box::kMNMajorA) ||
      !make_map(&mb, B, static_cast<uint64_t>(K), static_cast<uint64_t>(kN), Box::kMNMajor)) {
    set_error("trl_gemm3_pair_tn: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  Params p{nullptr, 0, splits > 1 ? workspace : C, M, static_cast<int>(K / kBK / splits)};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = launch<true, true, false, true>(ma, mb, mb, p, static_cast<unsigned>(splits), st, "gemm3_wgmma_kernel<tn>");
  if (rc != TRL_OK || splits == 1) return rc;
  const long long mn = M * kN;
  pair::pair_splitk_reduce_kernel<<<static_cast<unsigned>(ceil_div<long long>(mn / 4, 64)), 512, 0, st>>>(workspace, C, mn, splits);
  return check_launch("pair_splitk_reduce_kernel");
}

// trl_gemm3_pair_tn with the split-K sum inside the one launch, bit for bit the same C: clusters of splits / 8 CTAs
// add their slabs through distributed shared memory into 8 group partials, and the last CTA of each tile slice adds
// those in pair_splitk_reduce_kernel's order.  8 <= splits <= 64, splits % 8 == 0; `workspace` holds 8*M*256 floats,
// `tickets` M/8 int32 that are zero on entry and are left zero (one set per stream: concurrent calls must not share).
TRL_API int trl_gemm3_pair_tn_cluster(const float* A, const float* B, float* C, int64_t M, int64_t K, int splits,
                                      float* workspace, int* tickets, void* stream) {
  using namespace trl;
  using namespace trl::wg;
  TRL_REQUIRE(M >= kN && M % kN == 0 && K >= kBK, "trl_gemm3_pair_tn_cluster: bad sizes M=%lld K=%lld (M must be a multiple of 256)",
              (long long)M, (long long)K);
  TRL_REQUIRE(splits >= 8 && splits <= 64 && splits % 8 == 0,
              "trl_gemm3_pair_tn_cluster: splits=%d must be a multiple of 8 in [8, 64]", splits);
  TRL_REQUIRE(K % (static_cast<int64_t>(kBK) * splits) == 0,
              "trl_gemm3_pair_tn_cluster: K=%lld must be a multiple of 32*splits", (long long)K);
  TRL_REQUIRE(A && B && C && workspace && tickets, "trl_gemm3_pair_tn_cluster: null pointer");
  TRL_REQUIRE(aligned16(A) && aligned16(B) && aligned16(C) && aligned16(workspace),
              "trl_gemm3_pair_tn_cluster: pointers must be 16-byte aligned");
  CUtensorMap ma, mb;
  if (!make_map(&ma, A, static_cast<uint64_t>(K), static_cast<uint64_t>(M), Box::kMNMajorA) ||
      !make_map(&mb, B, static_cast<uint64_t>(K), static_cast<uint64_t>(kN), Box::kMNMajor)) {
    set_error("trl_gemm3_pair_tn_cluster: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  Params p{nullptr, 0, C, M, static_cast<int>(K / kBK / splits), workspace, reinterpret_cast<unsigned*>(tickets)};
  return launch<true, true, false, true, true>(ma, mb, mb, p, static_cast<unsigned>(splits),
                                               static_cast<cudaStream_t>(stream), "gemm3_wgmma_kernel<tn,cluster>");
}
