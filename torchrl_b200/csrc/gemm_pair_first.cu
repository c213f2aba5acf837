// gemm_pair_first.cu -- the dgrad GEMM of an MLP's second hidden layer with the first layer's backward as its epilogue
// (gemm3_wgmma_kernel with XK = obs_dim, csrc/gemm_wgmma.cuh): for an input that needs no gradient, dH1 = gz2 W2 feeds
// nothing but dW1 = (dH1 * act'(h1))^T x and db1 = colsum(dH1 * act'(h1)), so the launch writes the slab partials of
// trl_skinny_act_wgrad_partial (csrc/skinny.cu) instead of dH1: the (M x 256) dH1 is never stored nor read back.
// One instance per XK (1..24), in its own translation unit so that it builds beside csrc/gemm_pair.cu.
#include "gemm_wgmma.cuh"

// The slab partials of trl_skinny_act_wgrad_partial(gz2 W2, h1, x, M, 256, K, act, scratch), bit for bit: the dgrad
// runs on the transposed pre-split planes of W2 ((w_hi_t, w_lo_t) = (hi^T, lo^T), the K-major route of trl_gemm3_pair)
// and its epilogue sums each slab in skinny_tn_kernel's order.  scratch: trl_skinny_tn_scratch_floats(M, 256, K)
// floats, summed by trl_skinny_reduce_jobs (kind 1).  M <= 16896 (slabs of at most 64 rows), 1 <= K <= 24.
TRL_API int trl_gemm3_pair_dgrad_act_wgrad(const float* G, const float* w_hi_t, const float* w_lo_t, const float* Y,
                                           const float* X, int64_t M, int K, int act, float* scratch, void* stream) {
  using namespace trl;
  using namespace trl::wg;
  TRL_REQUIRE(M >= 1 && sk_rows_per_cta(M) <= 64, "trl_gemm3_pair_dgrad_act_wgrad: M=%lld not in [1, %d]", (long long)M,
              64 * kSkCtas);
  TRL_REQUIRE(K >= 1 && K <= 24, "trl_gemm3_pair_dgrad_act_wgrad: need 1<=K<=24 (K=%d)", K);
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_gemm3_pair_dgrad_act_wgrad: unknown activation %d", act);
  TRL_REQUIRE(G && w_hi_t && w_lo_t && Y && X && scratch, "trl_gemm3_pair_dgrad_act_wgrad: null pointer");
  TRL_REQUIRE(aligned16(G) && aligned16(w_hi_t) && aligned16(w_lo_t) && aligned16(Y) && aligned16(scratch),
              "trl_gemm3_pair_dgrad_act_wgrad: G/W/Y/scratch must be 16-byte aligned");
  CUtensorMap ma, mb, mb2, my;
  if (!make_map(&ma, G, static_cast<uint64_t>(M), kN, Box::kKMajor) || !make_map(&mb, w_hi_t, kN, kN, Box::kKMajor) ||
      !make_map(&mb2, w_lo_t, kN, kN, Box::kKMajor) || !make_map(&my, Y, static_cast<uint64_t>(M), kN, Box::kTile)) {
    set_error("trl_gemm3_pair_dgrad_act_wgrad: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  const int rows = sk_rows_per_cta(M);
  Params p{nullptr, act, nullptr, M, kN / kBK, scratch, nullptr, X, rows * (64 / rows), rows};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char* what = "gemm3_wgmma_kernel<nt,split,act_wgrad>";
#define TRL_XK(KK) \
  case KK: return launch<false, false, true, true, false, KK>(ma, mb, mb2, p, 1, st, what, &my)
  switch (K) {
    TRL_XK(1); TRL_XK(2); TRL_XK(3); TRL_XK(4); TRL_XK(5); TRL_XK(6); TRL_XK(7); TRL_XK(8);
    TRL_XK(9); TRL_XK(10); TRL_XK(11); TRL_XK(12); TRL_XK(13); TRL_XK(14); TRL_XK(15); TRL_XK(16);
    TRL_XK(17); TRL_XK(18); TRL_XK(19); TRL_XK(20); TRL_XK(21); TRL_XK(22); TRL_XK(23); TRL_XK(24);
  }
#undef TRL_XK
  return TRL_EUNSUPPORTED;
}
