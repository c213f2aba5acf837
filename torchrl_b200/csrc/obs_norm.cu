// obs_norm.cu -- K2: running mean/var observation normalisation (merge + filter halves).
//
// Replaces /root/reference/torchrl/env/base_wrapper.py
//   update_mean_var_count  :44-60   Chan parallel merge of (mean, var, count) with batch moments
//   Normalizer.update_estimate :75-82   batch mean / population variance over the N rows
//   Normalizer.filt        :91-94   clip((x - mean) / (sqrt(var) + 1e-4), -clip, clip)
//   NormObs.observation    :118-121 update THEN filter the same batch (training mode)
// State stays fp64 on the device (2*o+1 doubles) exactly like the reference's NumPy state:
// fp32 `count` would lose integer precision after 2^24 samples.  The batch moments are
// produced by synth_env_step_kernel (per-CTA partials -> last CTA); trl_obs_norm_moments
// computes them for an arbitrary (N,o) batch (host-env bridge / tests), trl_obs_norm_merge
// is the stand-alone merge used when the batch sums were first all-reduced across GPUs.  Both
// merges are reduce.cuh's chan_merge.
#include "reduce.cuh"

namespace trl {

// sums[j] = sum_n x[n][j], sums[o+j] = sum_n x[n][j]^2  (fp64).  One CTA per feature column block.
__global__ void obs_moments_kernel(const float* __restrict__ x, long long N, int o, double* __restrict__ sums) {
  __shared__ double sh[2][32];
  const int j = blockIdx.x;
  double s = 0.0, q = 0.0;
  for (long long n = threadIdx.x; n < N; n += blockDim.x) {
    const double v = static_cast<double>(x[n * o + j]);
    s += v;
    q += v * v;
  }
  s = warp_sum(s);
  q = warp_sum(q);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { sh[0][wid] = s; sh[1][wid] = q; }
  __syncthreads();
  if (wid == 0) {
    const int nw = blockDim.x >> 5;
    s = lane < nw ? sh[0][lane] : 0.0;
    q = lane < nw ? sh[1][lane] : 0.0;
    s = warp_sum(s);
    q = warp_sum(q);
    if (lane == 0) { sums[j] = s; sums[o + j] = q; }
  }
}

__global__ void obs_merge_kernel(const double* __restrict__ sums, double batch_n, int o, double* __restrict__ mean,
                                 double* __restrict__ var, double* __restrict__ count) {
  const int j = threadIdx.x;
  const double cnt = *count;
  __syncthreads();
  if (j < o) chan_merge(sums[j], sums[o + j], batch_n, cnt, mean[j], var[j]);
  if (j == 0) *count = cnt + batch_n;
}

__global__ void obs_filt_kernel(const float* __restrict__ raw, const double* __restrict__ mean,
                                const double* __restrict__ var, long long total, int o, double clip,
                                float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int j = static_cast<int>(i % o);
  double y = (static_cast<double>(raw[i]) - mean[j]) / (sqrt(var[j]) + 1e-4);
  y = fmin(fmax(y, -clip), clip);
  out[i] = static_cast<float>(y);
}

}  // namespace trl

TRL_API int trl_obs_norm_moments(const float* x, int64_t N, int obs_dim, double* sums, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && obs_dim >= 1, "trl_obs_norm_moments: bad sizes");
  TRL_REQUIRE(x && sums, "trl_obs_norm_moments: null pointer");
  obs_moments_kernel<<<obs_dim, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, N, obs_dim, sums);
  return check_launch("obs_moments_kernel");
}

TRL_API int trl_obs_norm_merge(const double* sums, double batch_n, int obs_dim, double* mean, double* var,
                               double* count, void* stream) {
  using namespace trl;
  TRL_REQUIRE(obs_dim >= 1 && obs_dim <= 1024, "trl_obs_norm_merge: obs_dim %d not in 1..1024", obs_dim);
  TRL_REQUIRE(batch_n > 0, "trl_obs_norm_merge: empty batch");
  TRL_REQUIRE(sums && mean && var && count, "trl_obs_norm_merge: null pointer");
  const int threads = ((obs_dim + 31) / 32) * 32;
  obs_merge_kernel<<<1, threads, 0, static_cast<cudaStream_t>(stream)>>>(sums, batch_n, obs_dim, mean, var, count);
  return check_launch("obs_merge_kernel");
}

TRL_API int trl_obs_norm_filt(const float* raw, const double* mean, const double* var, int64_t N, int obs_dim,
                              double clip, float* out, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0 && obs_dim >= 1, "trl_obs_norm_filt: bad sizes");
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(raw && mean && var && out, "trl_obs_norm_filt: null pointer");
  const long long total = N * obs_dim;
  obs_filt_kernel<<<static_cast<unsigned>(ceil_div<long long>(total, 256)), 256, 0,
                    static_cast<cudaStream_t>(stream)>>>(raw, mean, var, total, obs_dim, clip, out);
  return check_launch("obs_filt_kernel");
}
