// mlp_epilogue.cu -- K3/K8 support: fused bias+activation epilogue and its backward for the policy /
// value / Q MLPs (the GEMMs themselves stay in cuBLAS, as the north star allows for the small nets).
//
// Replaces, per hidden layer of MLPBase (/root/reference/torchrl/networks/base.py:24-44: Linear then
// activation), the separate PyTorch launches around the GEMM:
//   forward : cuBLASLt bias-epilogue kernel + tanh/relu elementwise kernel      -> 1 launch (in place)
//   backward: activation-backward elementwise kernel + bias-gradient reduce_kernel -> 1 launch
// ncu (profiles/launches_ppo_step_r1.md) showed these PyTorch epilogue/elementwise/reduce launches at
// ~30 % of a minibatch update; both kernels here are HBM-bound: 8 B/element forward, 12 B/element
// backward (+ H floats of bias gradient).
#include "reduce.cuh"

namespace trl {

enum { ACT_NONE = 0, ACT_TANH = 1, ACT_RELU = 2 };

__device__ __forceinline__ float act_fwd(float x, int act) {
  if (act == ACT_TANH) return tanhf(x);
  if (act == ACT_RELU) return fmaxf(x, 0.f);
  return x;
}
// derivative expressed through the OUTPUT y = act(x)
__device__ __forceinline__ float act_bwd_from_out(float y, int act) {
  if (act == ACT_TANH) return 1.f - y * y;
  if (act == ACT_RELU) return y > 0.f ? 1.f : 0.f;
  return 1.f;
}

// z (M,H) row-major, in place: z <- act(z + b).  H % 4 == 0 -> float4 path.
__global__ void __launch_bounds__(256) bias_act_fwd_kernel(float* __restrict__ z, const float* __restrict__ b,
                                                          long long M, int H, int act) {
  const long long total4 = M * H / 4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>((i * 4) % H);
    float4 v = reinterpret_cast<float4*>(z)[i];
    const float4 bb = *reinterpret_cast<const float4*>(b + c);
    v.x = act_fwd(v.x + bb.x, act); v.y = act_fwd(v.y + bb.y, act);
    v.z = act_fwd(v.z + bb.z, act); v.w = act_fwd(v.w + bb.w, act);
    reinterpret_cast<float4*>(z)[i] = v;
  }
}
__global__ void bias_act_fwd_scalar_kernel(float* __restrict__ z, const float* __restrict__ b, long long M, int H,
                                           int act) {
  const long long total = M * H;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    z[i] = act_fwd(z[i] + b[i % H], act);
}

// gz (M,H) <- g * act'(y)  (gz may alias g);  db[c] = sum_m gz[m][c].
// CTA = 256 threads = 8 row-groups x 32 column-lanes(x4 floats): covers 128 columns x ROWS_PER_CTA rows.
// Column sums: per-thread accumulation over its rows -> smem across the 8 row-groups -> per-CTA partial
// -> last CTA of each column block reduces the partials in fixed order (deterministic).
constexpr int kBwdRows = 128;   // rows per CTA (M=16384,H=256 -> 256 CTAs)

__global__ void __launch_bounds__(256) bias_act_bwd_kernel(const float* g, const float* __restrict__ y, float* gz,
                                                          float* __restrict__ db, float* __restrict__ partial,
                                                          unsigned* __restrict__ tickets, long long M, int H,
                                                          int act) {
  __shared__ float4 sh[8][32];
  const int lane = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + lane) * 4;               // first of this thread's 4 columns
  const long long row0 = static_cast<long long>(blockIdx.y) * kBwdRows;
  const bool col_ok = col < H;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col_ok) {
    const long long rend = min(row0 + kBwdRows, M);
#pragma unroll 4
    for (long long r = row0 + rg; r < rend; r += 8) {
      const long long off = r * H + col;
      float4 gv = *reinterpret_cast<const float4*>(g + off);
      const float4 yv = *reinterpret_cast<const float4*>(y + off);
      gv.x *= act_bwd_from_out(yv.x, act); gv.y *= act_bwd_from_out(yv.y, act);
      gv.z *= act_bwd_from_out(yv.z, act); gv.w *= act_bwd_from_out(yv.w, act);
      *reinterpret_cast<float4*>(gz + off) = gv;
      acc.x += gv.x; acc.y += gv.y; acc.z += gv.z; acc.w += gv.w;
    }
  }
  sh[rg][lane] = acc;
  __syncthreads();
  if (rg == 0 && col_ok) {
    float4 s = sh[0][lane];
#pragma unroll
    for (int k = 1; k < 8; ++k) { s.x += sh[k][lane].x; s.y += sh[k][lane].y; s.z += sh[k][lane].z; s.w += sh[k][lane].w; }
    *reinterpret_cast<float4*>(partial + static_cast<long long>(blockIdx.y) * H + col) = s;
  }
  if (!last_cta(&tickets[blockIdx.x], gridDim.y)) return;   // one ticket per column block
  // last CTA of this column block: all 8 row-groups share the partial rows (fixed assignment and fixed
  // combination order -> deterministic), instead of one row-group walking all of them serially
  {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (col_ok) {
#pragma unroll 4
      for (unsigned by = rg; by < gridDim.y; by += 8) {
        const float4 p = *reinterpret_cast<const float4*>(partial + static_cast<long long>(by) * H + col);
        s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
      }
    }
    __syncthreads();
    sh[rg][lane] = s;
    __syncthreads();
    if (rg == 0 && col_ok) {
      float4 t = sh[0][lane];
#pragma unroll
      for (int k = 1; k < 8; ++k) { t.x += sh[k][lane].x; t.y += sh[k][lane].y; t.z += sh[k][lane].z; t.w += sh[k][lane].w; }
      *reinterpret_cast<float4*>(db + col) = t;
    }
  }
}

}  // namespace trl

TRL_API int64_t trl_bias_act_bwd_scratch_floats(int64_t M, int H) {
  return trl::ceil_div<long long>(M, trl::kBwdRows) * H;
}

TRL_API int trl_bias_act_fwd(float* z, const float* bias, int64_t M, int H, int act, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && H >= 1, "trl_bias_act_fwd: bad sizes");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_bias_act_fwd: unknown activation %d", act);
  if (M == 0) return TRL_OK;
  TRL_REQUIRE(z && bias, "trl_bias_act_fwd: null pointer");
  const long long total = M * H;
  long long blocks = ceil_div<long long>(total / 4 + 1, 256);
  if (blocks > 8LL * kNumSM) blocks = 8LL * kNumSM;
  if (H % 4 == 0 && aligned16(z) && aligned16(bias))
    bias_act_fwd_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(z, bias, M, H, act);
  else
    bias_act_fwd_scalar_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(z, bias, M,
                                                                                                            H, act);
  return check_launch("bias_act_fwd_kernel");
}

// tickets: ceil(H/128) zero-initialised unsigned; scratch: trl_bias_act_bwd_scratch_floats(M,H) floats.
TRL_API int trl_bias_act_bwd(const float* grad, const float* out, float* grad_pre, float* dbias, int64_t M, int H,
                             int act, float* scratch, unsigned* tickets, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && H >= 4 && H % 4 == 0, "trl_bias_act_bwd: need M >= 1 and H a multiple of 4 (got %lld, %d)",
              (long long)M, H);
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_bias_act_bwd: unknown activation %d", act);
  TRL_REQUIRE(grad && out && grad_pre && dbias && scratch && tickets, "trl_bias_act_bwd: null pointer");
  TRL_REQUIRE(aligned16(grad) && aligned16(out) && aligned16(grad_pre) && aligned16(dbias) && aligned16(scratch),
              "trl_bias_act_bwd: pointers must be 16-byte aligned");
  const dim3 grid(static_cast<unsigned>(ceil_div(H, 128)), static_cast<unsigned>(ceil_div<long long>(M, kBwdRows)));
  bias_act_bwd_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(grad, out, grad_pre, dbias, scratch, tickets,
                                                                          M, H, act);
  return check_launch("bias_act_bwd_kernel");
}

// ---------------------------------------------------------------------------------------------------
// Error-compensated TF32 ("3xTF32") operand split: x = hi + lo with hi = x rounded to TF32 (10-bit
// mantissa, cvt.rna) and lo = x - hi (exact in fp32).  A fp32-faithful product on the tensor cores is
// then a_hi*b_hi + a_lo*b_hi + a_hi*b_lo (three TF32 GEMMs with fp32 accumulation; the dropped lo*lo
// term is O(2^-22) relative).  HBM-bound: 4 B read + 8 B written per element.
namespace trl {
__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi,
                                                        float* __restrict__ lo, long long n4, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 h, l;
    unsigned u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.x)); h.x = __uint_as_float(u); l.x = v.x - h.x;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.y)); h.y = __uint_as_float(u); l.y = v.y - h.y;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.z)); h.z = __uint_as_float(u); l.z = v.z - h.z;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.w)); h.w = __uint_as_float(u); l.w = v.w - h.w;
    reinterpret_cast<float4*>(hi)[i] = h;
    reinterpret_cast<float4*>(lo)[i] = l;
  }
  // tail (n not a multiple of 4)
  const long long t = n4 * 4 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t < n) {
    unsigned u;
    const float v = x[t];
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    hi[t] = __uint_as_float(u);
    lo[t] = v - __uint_as_float(u);
  }
}
__global__ void split_tf32_scalar_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo,
                                         long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    unsigned u;
    const float v = x[i];
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    hi[i] = __uint_as_float(u);
    lo[i] = v - __uint_as_float(u);
  }
}
}  // namespace trl

TRL_API int trl_split_tf32(const float* x, int64_t n, float* hi, float* lo, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 0, "trl_split_tf32: negative size");
  if (n == 0) return TRL_OK;
  TRL_REQUIRE(x && hi && lo, "trl_split_tf32: null pointer");
  if (!(aligned16(x) && aligned16(hi) && aligned16(lo))) {   // e.g. a weight view into the flat parameter buffer
    long long sb = ceil_div<long long>(n, 256);
    if (sb > 8LL * kNumSM) sb = 8LL * kNumSM;
    split_tf32_scalar_kernel<<<static_cast<unsigned>(sb), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, hi, lo, n);
    return check_launch("split_tf32_scalar_kernel");
  }
  const long long n4 = n / 4;
  long long blocks = ceil_div<long long>(n4 + 1, 256);
  if (blocks > 8LL * kNumSM) blocks = 8LL * kNumSM;
  if (blocks < 1) blocks = 1;
  split_tf32_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, hi, lo, n4, n);
  return check_launch("split_tf32_kernel");
}
