// common.cuh -- shared helpers for the torchrl_b200 sm_90a kernels.
//
// Conventions of every entry point in this library (see include/torchrl_b200.h):
//   * plain device pointers + sizes, no torch types; the caller owns all memory;
//   * asynchronous launch on the cudaStream_t passed as `void* stream` (never syncs);
//   * returns 0 on success, a negative TRL_E* code on argument errors, or the
//     positive cudaError_t of a failed launch; trl_last_error() gives the text.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// The public declarations (and the TRL_E* codes): a definition that disagrees with its declaration does not compile.
#include "../../include/torchrl_b200.h"

#define TRL_API extern "C" __attribute__((visibility("default")))

namespace trl {

constexpr int kNumSM = 132;  // H100 SXM

// thread-local last-error text (host side)
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define TRL_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      ::trl::set_error(__VA_ARGS__);      \
      return TRL_EINVAL;                  \
    }                                     \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
inline bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

template <typename T>
__host__ __device__ constexpr T ceil_div(T a, T b) { return (a + b - 1) / b; }

// ---- streaming (touch-once) global accesses: keep them out of L1 ------------------
__device__ __forceinline__ float ld_stream(const float* p) { return __ldcs(p); }
__device__ __forceinline__ float4 ld_stream(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ unsigned ld_stream(const unsigned* p) { return __ldcs(p); }
__device__ __forceinline__ unsigned char ld_stream(const unsigned char* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(float* p, float v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream(float4* p, float4 v) { __stcs(p, v); }

// ---- tanh on the MUFU pipe -----------------------------------------------------------
// tanh(x) = 1 - 2 / (exp(2x) + 1) as FMUL, MUFU.EX2, FADD, MUFU.RCP, FFMA (5 instructions; libdevice tanhf is ~25 with
// a branch).  ex2.approx is good to 2^-22 relative and rcp.approx to 1 ulp, so |abs err| < 2.5e-7 (2.31e-7 measured on
// an H100 over 2^20 points in [-20, 20]): a few ulp of the activations.  Saturation needs no clamp: exp -> +inf gives
// rcp -> +0 -> 1, exp -> 0 gives 1 - 2 = -1.
__device__ __forceinline__ float tanh_ex2(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.8853900817779268f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.f));
  return fmaf(-2.f, r, 1.f);
}

// b^n for a small positive integer n by repeated squaring (<= 2*log2(n) fp64 multiplies, a few ulp of double):
// Adam's bias corrections 1 - beta^t.  libdevice pow(double, double) is several hundred dependent fp64 instructions,
// which on one thread is microseconds -- on the serial tail of every optimizer step.
__device__ __forceinline__ double pow_int(double b, int n) {
  double r = 1.0;
  while (n > 0) {
    if (n & 1) r *= b;
    b *= b;
    n >>= 1;
  }
  return r;
}

// ---- warp reductions (block level and across CTAs: reduce.cuh) --------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// float atomic max/min via CAS-free integer trick (valid for non-NaN values)
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  if (v >= 0.f)
    atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else
    atomicMin(reinterpret_cast<unsigned*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
  if (v >= 0.f)
    atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v));
  else
    atomicMax(reinterpret_cast<unsigned*>(addr), __float_as_uint(v));
}

// ---- counter-based RNG: Philox4x32-10 (device "performance mode" noise/indices) ----
struct Philox {
  static __host__ __device__ __forceinline__ void round(uint32_t (&c)[4], uint32_t (&k)[2]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#ifdef __CUDA_ARCH__
    const uint32_t hi0 = __umulhi(M0, c[0]), hi1 = __umulhi(M1, c[2]);
#else
    const uint32_t hi0 = uint32_t((uint64_t(M0) * c[0]) >> 32), hi1 = uint32_t((uint64_t(M1) * c[2]) >> 32);
#endif
    const uint32_t lo0 = M0 * c[0], lo1 = M1 * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k[0], n1 = lo1, n2 = hi0 ^ c[3] ^ k[1], n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  }
  // 4 x uint32 for (key = seed, counter = (ctr_lo, ctr_hi, stream, 0))
  static __host__ __device__ __forceinline__ void gen(uint64_t seed, uint64_t ctr, uint32_t stream, uint32_t (&out)[4]) {
    uint32_t c[4] = {uint32_t(ctr), uint32_t(ctr >> 32), stream, 0u};
    uint32_t k[2] = {uint32_t(seed), uint32_t(seed >> 32)};
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      round(c, k);
      k[0] += 0x9E3779B9u;
      k[1] += 0xBB67AE85u;
    }
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
  }
};

// uint32 -> uniform in (0,1]
__device__ __forceinline__ float u32_to_unit(uint32_t x) { return (float(x >> 8) + 1.0f) * (1.0f / 16777216.0f); }

// Box-Muller: two uint32 -> two N(0,1)
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float u1 = u32_to_unit(a), u2 = u32_to_unit(b);
  const float r = sqrtf(-2.0f * logf(u1));
  float s, c;
  sincospif(2.0f * u2, &s, &c);
  z0 = r * c;
  z1 = r * s;
}

}  // namespace trl
