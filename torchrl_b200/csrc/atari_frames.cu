// atari_frames.cu -- the per-frame arithmetic of the reference's Atari chain (wrap_deepmind,
// /root/reference/torchrl/env/get_env.py:8-22) for frames stepped by host envs (env/atari_host.py):
//   trl_atari_warp_stack : WarpFrame (atari_wrapper.py:112-131: cv2.cvtColor RGB2GRAY, then cv2.resize INTER_AREA to
//                          84x84) and FrameStack.reset / FrameStack.step (atari_wrapper.py:134-168) in one launch;
//   trl_u8_lut_f32       : a 256-entry byte -> float32 map at the network input (ScaledFloatFrame, :171-180, or the
//                          plain widening when the chain does not scale).
// Both are bit-exact against OpenCV by construction (defined in oracle/atari_frames.py):
//   * gray = (9798 R + 19235 G + 3735 B + 16384) >> 15, OpenCV's 15-bit fixed-point RGB2GRAY for 8-bit images;
//   * INTER_AREA at a non-integer scale is OpenCV's resizeArea: per source row, buf[dx] += src[sx] * alpha over the
//     x table in table order; per output row sum = beta * buf for the first source row, sum += beta * buf for the
//     rest; then round half to even and saturate.  Every product and sum is rounded separately (__fmul_rn /
//     __fadd_rn: nvcc may not contract them to FMA) in OpenCV's order.  The tables (source index, fp32 weight) are
//     computeResizeAreaTab's, built once on the host (env/atari_host.py area_tables).
// One CTA per frame: the gray frame is staged in shared memory from 16-byte loads (48 bytes = 16 pixels per thread
// and step; 3W % 16 == 0 keeps every group inside the frame's 16-byte aligned rows), the 7,056 outputs are computed
// from the tables into shared memory, then the env's C-frame stack is shifted by one frame and the new frame
// appended (or, for a fresh env, the new frame fills all C slots) with 16-byte stores.
#include "common.cuh"

namespace trl {

constexpr int kWarpOut = 84;                       // WarpFrame's width and height
constexpr int kWarpFrame = kWarpOut * kWarpOut;    // 7056 bytes = 441 x 16
constexpr int kWarpThreads = 256;
constexpr int kWarpMaxSmem = 227 * 1024;           // sm_90 opt-in limit of dynamic shared memory per CTA

struct WarpStackParams {
  const uint8_t* __restrict__ frames;   // (M, H, W, 3) RGB
  const int* __restrict__ env_idx;      // (M) env of frame m, or nullptr: frame m is env m
  const uint8_t* __restrict__ fresh;    // (N) nonzero: a new episode (fill all C slots), or nullptr: every env fresh
  uint8_t* __restrict__ stack;          // (N, C, 84, 84) in place
  const int* __restrict__ tab_i;        // [xofs 85 | yofs 85 | xsrc nx | ysrc ny]
  const float* __restrict__ tab_w;      // [xw nx | yw ny]
  long long N;
  int H, W, C;
};

__device__ __forceinline__ uint32_t gray4(const uint32_t (&w)[12], int i0) {
  uint32_t out = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int b = 3 * (i0 + k);
    const uint32_t r = (w[b >> 2] >> (8 * (b & 3))) & 0xffu;
    const uint32_t g = (w[(b + 1) >> 2] >> (8 * ((b + 1) & 3))) & 0xffu;
    const uint32_t bl = (w[(b + 2) >> 2] >> (8 * ((b + 2) & 3))) & 0xffu;
    out |= ((9798u * r + 19235u * g + 3735u * bl + 16384u) >> 15) << (8 * k);
  }
  return out;
}

__global__ void __launch_bounds__(kWarpThreads) atari_warp_stack_kernel(const WarpStackParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  const long long m = blockIdx.x;
  const long long n = p.env_idx ? p.env_idx[m] : m;
  if (n < 0 || n >= p.N) return;
  const int HW = p.H * p.W;
  uint8_t* gray = smem;
  uint8_t* out = smem + HW;                         // HW % 16 == 0
  // ---- RGB -> gray, 16 pixels (three 16-byte loads) per thread and step
  const uint4* src = reinterpret_cast<const uint4*>(p.frames + m * 3LL * HW);
  for (int g = threadIdx.x; g < HW / 16; g += blockDim.x) {
    uint32_t w[12];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const uint4 v = __ldcs(src + 3 * g + q);
      w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
    }
    reinterpret_cast<uint4*>(gray)[g] = make_uint4(gray4(w, 0), gray4(w, 4), gray4(w, 8), gray4(w, 12));
  }
  __syncthreads();
  // ---- resizeArea to 84x84 from the tables, in OpenCV's order of operations
  const int* xofs = p.tab_i;
  const int* yofs = p.tab_i + kWarpOut + 1;
  const int* xsrc = p.tab_i + 2 * (kWarpOut + 1);
  const int nx = xofs[kWarpOut];
  const int* ysrc = xsrc + nx;
  const float* xw = p.tab_w;
  const float* yw = p.tab_w + nx;
  for (int o = threadIdx.x; o < kWarpFrame; o += blockDim.x) {
    const int dy = o / kWarpOut, dx = o - dy * kWarpOut;
    const int x0 = xofs[dx], x1 = xofs[dx + 1], y0 = yofs[dy], y1 = yofs[dy + 1];
    float sum = 0.f;
    for (int k = y0; k < y1; ++k) {
      const uint8_t* row = gray + ysrc[k] * p.W;
      float buf = 0.f;
      for (int j = x0; j < x1; ++j) buf = __fadd_rn(buf, __fmul_rn(static_cast<float>(row[xsrc[j]]), xw[j]));
      const float t = __fmul_rn(yw[k], buf);
      sum = k == y0 ? t : __fadd_rn(sum, t);
    }
    const int v = __float2int_rn(sum);
    out[o] = static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
  __syncthreads();
  // ---- FrameStack: fresh env -> all C slots; otherwise shift by one frame and append
  const bool fill = !p.fresh || p.fresh[n];
  uint4* st = reinterpret_cast<uint4*>(p.stack + n * p.C * static_cast<long long>(kWarpFrame));
  constexpr int kV = kWarpFrame / 16;
  for (int i = threadIdx.x; i < kV; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(out)[i];
    if (!fill)
      for (int c = 0; c + 1 < p.C; ++c) st[c * kV + i] = st[(c + 1) * kV + i];
    for (int c = fill ? 0 : p.C - 1; c < p.C; ++c) st[c * kV + i] = v;
  }
}

__global__ void __launch_bounds__(256) u8_lut_f32_kernel(const uint8_t* __restrict__ in, float* __restrict__ out,
                                                         long long n4, const float* __restrict__ lut) {
  __shared__ float t[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) t[i] = lut[i];
  __syncthreads();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint32_t v = reinterpret_cast<const uint32_t*>(in)[i];
    reinterpret_cast<float4*>(out)[i] = make_float4(t[v & 0xff], t[(v >> 8) & 0xff], t[(v >> 16) & 0xff], t[v >> 24]);
  }
}

}  // namespace trl

TRL_API int trl_atari_warp_stack(const uint8_t* frames, const int* env_idx, const uint8_t* fresh, uint8_t* stack,
                                 const int* tab_i, const float* tab_w, int64_t M, int64_t N, int H, int W, int C,
                                 void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 0 && N >= 0 && M <= 0x7fffffffLL, "trl_atari_warp_stack: bad size");
  TRL_REQUIRE(env_idx || M == N, "trl_atari_warp_stack: without env_idx there is one frame per env (M == N)");
  TRL_REQUIRE(H >= kWarpOut && W >= kWarpOut && (3 * W) % 16 == 0,
              "trl_atari_warp_stack: frames must be at least 84x84 with 3*W a multiple of 16, got %dx%d", H, W);
  TRL_REQUIRE(C >= 1 && C <= 255, "trl_atari_warp_stack: bad stack depth %d", C);
  const long long smem = static_cast<long long>(H) * W + kWarpFrame;
  TRL_REQUIRE(smem <= kWarpMaxSmem, "trl_atari_warp_stack: a %dx%d gray frame does not fit in shared memory", H, W);
  if (M == 0) return TRL_OK;
  TRL_REQUIRE(frames && stack && tab_i && tab_w, "trl_atari_warp_stack: null pointer");
  TRL_REQUIRE(aligned16(frames) && aligned16(stack), "trl_atari_warp_stack: frames and stack must be 16-byte aligned");
  if (smem > 48 * 1024) {
    const cudaError_t e =
        cudaFuncSetAttribute(atari_warp_stack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
  }
  const WarpStackParams p{frames, env_idx, fresh, stack, tab_i, tab_w, N, H, W, C};
  atari_warp_stack_kernel<<<static_cast<unsigned>(M), kWarpThreads, static_cast<size_t>(smem),
                            static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("atari_warp_stack_kernel");
}

TRL_API int trl_u8_lut_f32(const uint8_t* in, float* out, int64_t n, const float* lut, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 0 && n % 4 == 0, "trl_u8_lut_f32: element count must be a multiple of 4");
  if (n == 0) return TRL_OK;
  TRL_REQUIRE(in && out && lut && aligned4(in) && aligned16(out), "trl_u8_lut_f32: null or misaligned pointer");
  long long blocks = ceil_div<long long>(n / 4, 256);
  if (blocks > 16LL * kNumSM) blocks = 16LL * kNumSM;
  u8_lut_f32_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(in, out, n / 4, lut);
  return check_launch("u8_lut_f32_kernel");
}
