// atari_env.cu -- K1 for BASELINE.json config 4: synthetic Atari-shaped pixel env (4x84x84 uint8, 6 actions).
//
// The reference only wraps real ALE games (/root/reference/torchrl/env/atari_wrapper.py: WarpFrame :112-131,
// FrameStack :134-168 give the (4,84,84) uint8 observation); the synthetic game is defined by this build in
// oracle/synth_atari.py (pure integer arithmetic => the CUDA env is BIT-EXACT against it).  One CTA per env:
// shift the 4-frame stack by one frame, render the new 84x84 frame, advance the latent state.  HBM traffic
// per env-step: 21 KB read + 28 KB written (uint8) -- HBM-bound at large N.
#include "env_common.cuh"

namespace trl {

constexpr int kAH = 84, kAW = 84, kFrame = kAH * kAW;      // 7056 bytes = 441 x 16
constexpr int kPaddleY = 78, kPaddleW = 12, kBall = 4;

__device__ __forceinline__ uint8_t apixel(int x, int y, int bx, int by, int px) {
  if (x >= bx && x < bx + kBall && y >= by && y < by + kBall) return 255;
  if (y >= kPaddleY && y < kPaddleY + 2 && x >= px && x < px + kPaddleW) return 200;
  return static_cast<uint8_t>(((7 * x + 13 * y) & 31) + 16);
}
__device__ __forceinline__ void arender(uint8_t* frame, int bx, int by, int px) {
  for (int i = threadIdx.x; i < kFrame / 4; i += blockDim.x) {
    const int p = i * 4, y = p / kAW, x = p - y * kAW;       // 84 % 4 == 0: four pixels of one row
    const uint32_t v = apixel(x, y, bx, by, px) | (apixel(x + 1, y, bx, by, px) << 8) |
                       (apixel(x + 2, y, bx, by, px) << 16) | (static_cast<uint32_t>(apixel(x + 3, y, bx, by, px)) << 24);
    reinterpret_cast<uint32_t*>(frame)[i] = v;
  }
}

// latent: (N,5) int32 = bx, by, vx, vy, px
__global__ void __launch_bounds__(256) synth_atari_step_kernel(uint8_t* __restrict__ obs, int* __restrict__ latent,
                                                              const float* __restrict__ actions, int* __restrict__ elapsed,
                                                              float* __restrict__ reward, uint8_t* __restrict__ done,
                                                              uint8_t* __restrict__ time_limit, int max_steps) {
  const long long n = blockIdx.x;
  uint8_t* o = obs + n * 4 * kFrame;
  int* L = latent + n * 5;
  int bx = L[0], by = L[1], vx = L[2], vy = L[3], px = L[4];
  const int a = static_cast<int>(actions[n]);
  const int dx = (a == 2) ? 3 : (a == 3) ? -3 : (a == 4) ? 6 : (a == 5) ? -6 : 0;
  px = min(max(px + dx, 0), kAW - kPaddleW);
  bx += vx; by += vy;
  if (bx < 0) { bx = -bx; vx = -vx; }
  if (bx > kAW - kBall) { bx = 2 * (kAW - kBall) - bx; vx = -vx; }
  if (by < 0) { by = -by; vy = -vy; }
  int r = 0;
  bool miss = false;
  if (by >= kPaddleY - kBall) {
    if (bx >= px - 3 && bx <= px + kPaddleW - 1) { r = 1; by = 2 * (kPaddleY - kBall) - by; vy = -vy; }
    else { r = -1; miss = true; }
  }
  // shift the frame stack (frame c <- frame c+1), 16-byte vectors, barrier between overlapping moves
  for (int c = 0; c < 3; ++c) {
    const uint4* src = reinterpret_cast<const uint4*>(o + (c + 1) * kFrame);
    uint4* dst = reinterpret_cast<uint4*>(o + c * kFrame);
    for (int i = threadIdx.x; i < kFrame / 16; i += blockDim.x) dst[i] = src[i];
    __syncthreads();
  }
  arender(o + 3 * kFrame, bx, by, px);
  if (threadIdx.x == 0) {
    L[0] = bx; L[1] = by; L[2] = vx; L[3] = vy; L[4] = px;
    const int el = elapsed[n] + 1;
    elapsed[n] = el;
    const bool dn = miss || el >= max_steps;
    reward[n] = static_cast<float>(r);
    done[n] = dn ? 1 : 0;
    time_limit[n] = (dn && el == max_steps) ? 1 : 0;
  }
}

// reset envs whose mask is set (mask NULL: all); episode index = episode[n] - episode_bias, then episode[n]++
// unless `bump` is 0 (the collector's finalize kernel already advanced it: episode_bias = 1, bump = 0).
__global__ void __launch_bounds__(256) synth_atari_reset_kernel(uint8_t* __restrict__ obs, int* __restrict__ latent,
                                                               int* __restrict__ elapsed, unsigned* __restrict__ episode,
                                                               const unsigned* __restrict__ seeds,
                                                               const uint8_t* __restrict__ mask,
                                                               const int* __restrict__ zero_is_mask, int episode_bias,
                                                               int bump) {
  const long long n = blockIdx.x;
  if (mask && !mask[n]) return;
  if (zero_is_mask && zero_is_mask[n] != 0) return;
  const unsigned seed = seeds[n], ep = episode[n] - static_cast<unsigned>(episode_bias);
  const int h0 = static_cast<int>(counter_hash(seed, ep, 0) % 72u);
  const int h1 = static_cast<int>(counter_hash(seed, ep, 1) % 40u);
  const unsigned h2 = counter_hash(seed, ep, 2), h3 = counter_hash(seed, ep, 3);
  const int bx = 4 + h0, by = 4 + h1;
  const int vx = ((h2 & 1u) ? 1 : -1) * (1 + static_cast<int>((h2 >> 1) & 1u));
  const int vy = 1 + static_cast<int>(h3 & 1u);
  const int px = static_cast<int>(counter_hash(seed, ep, 4) % 73u);
  uint8_t* o = obs + n * 4 * kFrame;
  for (int c = 0; c < 4; ++c) arender(o + c * kFrame, bx, by, px);     // FrameStack.reset repeats the first frame
  if (threadIdx.x == 0) {
    int* L = latent + n * 5;
    L[0] = bx; L[1] = by; L[2] = vx; L[3] = vy; L[4] = px;
    elapsed[n] = 0;
    if (bump) episode[n] += 1u;
  }
}

// u8 -> f32 with scale (ScaledFloatFrame, atari_wrapper.py:171-180: obs / 255)
__global__ void u8_to_f32_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, long long n4, float scale) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint32_t v = reinterpret_cast<const uint32_t*>(in)[i];
    reinterpret_cast<float4*>(out)[i] = make_float4((v & 0xff) * scale, ((v >> 8) & 0xff) * scale,
                                                    ((v >> 16) & 0xff) * scale, (v >> 24) * scale);
  }
}

}  // namespace trl

TRL_API int trl_synth_atari_step(uint8_t* obs, int* latent, const float* actions, int* elapsed, float* reward,
                                 uint8_t* done, uint8_t* time_limit, int64_t N, int max_steps, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0, "trl_synth_atari_step: bad size");
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(obs && latent && actions && elapsed && reward && done && time_limit, "trl_synth_atari_step: null pointer");
  TRL_REQUIRE(aligned16(obs), "trl_synth_atari_step: obs must be 16-byte aligned");
  synth_atari_step_kernel<<<static_cast<unsigned>(N), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      obs, latent, actions, elapsed, reward, done, time_limit, max_steps);
  return check_launch("synth_atari_step_kernel");
}

TRL_API int trl_synth_atari_reset(uint8_t* obs, int* latent, int* elapsed, unsigned* episode, const unsigned* seeds,
                                  const uint8_t* mask, const int* zero_is_mask, int episode_bias, int bump, int64_t N,
                                  void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 0, "trl_synth_atari_reset: bad size");
  if (N == 0) return TRL_OK;
  TRL_REQUIRE(obs && latent && elapsed && episode && seeds, "trl_synth_atari_reset: null pointer");
  synth_atari_reset_kernel<<<static_cast<unsigned>(N), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      obs, latent, elapsed, episode, seeds, mask, zero_is_mask, episode_bias, bump);
  return check_launch("synth_atari_reset_kernel");
}

TRL_API int trl_u8_to_f32(const uint8_t* in, float* out, int64_t n, float scale, void* stream) {
  using namespace trl;
  TRL_REQUIRE(n >= 0 && n % 4 == 0, "trl_u8_to_f32: element count must be a multiple of 4");
  if (n == 0) return TRL_OK;
  TRL_REQUIRE(in && out && aligned4(in) && aligned16(out), "trl_u8_to_f32: null or misaligned pointer");
  long long blocks = ceil_div<long long>(n / 4, 256);
  if (blocks > 16LL * kNumSM) blocks = 16LL * kNumSM;
  u8_to_f32_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(in, out, n / 4, scale);
  return check_launch("u8_to_f32_kernel");
}
