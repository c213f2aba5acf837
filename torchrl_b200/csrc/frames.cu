// frames.cu -- frame-de-duplicated pixel replay (SURVEY.md 8(f).5): what the reference obtains on the host with
// LazyFrames (/root/reference/torchrl/env/atari_wrapper.py:142-168: "common frames between the observations are only
// stored once") inside MemoryEfficientReplayBuffer (/root/reference/torchrl/replay_buffers/memory_efficient_replay_buffer.py:
// 5-33), as a device data layout.
//
// A stored transition of the frame-stacked pixel env holds obs = frames [t-3 .. t] and next_obs = frames [t-2 .. t+1]:
// 8 frames of which 6 are copies.  The ring keeps per time row and env only
//     obs_last [T][N][F]   the NEWEST frame of obs (frame t),
//     next_last[T][N][F]   the newest frame of next_obs (frame t+1; NOT row t+1's obs_last when the episode ended),
//     age      [T][N]      min(steps since the episode started, C-1): how many older frames of obs are real history
// (2 of 8 frames: 4x less HBM, 56 GB -> 14 GB for the 1M-transition ring of BASELINE config 4), plus a C-1 deep
// history of the frames most recently overwritten by the ring, so that the OLDEST rows still reconstruct exactly.
//   trl_frame_ring_write   : one collector step -- newest frame of the env's (N,C,F) stack -> ring row *top (saving the
//                            frame it overwrites into the history when the ring is full)
//   trl_frame_stack_gather : minibatch assembly -- for sampled rows, rebuild both C-frame stacks as float32 * scale
//                            (ScaledFloatFrame fused: the bytes are read once, widened on the way out)
// FrameStack.reset repeats the first frame (atari_wrapper.py:118-126), hence "frame older than the episode" = the
// episode's first frame = obs_last of the row `age` steps back.  HBM-bound byte work; no tensor cores.
#include "common.cuh"

namespace trl {

constexpr int kFrameThreads = 256;

struct FrameWriteParams {
  const uint8_t* __restrict__ stack;   // (N, C, F) current frame stack of the env
  uint8_t* __restrict__ ring;          // (T, N, F)
  uint8_t* __restrict__ age_ring;      // (T, N) or nullptr
  const int* __restrict__ elapsed;     // (N) steps since the env's last reset (with age_ring)
  uint8_t* __restrict__ hist;          // (C-1, N, F) frames most recently overwritten, or nullptr
  int* __restrict__ hist_count;        // device counter of history pushes
  const int* __restrict__ top;         // device scalar: row to write
  const int* __restrict__ size;        // device scalar: rows already valid (== T: the write overwrites a live row)
  long long N, F;
  int C, T, frame;                     // frame = which of the C frames to store (C-1: the newest)
};

// hist slot of the frame m steps older than the oldest ring row, after `hc` history pushes (the gather's indexing)
__device__ __forceinline__ long long frame_hist_slot(int hc, int m, int C) {
  return ((static_cast<long long>(hc) - m) % (C - 1) + (C - 1)) % (C - 1);
}

// grid = (chunks, min(N, 65535)): a CTA copies a 16-byte-aligned slice of the frames of envs y, y + gridDim.y, ...
__global__ void __launch_bounds__(kFrameThreads) frame_ring_write_kernel(const FrameWriteParams p) {
  const int row = *p.top;
  const int size = p.hist ? *p.size : 0;
  const bool full = p.hist && size >= p.T;
  // the first write into an empty ring: the row's older frames precede the ring, and the gather reads them from the
  // history (row 0 of a mid-episode stack), so the frames older than `frame` in this stack are seeded into the slots
  // the gather reads them from -- the frame d steps back at frame_hist_slot(hc, d)
  const bool seed = p.hist && size == 0;
  const int hc = p.hist ? *p.hist_count : 0;
  const long long v16 = p.F / 16;
  for (long long n = blockIdx.y; n < p.N; n += gridDim.y) {
    const uint8_t* src = p.stack + (n * p.C + p.frame) * p.F;
    uint8_t* dst = p.ring + (static_cast<long long>(row) * p.N + n) * p.F;
    uint8_t* old = full ? p.hist + ((static_cast<long long>(hc) % (p.C - 1)) * p.N + n) * p.F : nullptr;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < v16;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      if (full) reinterpret_cast<uint4*>(old)[i] = reinterpret_cast<const uint4*>(dst)[i];
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    }
    if (seed) {
      for (int d = 1; d <= p.frame && d < p.C; ++d) {
        const uint4* s = reinterpret_cast<const uint4*>(p.stack + (n * p.C + p.frame - d) * p.F);
        uint4* h = reinterpret_cast<uint4*>(p.hist + (frame_hist_slot(hc, d, p.C) * p.N + n) * p.F);
        for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < v16;
             i += static_cast<long long>(gridDim.x) * blockDim.x)
          h[i] = s[i];
      }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && p.age_ring) {
      const int e = p.elapsed[n];
      p.age_ring[static_cast<long long>(row) * p.N + n] = static_cast<uint8_t>(e < p.C - 1 ? e : p.C - 1);
    }
  }
}

__global__ void frame_hist_advance_kernel(int* __restrict__ hist_count, const int* __restrict__ size, int T) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && *size >= T) *hist_count += 1;
}

struct FrameGatherParams {
  const uint8_t* __restrict__ obs_last;    // (T, N, F)
  const uint8_t* __restrict__ next_last;   // (T, N, F)
  const uint8_t* __restrict__ age;         // (T, N)
  const uint8_t* __restrict__ hist;        // (C-1, N, F)
  const int* __restrict__ hist_count;
  const long long* __restrict__ idx;       // sampled rows
  const int* __restrict__ pos;             // optional device scalar: use idx[(*pos)*rows + k]
  const int* __restrict__ top;
  const int* __restrict__ size;
  float* __restrict__ out_obs;             // (rows*N, C, F) float32
  float* __restrict__ out_next;            // (rows*N, C, F) float32
  long long N, F;
  int C, T, rows;
  float scale;
};

// CTA x's slice of both stacks of sample s = k*N + n
__device__ __forceinline__ void frame_stack_gather_one(const FrameGatherParams& p, const long long s) {
  const int k = static_cast<int>(s / p.N);
  const long long n = s % p.N;
  const int r = static_cast<int>(p.idx[(p.pos ? static_cast<long long>(*p.pos) * p.rows : 0) + k]);
  const int size = *p.size, top = *p.top;
  // rows older than r that are still in the ring: all of [0, r) before the first wrap, else back to the tail `top`
  const int back = size >= p.T ? (r - top + p.T) % p.T : r;
  const int a = p.age[static_cast<long long>(r) * p.N + n];
  const int hc = *p.hist_count;
  const long long v4 = p.F / 4;
  for (int j = 0; j <= p.C; ++j) {
    // frame j of the virtual (C+1)-frame window [t-(C-1) .. t+1]: obs = frames 0..C-1, next_obs = frames 1..C
    const uint8_t* src;
    if (j == p.C) {
      src = p.next_last + (static_cast<long long>(r) * p.N + n) * p.F;
    } else {
      int d = p.C - 1 - j;                   // steps back from row r
      if (d > a) d = a;                      // older than the episode: its first frame (FrameStack.reset)
      if (d <= back) {
        src = p.obs_last + (static_cast<long long>((r - d + p.T) % p.T) * p.N + n) * p.F;
      } else {                               // overwritten by the ring: the (d - back)-th newest history entry
        const int m = d - back;
        src = p.hist + (frame_hist_slot(hc, m, p.C) * p.N + n) * p.F;
      }
    }
    float* o1 = j < p.C ? p.out_obs + (s * p.C + j) * p.F : nullptr;
    float* o2 = j > 0 ? p.out_next + (s * p.C + (j - 1)) * p.F : nullptr;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < v4;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const uint32_t v = reinterpret_cast<const uint32_t*>(src)[i];
      const float4 f = make_float4((v & 0xff) * p.scale, ((v >> 8) & 0xff) * p.scale, ((v >> 16) & 0xff) * p.scale,
                                   (v >> 24) * p.scale);
      if (o1) reinterpret_cast<float4*>(o1)[i] = f;
      if (o2) reinterpret_cast<float4*>(o2)[i] = f;
    }
  }
}

// grid = (chunks, min(rows*N, 65535)): CTA (x, y) rebuilds its slice of the samples y, y + gridDim.y, ... (grid y is
// limited to 65535, a batch of samples is not)
__global__ void __launch_bounds__(kFrameThreads) frame_stack_gather_kernel(const FrameGatherParams p) {
  const long long samples = static_cast<long long>(p.rows) * p.N;
  for (long long s = blockIdx.y; s < samples; s += gridDim.y) frame_stack_gather_one(p, s);
}

}  // namespace trl

// Store frame `frame` (0-based; C-1 = newest) of every env's (N, C, F) uint8 stack at ring row *top.  age_ring /
// elapsed (both or neither): also record min(elapsed, C-1).  hist / hist_count / size (all or none): when the ring is
// full the overwritten frame is pushed into the (C-1)-deep history first; call trl_frame_hist_advance once per step
// after all writes of that step.  When the ring is empty (*size == 0) the stack's frames older than `frame` are
// seeded into the history, so a first row recorded mid-episode (age > 0) rebuilds its real older frames.  F % 16 == 0,
// 16-byte aligned buffers.
TRL_API int trl_frame_ring_write(const uint8_t* stack, uint8_t* ring, uint8_t* age_ring, const int* elapsed, uint8_t* hist,
                                 int* hist_count, const int* top, const int* size, int64_t N, int C, int64_t F, int T,
                                 int frame, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 1 && C >= 2 && F >= 16 && F % 16 == 0 && T >= 1 && frame >= 0 && frame < C,
              "trl_frame_ring_write: bad sizes N=%lld C=%d F=%lld T=%d frame=%d", (long long)N, C, (long long)F, T, frame);
  TRL_REQUIRE(stack && ring && top, "trl_frame_ring_write: null pointer");
  TRL_REQUIRE((age_ring == nullptr) == (elapsed == nullptr), "trl_frame_ring_write: age_ring and elapsed go together");
  TRL_REQUIRE((hist == nullptr) == (hist_count == nullptr) && (hist == nullptr || size != nullptr),
              "trl_frame_ring_write: hist, hist_count and size go together");
  TRL_REQUIRE(aligned16(stack) && aligned16(ring) && aligned16(hist), "trl_frame_ring_write: buffers must be 16-byte aligned");
  FrameWriteParams p{stack, ring, age_ring, elapsed, hist, hist_count, top, size, N, F, C, T, frame};
  const unsigned chunks = static_cast<unsigned>(ceil_div<long long>(F / 16, kFrameThreads) < 4 ? ceil_div<long long>(F / 16, kFrameThreads) : 4);
  frame_ring_write_kernel<<<dim3(chunks, static_cast<unsigned>(N < 65535 ? N : 65535)), kFrameThreads, 0,
                            static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("frame_ring_write_kernel");
}

TRL_API int trl_frame_hist_advance(int* hist_count, const int* size, int T, void* stream) {
  using namespace trl;
  TRL_REQUIRE(hist_count && size && T >= 1, "trl_frame_hist_advance: bad arguments");
  frame_hist_advance_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(hist_count, size, T);
  return check_launch("frame_hist_advance_kernel");
}

// out_obs / out_next (rows*N, C, F) float32 = scale * the C-frame stacks of the sampled rows idx[(*pos)*rows + k]
// (pos NULL: idx[k]), rebuilt from the de-duplicated ring.
TRL_API int trl_frame_stack_gather(const uint8_t* obs_last, const uint8_t* next_last, const uint8_t* age, const uint8_t* hist,
                                   const int* hist_count, const int64_t* idx, const int* pos, int rows, const int* top,
                                   const int* size, int64_t N, int C, int64_t F, int T, float scale, float* out_obs,
                                   float* out_next, void* stream) {
  using namespace trl;
  TRL_REQUIRE(N >= 1 && C >= 2 && F >= 16 && F % 16 == 0 && T >= 1 && rows >= 0, "trl_frame_stack_gather: bad sizes");
  if (rows == 0) return TRL_OK;
  TRL_REQUIRE(obs_last && next_last && age && hist && hist_count && idx && top && size && out_obs && out_next,
              "trl_frame_stack_gather: null pointer");
  TRL_REQUIRE(aligned16(obs_last) && aligned16(next_last) && aligned16(hist) && aligned16(out_obs) && aligned16(out_next),
              "trl_frame_stack_gather: buffers must be 16-byte aligned");
  FrameGatherParams p{obs_last, next_last, age, hist, hist_count, reinterpret_cast<const long long*>(idx), pos, top, size,
                      out_obs, out_next, N, F, C, T, rows, scale};
  long long chunks = ceil_div<long long>(F / 4, 4LL * kFrameThreads);
  if (chunks < 1) chunks = 1;
  const long long samples = static_cast<long long>(rows) * N;
  const unsigned grid_samples = samples < 65535 ? static_cast<unsigned>(samples) : 65535u;
  frame_stack_gather_kernel<<<dim3(static_cast<unsigned>(chunks), grid_samples), kFrameThreads, 0,
                              static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("frame_stack_gather_kernel");
}
