// gae_tma.cu -- K6 at scale: the GAE / discounted-return scan of csrc/gae.cu as a PERSISTENT kernel whose input
// tiles are staged in shared memory by TMA (cp.async.bulk.tensor), two tiles in flight per SM.
//
// Same recurrences and the same chunk composition as gae_chunked_kernel (gae_common.cuh;
// /root/reference/torchrl/replay_buffers/on_policy.py:16-70).  What changes is how the bytes move: in
// gae_chunked_kernel every thread holds its loads in registers (64 regs x 1024 threads -> one CTA per SM), so an SM
// alternates between a load phase and a store phase and the next CTA's loads only start when the previous CTA has
// retired (ncu: 41.9 % warps active, long-scoreboard stalls, 62.5 % of DRAM peak).  Here one elected thread asks
// the TMA engine for the NEXT (64 timesteps x 128 envs) tile of rewards / values / terminals / time_limits
// (80.5 KB, four boxes) while the 512 compute threads work on the current one out of shared memory: loads never
// wait on stores, registers hold one tile's worth of data only while it is being scanned.
//   work item   = (env group of 128, time tile of 64), tiles of one group visited from the last to the first
//                 (the carry x_{t0} flows to the earlier tile through shared memory);
//   CTA         = 16 warps: warp w scans the 4 timesteps [t0 + 4w, t0 + 4w + 4), lane = 4 consecutive envs
//                 (LDS.128 rows of 512 B: conflict-free), composition of the 16 chunk maps through shared memory;
//   grid        = min(#groups, kNumSM = 132) persistent CTAs, group g -> CTA g % grid.
// Algorithmic traffic is unchanged: 10 B read + 8 B written per (t, n) element, + 4 B per env for last_value.
#include "gae_common.cuh"
#include <cuda.h>

namespace trl {
namespace gaetma {

constexpr int kG = 128;                    // envs per group
constexpr int kTT = 64;                    // timesteps per tile
constexpr int kTC = 4;                     // timesteps per warp
constexpr int kW = kTT / kTC;              // 16 warps
constexpr int kThreads = 32 * kW;          // 512
constexpr int kStages = 2;
constexpr int kRBytes = kTT * kG * 4;          // 32768
constexpr int kVBytes = (kTT + 1) * kG * 4;    // 33280: one extra row = V of the first step of the later tile
constexpr int kFBytes = kTT * kG;              // 8192
constexpr int kOffV = kRBytes, kOffT = kOffV + kVBytes, kOffL = kOffT + kFBytes;
constexpr int kStageBytes = kOffL + kFBytes;   // 82432 (a multiple of 128)
constexpr int kTxBytes = kRBytes + kVBytes + 2 * kFBytes;
constexpr int kScanFloats = (2 * kW + 1) * kG; // chunk maps (a, b) per warp + the tile-to-tile carry
constexpr int kSmemBytes = kStages * kStageBytes + kScanFloats * 4 + 64 /*barriers*/ + 128 /*align*/;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c_inner, int c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c_inner), "r"(c_outer)
      : "memory");
}

struct TmaGaeParams {
  const float* __restrict__ last_value;    // (N)
  float* __restrict__ advs;                // (T,N)
  float* __restrict__ rets;                // (T,N)
  long long T, N;
  float gamma, gamma_tau;
  int filter;
  int groups;                              // N / 128
  int tiles;                               // ceil(T / 64)
};

template <int MODE>
__global__ void __launch_bounds__(kThreads, 1)
gae_tma_kernel(const __grid_constant__ CUtensorMap map_r, const __grid_constant__ CUtensorMap map_v,
               const __grid_constant__ CUtensorMap map_t, const __grid_constant__ CUtensorMap map_l, const TmaGaeParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~static_cast<uintptr_t>(127));
  float* scan = reinterpret_cast<float*>(smem + kStages * kStageBytes);
  float* sa = scan;                        // [kW][kG]
  float* sb = scan + kW * kG;              // [kW][kG]
  float* sc = scan + 2 * kW * kG;          // [kG] carry to the earlier tile
  uint64_t* full = reinterpret_cast<uint64_t*>(scan + kScanFloats);

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const long long N = p.N, T = p.T;
  const float g = p.gamma, gt = p.gamma_tau;
  const int filter = p.filter;
  const int my_groups = (p.groups - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int n_items = my_groups * p.tiles;

  if (tid == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_r)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_v)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_t)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_l)) : "memory");
    for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // item i of this CTA: group blockIdx.x + (i / tiles) * gridDim.x, tile j = i % tiles covering
  // [T - 64 (j + 1), T - 64 j): the earliest tile may start below 0 (TMA fills what lies outside with zeros)
  auto issue = [&](int i) {
    const int s = i & 1;
    const int grp = static_cast<int>(blockIdx.x) + (i / p.tiles) * static_cast<int>(gridDim.x);
    const int t0 = static_cast<int>(T) - kTT * (i % p.tiles + 1);
    uint8_t* st = smem + s * kStageBytes;
    mbar_arrive_expect_tx(&full[s], kTxBytes);
    tma_load_2d(st, &map_r, &full[s], grp * kG, t0);
    tma_load_2d(st + kOffV, &map_v, &full[s], grp * kG, t0);
    tma_load_2d(st + kOffT, &map_t, &full[s], grp * kG, t0);
    tma_load_2d(st + kOffL, &map_l, &full[s], grp * kG, t0);
  };
  if (tid == 0) {
    if (n_items > 0) issue(0);
    if (n_items > 1) issue(1);
  }

  float carry[4] = {0.f, 0.f, 0.f, 0.f};
  for (int it = 0; it < n_items; ++it) {
    const int s = it & 1;
    const int tile = it % p.tiles;
    const int grp = static_cast<int>(blockIdx.x) + (it / p.tiles) * static_cast<int>(gridDim.x);
    const long long env0 = static_cast<long long>(grp) * kG + lane * 4;
    const long long t0 = T - static_cast<long long>(kTT) * (tile + 1) + static_cast<long long>(w) * kTC;   // may be < 0
    float lastv[4] = {0.f, 0.f, 0.f, 0.f};
    if (tile == 0 && (w == kW - 1 || MODE == MODE_DISC)) load_f<4>(p.last_value + env0, lastv);
    if (tile == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) carry[i] = (MODE == MODE_DISC) ? lastv[i] : 0.f;
    }
    mbar_wait(&full[s], (it >> 1) & 1);
    const uint8_t* st = smem + s * kStageBytes;
    float r[kTC][4], v[kTC][4], vn[4];
    unsigned ft[kTC], fl[kTC];
#pragma unroll
    for (int k = 0; k < kTC; ++k) {
      const int row = w * kTC + k;
      const float4 rr = *reinterpret_cast<const float4*>(st + (row * kG + lane * 4) * 4);
      const float4 vv = *reinterpret_cast<const float4*>(st + kOffV + (row * kG + lane * 4) * 4);
      r[k][0] = rr.x; r[k][1] = rr.y; r[k][2] = rr.z; r[k][3] = rr.w;
      v[k][0] = vv.x; v[k][1] = vv.y; v[k][2] = vv.z; v[k][3] = vv.w;
      ft[k] = *reinterpret_cast<const unsigned*>(st + kOffT + row * kG + lane * 4);
      fl[k] = *reinterpret_cast<const unsigned*>(st + kOffL + row * kG + lane * 4);
    }
    {
      const float4 vv = *reinterpret_cast<const float4*>(st + kOffV + ((w * kTC + kTC) * kG + lane * 4) * 4);
      vn[0] = vv.x; vn[1] = vv.y; vn[2] = vv.z; vn[3] = vv.w;
      if (tile == 0 && w == kW - 1) {         // the step after the last stored row: V_T = last_value
#pragma unroll
        for (int i = 0; i < 4; ++i) vn[i] = lastv[i];
      }
    }
    // ---- pass 1: per-step coefficients, chunk composition (as gae_chunked_kernel) ----------------------------
    float ca[4], cb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { ca[i] = 0.f; cb[i] = 1.f; }
#pragma unroll
    for (int k = kTC - 1; k >= 0; --k) {
      const bool live = (t0 + k) >= 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned term = (ft[k] >> (8 * i)) & 0xffu, tl = (fl[k] >> (8 * i)) & 0xffu;
        const float vnext = (k == kTC - 1) ? vn[i] : v[(k + 1) % kTC][i];
        float ak, bk;
        coeffs<MODE>(r[k][i], v[k][i], vnext, term, tl, g, gt, filter, ak, bk);
        if (!live) { ak = 0.f; bk = 1.f; }   // identity for the ragged head (t < 0)
        r[k][i] = ak;
        ca[i] = fmaf(bk, ca[i], ak);
        cb[i] = bk * cb[i];
      }
    }
    *reinterpret_cast<float4*>(sa + w * kG + lane * 4) = make_float4(ca[0], ca[1], ca[2], ca[3]);
    *reinterpret_cast<float4*>(sb + w * kG + lane * 4) = make_float4(cb[0], cb[1], cb[2], cb[3]);
    __syncthreads();
    // every thread has copied its part of stage s into registers: refill it with the tile after the next one, so
    // that two tiles (2 x 80.5 KB) stay in flight per SM while this one is scanned and stored
    if (tid == 0 && it + 2 < n_items) issue(it + 2);
    // ---- carry-in: compose the later chunks of this tile onto `carry` --------------------------------------------
    float x[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = carry[i];
    for (int w2 = kW - 1; w2 > w; --w2) {
      const float4 a4 = *reinterpret_cast<const float4*>(sa + w2 * kG + lane * 4);
      const float4 b4 = *reinterpret_cast<const float4*>(sb + w2 * kG + lane * 4);
      x[0] = fmaf(b4.x, x[0], a4.x); x[1] = fmaf(b4.y, x[1], a4.y);
      x[2] = fmaf(b4.z, x[2], a4.z); x[3] = fmaf(b4.w, x[3], a4.w);
    }
    // ---- pass 2: replay from registers, write outputs ----------------------------------------------------------------
#pragma unroll
    for (int k = kTC - 1; k >= 0; --k) {
      const long long t = t0 + k;
      float oa[4], orr[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned term = (ft[k] >> (8 * i)) & 0xffu, tl = (fl[k] >> (8 * i)) & 0xffu;
        float bk = bcoef<MODE>(term, tl, g, gt, filter);
        if (t < 0) bk = 1.f;
        x[i] = fmaf(bk, x[i], r[k][i]);
        if (MODE == MODE_GAE) { oa[i] = x[i]; orr[i] = x[i] + v[k][i]; }
        else { oa[i] = x[i] - v[k][i]; orr[i] = x[i]; }
      }
      if (t >= 0) {
        store_f<4>(p.advs + t * N + env0, oa);
        store_f<4>(p.rets + t * N + env0, orr);
      }
    }
    // ---- hand x at the start of this tile to the earlier tile of the same group ------------------------------------
    if (w == 0) *reinterpret_cast<float4*>(sc + lane * 4) = make_float4(x[0], x[1], x[2], x[3]);
    __syncthreads();       // also: every read of sa / sb / this stage is done before the next item overwrites them
    {
      const float4 c4 = *reinterpret_cast<const float4*>(sc + lane * 4);
      carry[0] = c4.x; carry[1] = c4.y; carry[2] = c4.z; carry[3] = c4.w;
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// (T x N) row-major array of `elem` bytes per element, box = (128 envs, box_rows timesteps), no swizzle
static bool make_map(CUtensorMap* map, const void* base, long long T, long long N, int elem, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return false;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(N), static_cast<cuuint64_t>(T)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(N) * elem};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kG), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  return enc(map, elem == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base),
             gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace gaetma

bool gae_tma_supported(const GaeParams& p) {
  return p.N >= gaetma::kG && p.N % gaetma::kG == 0 && p.T >= 1 && p.T < (1LL << 30) && p.N < (1LL << 31) &&
         aligned16(p.rewards) && aligned16(p.values) && aligned16(p.terminals) && aligned16(p.time_limits) &&
         aligned16(p.last_value) && aligned16(p.advs) && aligned16(p.rets);
}

int gae_tma_launch(const GaeParams& p, int mode, cudaStream_t st) {
  using namespace gaetma;
  CUtensorMap mr, mv, mt, ml;
  if (!make_map(&mr, p.rewards, p.T, p.N, 4, kTT) || !make_map(&mv, p.values, p.T, p.N, 4, kTT + 1) ||
      !make_map(&mt, p.terminals, p.T, p.N, 1, kTT) || !make_map(&ml, p.time_limits, p.T, p.N, 1, kTT)) {
    set_error("gae_tma: cuTensorMapEncodeTiled failed");
    return TRL_EUNSUPPORTED;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gae_tma_kernel<MODE_GAE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gae_tma_kernel<MODE_DISC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
    attr_set = true;
  }
  TmaGaeParams q{p.last_value, p.advs, p.rets, p.T, p.N, p.gamma, p.gamma_tau, p.filter,
                 static_cast<int>(p.N / kG), static_cast<int>(ceil_div<long long>(p.T, kTT))};
  const unsigned grid = static_cast<unsigned>(q.groups < kNumSM ? q.groups : kNumSM);
  if (mode == MODE_GAE) gae_tma_kernel<MODE_GAE><<<grid, kThreads, kSmemBytes, st>>>(mr, mv, mt, ml, q);
  else gae_tma_kernel<MODE_DISC><<<grid, kThreads, kSmemBytes, st>>>(mr, mv, mt, ml, q);
  return check_launch("gae_tma_kernel");
}

}  // namespace trl
