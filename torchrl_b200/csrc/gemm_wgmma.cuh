// gemm_wgmma.cuh -- fp32-faithful (3xTF32) warpgroup-MMA GEMM for the 256-wide MLP layers on sm_90a.
//
//   C[M x 256] (+ bias, activation) = A . B          3 products per 8-deep K step: lo*hi, hi*lo, hi*hi
//
// Every operand element is split into x = hi + lo (hi = TF32-rounded, lo = exact remainder) and each K step issues
// three wgmma.mma_async.m64n128k8.tf32 ("3xTF32"; the dropped lo*lo term is O(2^-22) relative).  The tensor core's
// fp32 accumulation truncates, so the error grows ~linearly with the number of adds into a running sum: hi*hi goes to
// one register accumulator and the two small correction products to a second one, summed in the epilogue, so that the
// large sum takes one add per K step instead of three.  Callers keep K / splits <= 256 where accuracy matters (the
// wgrad shape splits K).
//
// One CTA per 128 x 128 output tile and K slab (gridDim = (M tiles, 2 column halves, splits)), 288 threads:
//   warp 8       TMA producer : cp.async.bulk.tensor 2D loads of the raw fp32 A / B tiles (no swizzle) into a
//                               2-stage ring, mbarrier complete_tx
//   warps 0..7   two consumer warpgroups.  Per K block of 32: split raw -> (hi, lo) while re-laying the tile out as the
//                               K-major SWIZZLE_128B canonical layout wgmma reads (this is also where M/N-major sources --
//                               the dgrad B and both wgrad operands -- are transposed: wgmma takes tf32 operands from
//                               shared memory only K-major), release the raw stage, then warpgroup w issues the 12
//                               wgmma of its 64 rows into two register accumulators (see above).  The hi/lo tiles
//                               are double-buffered, so the MMAs of block kb run while block kb + 1 is converted.
//   epilogue                  accumulator fragments -> bias / activation -> global (float2 per thread, 32-byte rows).
// Shapes (template flags):
//   AMN = false: A (M x K) row-major;  AMN = true: A (K x M) row-major (reduction index = row index)
//   BMN = false: B (256 x K) row-major; BMN = true: B (K x 256) row-major
//   BSPLIT: B arrives as two pre-split planes (hi = tf32(w), lo = w - hi) and is only re-laid out, not split.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace trl {
namespace wg {

constexpr int kBM = 128, kBN = 128, kN = 256, kBK = 32;
constexpr int kRawStages = 2;
constexpr int kTileBytes = 128 * kBK * 4;                 // 16 KB: one 128 x 32 fp32 tile
constexpr int kRawStageBytes = 3 * kTileBytes;            // A | B (hi) | B lo (pre-split B only)
constexpr int kHiLoBytes = 4 * kTileBytes;                // A hi | A lo | B hi | B lo
constexpr int kConsumers = 256;                           // two warpgroups
constexpr int kThreads = kConsumers + 32;                 // + TMA warp
constexpr int kSmemBytes = 2 * kHiLoBytes + kRawStages * kRawStageBytes + 1024 /*align*/ + 64 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "fits one sm_90 CTA");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
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
// named barrier of the two consumer warpgroups (the TMA warp does not take part)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

// K-major SWIZZLE_128B canonical layout: rows of 32 fp32 (128 B), 16-byte chunk c of row r stored at chunk c ^ (r & 7),
// 8-row atoms of 1024 B.  Descriptor: start >> 4, LBO unused (1), SBO = 1024 B, layout type 1 (128B swizzle).
__device__ __forceinline__ uint64_t desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// d[64] += A(64 x 8) . B(128 x 8)^T, both K-major in shared memory, tf32 inputs, fp32 accumulate (one warpgroup)
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(1));
}

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w));
}
__device__ __forceinline__ float4 tf32_hi(const float4 v) {
  float4 h;
  unsigned u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.x)); h.x = __uint_as_float(u);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.y)); h.y = __uint_as_float(u);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.z)); h.z = __uint_as_float(u);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v.w)); h.w = __uint_as_float(u);
  return h;
}

// float4 unit u (0..1023) of a 128 x 32 tile: its row of the K-major destination and its 16-byte chunk (4 reduction
// indices), read from the raw tile as TMA delivered it: (128 rows x 32) for K-major sources, (32 x 128) for M/N-major
__device__ __forceinline__ float4 load_unit(uint32_t raw, int u, bool mn, int& row, int& chunk) {
  if (!mn) {
    row = u >> 3; chunk = u & 7;
    return lds128(raw + static_cast<uint32_t>(u) * 16u);
  }
  row = u & 127; chunk = u >> 7;
  const uint32_t a = raw + static_cast<uint32_t>(chunk * 4 * 128 + row) * 4u;
  return make_float4(lds32(a), lds32(a + 512u), lds32(a + 1024u), lds32(a + 1536u));
}
__device__ __forceinline__ uint32_t sw128(int row, int chunk) {
  return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}

struct Params {
  const float* __restrict__ bias;  // (256) added in the epilogue, or nullptr
  int act;                         // 0 none, 1 tanh, 2 relu (after the bias)
  float* __restrict__ C;           // (splits, M, 256) when splits > 1 else (M, 256)
  long long M;                     // output rows
  int k_blocks_per_split;          // K blocks (of 32) accumulated by one CTA
};

// TANH_MUFU: tanh as tanh_ex2 (common.cuh, |abs err| < 2.5e-7) instead of libdevice tanhf
template <bool AMN, bool BMN, bool BSPLIT, bool TANH_MUFU>
__global__ void __launch_bounds__(kThreads, 1)
gemm3_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                   const __grid_constant__ CUtensorMap map_b2, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* hilo = smem;                                    // [2][A hi | A lo | B hi | B lo]
  uint8_t* raw = smem + 2 * kHiLoBytes;                    // [kRawStages][A | B | B lo]
  uint64_t* bars = reinterpret_cast<uint64_t*>(raw + kRawStages * kRawStageBytes);
  uint64_t* full = bars;                                   // [kRawStages] TMA -> consumers
  uint64_t* empty = bars + kRawStages;                     // [kRawStages] consumers -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, n0 = blockIdx.y * kBN, split = blockIdx.z;
  const int nkb = p.k_blocks_per_split;
  const int kb0 = split * nkb;

  if (threadIdx.x == kConsumers) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b)) : "memory");
    if (BSPLIT) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b2)) : "memory");
    for (int s = 0; s < kRawStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumers / 32);               // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumers / 32) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % kRawStages;
        const uint32_t ph = (kb / kRawStages) & 1;
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = raw + s * kRawStageBytes;
        mbar_arrive_expect_tx(&full[s], (BSPLIT ? 3 : 2) * kTileBytes);
        const int k0 = (kb0 + kb) * kBK;
        if (AMN) tma_load_2d(st, &map_a, &full[s], m_blk * kBM, k0);
        else tma_load_2d(st, &map_a, &full[s], k0, m_blk * kBM);
        if (BMN) tma_load_2d(st + kTileBytes, &map_b, &full[s], n0, k0);
        else tma_load_2d(st + kTileBytes, &map_b, &full[s], k0, n0);
        if (BSPLIT) {
          if (BMN) tma_load_2d(st + 2 * kTileBytes, &map_b2, &full[s], n0, k0);
          else tma_load_2d(st + 2 * kTileBytes, &map_b2, &full[s], k0, n0);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  const int ct = threadIdx.x, wgi = warp >> 2;
  float acc[64], cor[64];                                  // hi*hi | lo*hi + hi*lo
#pragma unroll
  for (int i = 0; i < 64; ++i) { acc[i] = 0.f; cor[i] = 0.f; }
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % kRawStages;
    const uint32_t ph = (kb / kRawStages) & 1;
    const uint32_t rs = smem_u32(raw + s * kRawStageBytes);
    const uint32_t hs = smem_u32(hilo + (kb & 1) * kHiLoBytes);
    mbar_wait(&full[s], ph);
    // per operand: all loads of this thread first (independent accesses in flight), then split and store
    {
      float4 va[4];
      int ra[4], ca[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) va[i] = load_unit(rs, ct + i * kConsumers, AMN, ra[i], ca[i]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 h = tf32_hi(va[i]);
        const uint32_t o = sw128(ra[i], ca[i]);
        sts128(hs + o, h);
        sts128(hs + kTileBytes + o, make_float4(va[i].x - h.x, va[i].y - h.y, va[i].z - h.z, va[i].w - h.w));
      }
    }
    {
      float4 vb[4], vl[4];
      int rb[4], cb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) vb[i] = load_unit(rs + kTileBytes, ct + i * kConsumers, BMN, rb[i], cb[i]);
      if (BSPLIT) {
#pragma unroll
        for (int i = 0; i < 4; ++i) vl[i] = load_unit(rs + 2 * kTileBytes, ct + i * kConsumers, BMN, rb[i], cb[i]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);               // raw stage s may be refilled
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t o = sw128(rb[i], cb[i]);
        if (BSPLIT) {
          sts128(hs + 2 * kTileBytes + o, vb[i]);
          sts128(hs + 3 * kTileBytes + o, vl[i]);
        } else {
          const float4 h = tf32_hi(vb[i]);
          sts128(hs + 2 * kTileBytes + o, h);
          sts128(hs + 3 * kTileBytes + o, make_float4(vb[i].x - h.x, vb[i].y - h.y, vb[i].z - h.z, vb[i].w - h.w));
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
    consumers_sync();
    const uint64_t da_hi = desc_k_sw128(hs + wgi * 64 * 128), da_lo = desc_k_sw128(hs + kTileBytes + wgi * 64 * 128);
    const uint64_t db_hi = desc_k_sw128(hs + 2 * kTileBytes), db_lo = desc_k_sw128(hs + 3 * kTileBytes);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int k = 0; k < kBK / 8; ++k) {
      const uint64_t adv = static_cast<uint64_t>((k * 8 * 4) >> 4);   // +32 B per K step inside the 128 B row
      wgmma_m64n128k8_tf32(cor, da_lo + adv, db_hi + adv);
      wgmma_m64n128k8_tf32(cor, da_hi + adv, db_lo + adv);
      wgmma_m64n128k8_tf32(acc, da_hi + adv, db_hi + adv);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
    consumers_sync();                                      // the MMAs of block kb - 1 (both warpgroups) are complete:
                                                           // its hi/lo buffer may be rewritten
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");

  // -------------------------------------------------------------------- epilogue
  // fragment i of this thread: rows r0 and r0 + 8, columns n0 + 8 (i / 4) + 2 (lane % 4) + {0, 1}
  const int wl = warp & 3;
  const long long r0 = static_cast<long long>(m_blk) * kBM + wgi * 64 + wl * 16 + (lane >> 2);
  float* cbase = p.C + static_cast<long long>(split) * p.M * kN;
  const bool has_bias = p.bias != nullptr;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = n0 + j * 8 + 2 * (lane & 3);
    float2 b = make_float2(0.f, 0.f);
    if (has_bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long row = r0 + 8 * h;
      float2 v = make_float2(acc[4 * j + 2 * h] + cor[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + cor[4 * j + 2 * h + 1]);
      if (has_bias) {   // fused Linear epilogue: z + b, then the activation (same op order as bias_act_fwd_kernel)
        v.x += b.x; v.y += b.y;
        if (p.act == 1) {
          if (TANH_MUFU) { v.x = tanh_ex2(v.x); v.y = tanh_ex2(v.y); }
          else { v.x = tanhf(v.x); v.y = tanhf(v.y); }
        } else if (p.act == 2) {
          v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f);
        }
      }
      if (row < p.M) *reinterpret_cast<float2*>(cbase + row * kN + col) = v;
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode() {
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

// (rows x cols) fp32 row-major operand, unswizzled boxes of one 128 x 32 tile: K-major (cols = K): 32 contiguous
// elements x 128 rows; M/N-major (rows = K): 128 contiguous elements x 32 reduction rows.  Out-of-range rows are
// filled with zeros (ragged M).
inline bool make_map(CUtensorMap* map, const float* base, uint64_t rows, uint64_t cols, bool mn_major) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return false;
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {cols * sizeof(float)};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(mn_major ? 128 : kBK), static_cast<cuuint32_t>(mn_major ? kBK : 128)};
  const cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// grid: (ceil(M / 128), 2, splits); p.C is the split-K workspace when splits > 1
template <bool AMN, bool BMN, bool BSPLIT, bool TANH_MUFU>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mb2, const Params& p, unsigned splits,
           cudaStream_t st, const char* what) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm3_wgmma_kernel<AMN, BMN, BSPLIT, TANH_MUFU>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
    attr_set = true;
  }
  const dim3 grid(static_cast<unsigned>(ceil_div<long long>(p.M, kBM)), kN / kBN, splits);
  gemm3_wgmma_kernel<AMN, BMN, BSPLIT, TANH_MUFU><<<grid, kThreads, kSmemBytes, st>>>(ma, mb, mb2, p);
  return check_launch(what);
}

}  // namespace wg
}  // namespace trl
