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
// One CTA per 128 x 128 output tile and K slab (gridDim = (M tiles, 2 column halves, splits)), 384 threads:
//   warps 8..11  producer     : one thread issues cp.async.bulk.tensor 2D loads of one K block (32 deep) per ring stage, mbarrier
//                               complete_tx.  K-major operands arrive SWIZZLE_128B, i.e. already in the canonical
//                               layout the wgmma B descriptor reads (16-byte chunk c of row r at chunk c ^ (r & 7)).
//   warps 0..7   two consumer warpgroups.  Per K block:
//                  A: each thread loads its m64k8 register fragments straight from the TMA tile, splits them with
//                     cvt.rna in registers and issues the register-A form of wgmma (no A planes in shared memory);
//                  B: pre-split K-major planes (the forward) are read by the MMAs where TMA put them.  Every other B
//                     is converted once by the consumers into the stage's hi / lo planes -- raw K-major: split in
//                     place; N-major (dgrad, wgrad): transposed, since wgmma takes tf32 operands from shared memory
//                     only K-major -- and handed to both warpgroups through an mbarrier;
//                  warpgroup w issues the 12 wgmma of its 64 rows into two register accumulators (see above), waits
//                  for them and releases the stage to the producer.  The ring is 2-4 stages deep (as many as fit), so
//                  TMA runs ahead of the MMAs and the two warpgroups drift against each other without a CTA barrier.
//   epilogue                  accumulator fragments -> bias / activation -> global (float2 per thread, 32-byte rows).
//   CLUSTER (split-K wgrad):  the splits are summed inside the launch instead (see the epilogue below).
//   XK > 0 (dgrad dH1 = gz2 W2 of a first layer with XK inputs): dH1 is never stored; the epilogue reduces it to the
//                             first layer's weight / bias gradient slab partials (see there).
// Shapes (template flags):
//   AMN = false: A (M x K) row-major;  AMN = true: A (K x M) row-major (reduction index = row index)
//   BMN = false: B (256 x K) row-major; BMN = true: B (K x 256) row-major
//   BSPLIT: B arrives as two pre-split planes (hi = tf32(w), lo = w - hi) and is only re-laid out, not split.
#pragma once
#include "common.cuh"
#include "reduce.cuh"
#include "skinny_common.cuh"
#include <cuda.h>

namespace trl {
namespace wg {

constexpr int kBM = 128, kBN = 128, kN = 256, kBK = 32;
constexpr int kTileBytes = 128 * kBK * 4;                 // 16 KB: one 128 x 32 fp32 tile
constexpr int kConsumers = 256;                           // two warpgroups
constexpr int kThreads = kConsumers + 128;                // + producer warpgroup (one TMA thread)
// Registers per thread: 168 at launch (__launch_bounds__(384, 1)); the producer warpgroup drops to 40 and the consumers
// take 232 (8 x 32 x 232 + 4 x 32 x 40 <= 64 K), which holds both accumulators and the A fragments of a K block.
constexpr int kProducerRegs = 40, kConsumerRegs = 232;

// Ring stage: A | B hi | B lo [| raw N-major B | raw N-major B lo plane].  The stage count fills ~200 KB.
// XK > 0: a 128 x 128 tile of the first layer's activations h1 and the CTA's rows of its input x ([128][KP]) follow the
// ring, and the ring gives up its fourth stage for them (227 KB in all; the dgrad has only 8 K blocks).
template <bool BMN, bool BSPLIT, int XK = 0>
struct Ring {
  static constexpr int kTiles = 3 + (BMN ? (BSPLIT ? 2 : 1) : 0);
  static constexpr int kStageBytes = kTiles * kTileBytes;
  static constexpr int kYBytes = XK ? kBM * kBN * 4 : 0;
  static constexpr int kXBytes = XK ? kBM * ((XK + 3) & ~3) * 4 : 0;
  static constexpr int kStages = XK ? 3 : ((200 * 1024) / kStageBytes < 4 ? (200 * 1024) / kStageBytes : 4);
  static constexpr int kSmemBytes = kStages * kStageBytes + kYBytes + kXBytes + 1024 /*align*/ + 128 /*barriers*/;
  static constexpr bool kConvertB = BMN || !BSPLIT;       // the consumers write the B planes
  static_assert(kStages >= 2 && kSmemBytes <= 227 * 1024, "fits one sm_90 CTA");
};

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

// d[64] += A(64 x 8) . B(128 x 8)^T, A from registers (this thread's m64k8 tf32 fragment: rows gid, gid + 8 of its
// warp's 16, k = tid, tid + 4 as a = {(gid, tid), (gid + 8, tid), (gid, tid + 4), (gid + 8, tid + 4)}), B K-major in
// shared memory, fp32 accumulate (one warpgroup)
__device__ __forceinline__ void wgmma_m64n128k8_tf32_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
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
// Thread-block cluster: this CTA's rank, the cluster's size, the split barrier (arrive releases this thread's shared
// memory writes, wait acquires every thread's) and a 16-byte load from the same offset of rank r's shared memory.
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_size() {
  uint32_t n;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
  return n;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ float4 ld_cluster128(uint32_t addr, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(addr), "r"(rank));
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(remote)
               : "memory");
  return v;
}
__device__ __forceinline__ uint32_t tf32_bits(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return u;
}
__device__ __forceinline__ float4 tf32_hi(const float4 v) {
  return make_float4(__uint_as_float(tf32_bits(v.x)), __uint_as_float(tf32_bits(v.y)), __uint_as_float(tf32_bits(v.z)),
                     __uint_as_float(tf32_bits(v.w)));
}
__device__ __forceinline__ float4 sub4(const float4 a, const float4 b) {
  return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}

// float4 unit u (0..1023) of a raw M/N-major 128 x 32 tile as TMA delivered it (32 reduction rows x 128): its row of
// the K-major destination and its 16-byte chunk (4 reduction indices)
__device__ __forceinline__ float4 load_unit_mn(uint32_t raw, int u, int& row, int& chunk) {
  row = u & 127; chunk = u >> 7;
  const uint32_t a = raw + static_cast<uint32_t>(chunk * 4 * 128 + row) * 4u;
  return make_float4(lds32(a), lds32(a + 512u), lds32(a + 1024u), lds32(a + 1536u));
}
__device__ __forceinline__ uint32_t sw128(int row, int chunk) {
  return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}

// Byte offset of A element (m, k) of the block in its stage slot.
//   K-major A: one 32 x 128 box, SWIZZLE_128B.  A warp's fragment load (fixed k chunk, rows gid = 0..7, k & 3 = tid)
//     hits chunk c ^ gid, word tid: 32 distinct banks.
//   M-major A: four 32 (m) x 32 (k) boxes, SWIZZLE_128B: row k holds 32 m.  A warp's load (m = 16 w + gid + 8 h, k =
//     tid + 4 c) hits chunk ((m & 31) >> 2) ^ (k & 7), word m & 3: (gid >> 2, tid) = (0, 1) and (1, 0) share a chunk, so
//     2 wavefronts, 16 distinct banks.
template <bool AMN>
__device__ __forceinline__ uint32_t a_offset(int m, int k) {
  if (!AMN) return static_cast<uint32_t>(m * 128 + ((((k >> 2) ^ (m & 7))) << 4) + (k & 3) * 4);
  return static_cast<uint32_t>((m >> 5) * 4096 + k * 128 + ((((m & 31) >> 2) ^ (k & 7)) << 4) + (m & 3) * 4);
}

struct Params {
  const float* __restrict__ bias;  // (256) added in the epilogue, or nullptr
  int act;                         // 0 none, 1 tanh, 2 relu (after the bias)
  float* __restrict__ C;           // (splits, M, 256) when splits > 1 else (M, 256)
  long long M;                     // output rows
  int k_blocks_per_split;          // K blocks (of 32) accumulated by one CTA
  float* __restrict__ ws;          // CLUSTER: (8, M, 256) group partials
  unsigned* tickets;               // CLUSTER: M / 8 arrival counters (8 row slices per 128 x 128 tile), zero on entry
  const float* __restrict__ X;     // XK: the first layer's input (M, XK)
  int wg_rows;                     // XK: rows per consumer warpgroup, a whole number of slabs (<= 64)
  int slab_rows;                   // XK: rows per slab, sk_rows_per_cta(M)
};

// CLUSTER epilogue, shared memory: the CTA's 128 x 128 tile (acc + cor), rows padded so that a warp's float2 fragment
// stores take 2 wavefronts.  It lives in the (then idle) ring.
constexpr int kTileLd = kBN + 8;

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// TANH_MUFU: tanh as tanh_ex2 (common.cuh, |abs err| < 2.5e-7) instead of libdevice tanhf.
// CLUSTER: split-K (splits = 8 c) summed inside the launch, in the order of pair_splitk_reduce_kernel (csrc/gemm_pair.cu:
// group g = 0..7 adds splits g, g + 8, ... to 0 in turn, then the 8 group sums are combined as a balanced tree).
// Launched in clusters of c CTAs along z; rank j of cluster g owns split g + 8 j.  After the main loop every CTA puts
// its tile into its ring, rank j adds row slice j of the c tiles in rank order through distributed shared memory and
// stores the group-g partial to p.ws; the last of the 8 CTAs holding slice j of a tile (last_cta) adds the 8 group
// partials and writes C.  No bias / activation.
// XK > 0: the dgrad dH1 = gz2 W2 (K-major pre-split planes) of an MLP whose first layer h1 = act(x W1^T + b1) has XK
// inputs; instead of dH1 the launch writes the slab partials of skinny_tn_kernel<XK, true> (csrc/skinny.cu) for
// dW1 = (dH1 * act'(h1))^T x and db1, bit for bit.  The tile rows follow the slabs (sk_rows_per_cta rows each): each
// warpgroup owns p.wg_rows rows, a whole number of slabs, so a CTA covers 2 p.wg_rows <= 128 rows (the rows of its
// m64 MMAs past p.wg_rows are computed and dropped).  The producer warpgroup TMA-loads the tile's h1 rows (map_y) and
// stages the tile's x rows while the main loop runs; after the last MMA the tile goes into the idle ring and each
// warpgroup re-reads it in the skinny kernel's row-lane order (skinny_common.cuh).  No bias / activation.
template <bool AMN, bool BMN, bool BSPLIT, bool TANH_MUFU, bool CLUSTER = false, int XK = 0>
__global__ void __launch_bounds__(kThreads, 1)
gemm3_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                   const __grid_constant__ CUtensorMap map_b2, const __grid_constant__ CUtensorMap map_y, const Params p) {
  static_assert(XK == 0 || (!AMN && !BMN && BSPLIT && !CLUSTER), "the first-layer epilogue is a K-major pre-split dgrad");
  using R = Ring<BMN, BSPLIT, XK>;
  constexpr int XKP = (XK + 3) & ~3;
  constexpr int S = R::kStages;
  constexpr int kA = 0, kBhi = kTileBytes, kBlo = 2 * kTileBytes, kBraw = 3 * kTileBytes, kBraw2 = 4 * kTileBytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  float* ytile = reinterpret_cast<float*>(ring + S * R::kStageBytes);   // XK: [128][128] h1 rows
  float* xs = reinterpret_cast<float*>(ring + S * R::kStageBytes + R::kYBytes);   // XK: [128][XKP] x rows
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + S * R::kStageBytes + R::kYBytes + R::kXBytes);
  uint64_t* full = bars;                                   // [S] TMA -> consumers
  uint64_t* empty = bars + S;                              // [S] consumers' MMAs done -> TMA
  uint64_t* conv = bars + 2 * S;                           // [S] B planes written -> both warpgroups (kConvertB)
  uint64_t* ybar = bars + 3 * S;                           // XK: h1 tile landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, n0 = blockIdx.y * kBN;
  const int c_size = CLUSTER ? static_cast<int>(cluster_size()) : 1, c_rank = CLUSTER ? static_cast<int>(cluster_rank()) : 0;
  const int split = CLUSTER ? static_cast<int>(blockIdx.z) / c_size + 8 * c_rank : static_cast<int>(blockIdx.z);
  const int nkb = p.k_blocks_per_split;
  const int kb0 = split * nkb;
  const int m_row0 = XK ? m_blk * 2 * p.wg_rows : m_blk * kBM;   // first row of the A box

  if (threadIdx.x == kConsumers) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b)) : "memory");
    if (BSPLIT) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b2)) : "memory");
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumers / 32);               // one arrival per consumer warp
      mbar_init(&conv[s], kConsumers / 32);
    }
    if (XK) mbar_init(ybar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kConsumers / 32) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == kConsumers / 32 && lane == 0) {
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % S;
        const uint32_t ph = (kb / S) & 1;
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = ring + s * R::kStageBytes;
        mbar_arrive_expect_tx(&full[s], (BSPLIT ? 3 : 2) * kTileBytes);
        const int k0 = (kb0 + kb) * kBK;
        if (AMN) {
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_load_2d(st + kA + j * 4096, &map_a, &full[s], m_blk * kBM + 32 * j, k0);
        } else {
          tma_load_2d(st + kA, &map_a, &full[s], k0, m_row0);
        }
        if (BMN) {
          tma_load_2d(st + kBraw, &map_b, &full[s], n0, k0);
          if (BSPLIT) tma_load_2d(st + kBraw2, &map_b2, &full[s], n0, k0);
        } else {
          tma_load_2d(st + kBhi, &map_b, &full[s], k0, n0);
          if (BSPLIT) tma_load_2d(st + kBlo, &map_b2, &full[s], k0, n0);
        }
        if (XK && kb == (nkb < S ? nkb : S) - 1) {       // behind the ring's first fill: the h1 rows of the tile
          mbar_arrive_expect_tx(ybar, R::kYBytes);
          tma_load_2d(ytile, &map_y, ybar, n0, m_row0);
        }
      }
    }
    if constexpr (XK > 0) {
      // warps 9..11 stage the tile's x rows for the epilogue, then signal the consumers (named barrier 1)
      if (warp > kConsumers / 32) {
        const long long nx = p.M - m_row0;
        stage_rows<XK>(xs, p.X, m_row0, static_cast<int>(nx < 2 * p.wg_rows ? nx : 2 * p.wg_rows),
                       threadIdx.x - kConsumers - 32, 96);
        named_arrive(1, kConsumers + 96);
      }
    }
    if constexpr (CLUSTER) {
      // the producer warps pass every CTA and cluster barrier of the consumers' epilogue (same order, see there):
      // no thread of a cluster exits while a peer may still read its shared memory
      __syncwarp();
      __syncthreads();
      cluster_arrive();
      cluster_wait();
      cluster_arrive();
      last_cta(p.tickets + (m_blk * 2 + blockIdx.y) * 8 + c_rank, 8u);
      cluster_wait();
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
  const int ct = threadIdx.x, wgi = warp >> 2, wl = warp & 3;
  const int gid = lane >> 2, tid = lane & 3;
  const int am = (XK ? wgi * p.wg_rows : wgi * 64) + wl * 16 + gid;   // this thread's fragment rows: am, am + 8
  float acc[64], cor[64];                                  // hi*hi | lo*hi + hi*lo
#pragma unroll
  for (int i = 0; i < 64; ++i) { acc[i] = 0.f; cor[i] = 0.f; }
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % S;
    const uint32_t ph = (kb / S) & 1;
    const uint32_t st = smem_u32(ring + s * R::kStageBytes);
    mbar_wait(&full[s], ph);
    if (R::kConvertB) {
      // all loads of this thread first (independent accesses in flight), then split / re-lay out and store
      float4 vb[4], vl[4];
      int rb[4], cb[4];
      if (BMN) {
#pragma unroll
        for (int i = 0; i < 4; ++i) vb[i] = load_unit_mn(st + kBraw, ct + i * kConsumers, rb[i], cb[i]);
        if (BSPLIT) {
#pragma unroll
          for (int i = 0; i < 4; ++i) vl[i] = load_unit_mn(st + kBraw2, ct + i * kConsumers, rb[i], cb[i]);
        }
      } else {                                             // raw K-major B, already swizzled: split in place
#pragma unroll
        for (int i = 0; i < 4; ++i) vb[i] = lds128(st + kBhi + static_cast<uint32_t>(ct + i * kConsumers) * 16u);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t o = BMN ? sw128(rb[i], cb[i]) : static_cast<uint32_t>(ct + i * kConsumers) * 16u;
        if (BSPLIT) {
          sts128(st + kBhi + o, vb[i]);
          sts128(st + kBlo + o, vl[i]);
        } else {
          const float4 h = tf32_hi(vb[i]);
          sts128(st + kBhi + o, h);
          sts128(st + kBlo + o, sub4(vb[i], h));
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
      __syncwarp();
      if (lane == 0) mbar_arrive(&conv[s]);
    }
    // A fragments of the 4 K steps, split in registers
    uint32_t ahi[kBK / 8][4], alo[kBK / 8][4];
    {
      float av[kBK / 8][4];
#pragma unroll
      for (int k = 0; k < kBK / 8; ++k)
#pragma unroll
        for (int r = 0; r < 4; ++r) av[k][r] = lds32(st + kA + a_offset<AMN>(am + 8 * (r & 1), 8 * k + tid + 4 * (r >> 1)));
#pragma unroll
      for (int k = 0; k < kBK / 8; ++k)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          ahi[k][r] = tf32_bits(av[k][r]);
          alo[k][r] = __float_as_uint(av[k][r] - __uint_as_float(ahi[k][r]));
        }
    }
    if (R::kConvertB) mbar_wait(&conv[s], ph);
    const uint64_t db_hi = desc_k_sw128(st + kBhi), db_lo = desc_k_sw128(st + kBlo);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int k = 0; k < kBK / 8; ++k) {
      const uint64_t adv = static_cast<uint64_t>((k * 8 * 4) >> 4);   // +32 B per K step inside the 128 B row
      wgmma_m64n128k8_tf32_rs(cor, alo[k], db_hi + adv);
      wgmma_m64n128k8_tf32_rs(cor, ahi[k], db_lo + adv);
      wgmma_m64n128k8_tf32_rs(acc, ahi[k], db_hi + adv);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);                 // this warp is done with stage s
  }

  // -------------------------------------------------------------------- epilogue
  // fragment i of this thread: rows r0 and r0 + 8, columns n0 + 8 (i / 4) + 2 (lane % 4) + {0, 1}
  if constexpr (XK > 0) {
    named_sync(2, kConsumers);                              // every consumer warp is past its last MMA: the ring is idle
    // the warpgroup's 64 fragment rows (acc + cor: the value the plain dgrad stores) at rows 64 wgi + 0..63
    float* tile = reinterpret_cast<float*>(ring);
    const int lr = wgi * 64 + wl * 16 + gid;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(tile + (lr + 8 * h) * kTileLd + j * 8 + 2 * tid) =
            make_float2(acc[4 * j + 2 * h] + cor[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + cor[4 * j + 2 * h + 1]);
    named_sync(1, kConsumers + 96);                         // the tile and the x rows are in shared memory
    mbar_wait(ybar, 0);                                     // so are the h1 rows
    // skinny_tn_kernel's layout over the warpgroup's 128 columns: warp wl owns 32, lane = (row lane, column quad)
    const int rl = lane >> 3, cc = wl * 32 + (lane & 7) * 4;
    const int spw = p.wg_rows / p.slab_rows;
    const uint32_t g_u32 = smem_u32(tile + (wgi * 64) * kTileLd + cc), y_u32 = smem_u32(ytile + cc);
    for (int sl = 0; sl < spw; ++sl) {
      const long long slab = static_cast<long long>(m_blk * 2 + wgi) * spw + sl;
      const long long row0 = slab * p.slab_rows;
      if (row0 >= p.M) break;
      const int nrows = static_cast<int>(p.M - row0 < p.slab_rows ? p.M - row0 : p.slab_rows);
      const int gr0 = sl * p.slab_rows, br0 = wgi * p.wg_rows + sl * p.slab_rows;   // slab row 0 in the tile / box
      float wacc[XKP][4];
#pragma unroll
      for (int k = 0; k < XKP; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) wacc[k][j] = 0.f;
      float4 asum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
      for (int r = rl; r < nrows; r += 4) {
        const float4 g = lds128(g_u32 + static_cast<uint32_t>((gr0 + r) * kTileLd) * 4u);
        const float4 y = lds128(y_u32 + static_cast<uint32_t>((br0 + r) * kBN) * 4u);
        act_wgrad_row<XK>(wacc, asum, g, y, xs + (br0 + r) * XKP, p.act);
      }
      act_wgrad_store<XK>(p.ws + slab * (XK + 1) * kN, wacc, asum, kN, n0 + cc, rl);
    }
    return;
  }
  if constexpr (CLUSTER) {
    __syncthreads();                                        // every warp is past its last MMA: the ring is idle
    float* tile = reinterpret_cast<float*>(ring);
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(tile + (am + 8 * h) * kTileLd + j * 8 + 2 * tid) =
            make_float2(acc[4 * j + 2 * h] + cor[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + cor[4 * j + 2 * h + 1]);
    cluster_arrive();
    cluster_wait();                                         // every tile of the cluster is in shared memory
    // row slice c_rank (of c_size, as even as 128 rows allow), 32 float4 per row
    const int r_lo = c_rank * kBM / c_size, n_vec = ((c_rank + 1) * kBM / c_size - r_lo) * (kBN / 4);
    const long long slab = p.M * kN;
    const uint32_t tile_u32 = smem_u32(tile);
    for (int v = ct; v < n_vec; v += kConsumers) {
      const int r = r_lo + v / (kBN / 4), q4 = v % (kBN / 4);
      const uint32_t a = tile_u32 + static_cast<uint32_t>(r * kTileLd + 4 * q4) * 4u;
      float4 x[8];
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (q < c_size) x[q] = ld_cluster128(a, static_cast<uint32_t>(q));
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (q < c_size) { s.x += x[q].x; s.y += x[q].y; s.z += x[q].z; s.w += x[q].w; }
      const long long o = (static_cast<long long>(m_blk) * kBM + r) * kN + n0 + 4 * q4;
      *reinterpret_cast<float4*>(p.ws + (static_cast<long long>(blockIdx.z) / c_size) * slab + o) = s;
    }
    cluster_arrive();                                       // done with the peers' shared memory
    if (last_cta(p.tickets + (m_blk * 2 + blockIdx.y) * 8 + c_rank, 8u)) {
      for (int v = ct; v < n_vec; v += kConsumers) {
        const long long o = (static_cast<long long>(m_blk) * kBM + r_lo + v / (kBN / 4)) * kN + n0 + 4 * (v % (kBN / 4));
        float4 t[8];
#pragma unroll
        for (int g = 0; g < 8; ++g) t[g] = __ldcg(reinterpret_cast<const float4*>(p.ws + g * slab + o));
#define TRL_T3(c) (((t[0].c + t[1].c) + (t[2].c + t[3].c)) + ((t[4].c + t[5].c) + (t[6].c + t[7].c)))
        *reinterpret_cast<float4*>(p.C + o) = make_float4(TRL_T3(x), TRL_T3(y), TRL_T3(z), TRL_T3(w));
#undef TRL_T3
      }
    }
    cluster_wait();                                         // nobody in the cluster reads this CTA's tile any more
    return;
  }
  const long long r0 = static_cast<long long>(m_blk) * kBM + am;
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

// How an operand's 128 x 32 tile is boxed:
//   kKMajor  : reduction index = column.  One 32 x 128 box, SWIZZLE_128B (the wgmma K-major layout).
//   kMNMajor : reduction index = row.  One 128 x 32 box, no swizzle (transposed by the consumers).
//   kMNMajorA: reduction index = row.  32 x 32 boxes (four per tile), SWIZZLE_128B (the register-A fragment loads).
//   kTile    : a whole 128 x 128 output tile, no swizzle (XK: the h1 rows read by the epilogue).
enum class Box { kKMajor, kMNMajor, kMNMajorA, kTile };

// (rows x cols) fp32 row-major operand.  Out-of-range rows are filled with zeros (ragged M).
inline bool make_map(CUtensorMap* map, const float* base, uint64_t rows, uint64_t cols, Box box_kind) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return false;
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {cols * sizeof(float)};
  const bool plain = box_kind == Box::kMNMajor || box_kind == Box::kTile;
  const cuuint32_t inner = plain ? 128 : kBK;
  const cuuint32_t box[2] = {inner, static_cast<cuuint32_t>(box_kind == Box::kKMajor || box_kind == Box::kTile ? 128 : kBK)};
  const cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE,
             plain ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// grid: (ceil(M / 128), 2, splits) (XK: ceil(M / (2 p.wg_rows)) row blocks); p.C is the split-K workspace when splits > 1 (CLUSTER: clusters of splits / 8
// CTAs along z, p.C the sum)
template <bool AMN, bool BMN, bool BSPLIT, bool TANH_MUFU, bool CLUSTER = false, int XK = 0>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mb2, const Params& p, unsigned splits,
           cudaStream_t st, const char* what, const CUtensorMap* my = nullptr) {
  constexpr int kSmem = Ring<BMN, BSPLIT, XK>::kSmemBytes;
  auto kernel = gemm3_wgmma_kernel<AMN, BMN, BSPLIT, TANH_MUFU, CLUSTER, XK>;
  const CUtensorMap& mys = my ? *my : mb2;                  // map_y is read by the XK instances only
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
    attr_set = true;
  }
  const dim3 grid(static_cast<unsigned>(ceil_div<long long>(p.M, XK ? 2 * p.wg_rows : kBM)), kN / kBN, splits);
  if constexpr (CLUSTER) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = splits / 8;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, ma, mb, mb2, mys, p);
    if (e != cudaSuccess) { set_error("%s: %s", what, cudaGetErrorString(e)); return static_cast<int>(e); }
  } else {
    kernel<<<grid, kThreads, kSmem, st>>>(ma, mb, mb2, mys, p);
  }
  return check_launch(what);
}

}  // namespace wg
}  // namespace trl
