// skinny.cu -- the "skinny" Linear layers of the small MLPs: first layer (K = obs_dim, e.g. 17 -> 256) and
// output layer (256 -> act_dim / 1).  K3/K8 support (networks/base.py:24-44, networks/nets.py:13-52).
//
// These products have one tiny dimension: each streams ONE big (M x H) activation matrix (16.8 MB at M = 16384,
// H = 256 => ~3 us at HBM speed) and a few KB of everything else; cuBLAS serves them with generic sgemm / gemv
// kernels at 9-14 us each.  Four HBM-bound fp32 kernels, one pass over the big matrix each, sharing one scheme:
//   * the CTA owns a slab of rows; the skinny operand of the slab is staged in shared memory, zero-padded to a
//     multiple of 4 columns so it is read back with broadcast LDS.128;
//   * the weights a thread needs live in REGISTERS for the whole slab (no per-FMA shared-memory traffic);
//   * the big matrix moves as float4, several independent 16-byte accesses in flight per thread.
//   skinny_k_fwd   : Y (M,H)  = act(X (M,K) . W (H,K)^T + b)                    K <= 24, H % 4 == 0, H <= 1024
//   skinny_tn      : Out (H,K) = A (M,H)^T . B (M,K)  [+ column sums of B]       K <= 24, H % 32 == 0, H <= 256
//   skinny_n_fwd   : Y (M,N)  = X (M,H) . W (N,H)^T + b                          N <= 8, H in {128, 256}
//   skinny_n_dgrad : dX (M,H) = G (M,N) . W (N,H)                                N <= 8, H % 4 == 0, H <= 1024
// and three backward fusions that remove a whole pass over the (M x H) matrix each:
//   skinny_act_wgrad   : dW1 = (G * act'(Y))^T X,  db1 = colsum(G * act'(Y))    (first layer: gz never stored)
//   skinny_n_dgrad_act : gz = (G . W) * act'(Y),  db = colsum(gz)               (output-layer dgrad + act backward)
//   skinny_n_dgrad_act_wgrad : the above and dW = G^T Y, db_out = colsum(G)     (H = 256: the output layer's whole
//                        backward in one pass over Y; skinny_tn's slab partials bit for bit)
// Reductions have a fixed combination order (deterministic, run-to-run bit-identical).
#include "skinny_common.cuh"

namespace trl {

__device__ __forceinline__ float sk_tanh(float x) { return tanh_ex2(x); }   // common.cuh: 2 MUFU ops, abs err < 2.5e-7

// activation of four values; `act` is uniform, so this is one branch per float4
__device__ __forceinline__ float4 sk_act4(float4 v, int act) {
  if (act == 1) return make_float4(sk_tanh(v.x), sk_tanh(v.y), sk_tanh(v.z), sk_tanh(v.w));
  if (act == 2) return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
  return v;
}

// run-time K (the <= 8 wide output-layer gradient): [nrows][KP], zero padded
template <int KP>
__device__ __forceinline__ void stage_rows_rt(float* __restrict__ dst, const float* __restrict__ src, long long row0,
                                              int nrows, int K, int tid, int nthr) {
  for (int i = tid; i < nrows * KP; i += nthr) {
    const int r = i / KP, k = i - r * KP;
    dst[i] = (k < K) ? __ldg(src + (row0 + r) * K + k) : 0.f;
  }
}

// acc[j] += a_j * b[k] for the K real columns of a staged row (KP/4 broadcast LDS.128; the padding is never multiplied)
#define TRL_SK_FMA4(ACC, S, WK)                                                          \
  ACC.x = fmaf(S, WK[0], ACC.x); ACC.y = fmaf(S, WK[1], ACC.y);                          \
  ACC.z = fmaf(S, WK[2], ACC.z); ACC.w = fmaf(S, WK[3], ACC.w)

// ------------------------------------------------------------------------------------------------- skinny_k_fwd
// thread = (column group of 4, row lane); W[k][4 cols] in registers for the K real columns (K is a template
// parameter: no multiply-adds on padding); per row: KP/4 broadcast LDS.128, 4*K FMA, activation, one 16-byte store
// (a warp writes 512 contiguous bytes).
// W (H x K, K odd in general) reaches the registers through shared memory: one coalesced pass over W writes it
// TRANSPOSED ([K][H + 4]), and each thread then fetches its 4 columns of every k with one conflict-free LDS.128.
// (Reading W[4cg + j][k] straight from global memory costs 4*K scalar loads per thread, each touching 32 different
// sectors per warp: ncu showed that preamble -- lg_throttle -- taking longer than the slab itself.)
template <int K>
__global__ void __launch_bounds__(256, 2) skinny_k_fwd_kernel(const float* __restrict__ X, const float* __restrict__ W,
                                                             const float* __restrict__ bias, float* __restrict__ Y,
                                                             long long M, int H, int act, int rows_per_cta) {
  constexpr int KP = (K + 3) & ~3;
  extern __shared__ __align__(16) float sk_smem[];
  const int tid = threadIdx.x;
  const long long row0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  if (row0 >= M) return;
  const int nrows = static_cast<int>(min(static_cast<long long>(rows_per_cta), M - row0));
  const int HS = H + 4;
  float* wt = sk_smem + rows_per_cta * KP;               // [K][HS]
  {
    int h = tid / K, k = tid - h * K;
    constexpr int dh = 256 / K, dk = 256 % K;
    for (int i = tid; i < H * K; i += 256) {
      wt[k * HS + h] = __ldg(W + i);
      h += dh; k += dk;
      if (k >= K) { k -= K; ++h; }
    }
  }
  stage_rows<K>(sk_smem, X, row0, nrows, tid, 256);
  const int cpg = H >> 2;
  const int RL = 256 / cpg;
  const bool active = tid < RL * cpg;
  const int cg = tid % cpg, rl = tid / cpg;
  __syncthreads();
  if (!active) return;
  float w[KP][4];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float4 v = *reinterpret_cast<const float4*>(wt + k * HS + 4 * cg);
    w[k][0] = v.x; w[k][1] = v.y; w[k][2] = v.z; w[k][3] = v.w;
  }
  const float4 bb = *reinterpret_cast<const float4*>(bias + 4 * cg);
  float* yp = Y + (row0 + rl) * H + 4 * cg;
  const long long ystep = static_cast<long long>(RL) * H;
  for (int r = rl; r < nrows; r += RL, yp += ystep) {
    const float4* xr = reinterpret_cast<const float4*>(sk_smem + r * KP);
    float4 acc = bb;
#pragma unroll
    for (int q = 0; q < KP / 4; ++q) {
      const float4 xv = xr[q];
      if (4 * q < K) { TRL_SK_FMA4(acc, xv.x, w[4 * q]); }
      if (4 * q + 1 < K) { TRL_SK_FMA4(acc, xv.y, w[4 * q + 1]); }
      if (4 * q + 2 < K) { TRL_SK_FMA4(acc, xv.z, w[4 * q + 2]); }
      if (4 * q + 3 < K) { TRL_SK_FMA4(acc, xv.w, w[4 * q + 3]); }
    }
    *reinterpret_cast<float4*>(yp) = sk_act4(acc, act);
  }
}

// ------------------------------------------------------------------------------------------------- skinny_tn
// Out[h][k] = sum_m A[m][h] * B[m][k].  One warp owns 32 columns of A: lane = (row lane 0..3) x (column group of 4),
// so one warp-wide LDG.128 fetches four full 128-byte row segments.  acc[K][4 cols] in registers (K is a template
// parameter); the B slab is broadcast from shared memory (16 FMA per LDS.128).  U rows per row lane are requested
// before the first is used (U 16-byte loads in flight per thread, 2U with the fused activation gradient).  After the
// slab: butterfly over the 4 row lanes, then the CTA writes its partial k-major ([K+1][H], row K = column sums of B);
// skinny_tn_reduce sums the CTAs in a fixed order.
// ACT = true: A is not read but formed on the fly as G * act'(Yact) (first-layer backward: the activation
// gradient is never written to memory) and row K of the partial receives the column sums of A (the bias gradient).
template <int K, bool ACT>
__global__ void __launch_bounds__(256, 2) skinny_tn_kernel(const float* __restrict__ A, const float* __restrict__ Yact,
                                                          const float* __restrict__ B, int want_colsum, int act,
                                                          float* __restrict__ partial, long long M, int H,
                                                          int rows_per_cta) {
  constexpr int KP = (K + 3) & ~3;
  // rows in flight per row lane: bounded by the registers left beside the K*4 accumulators (128 per thread)
  constexpr int U = ACT ? (K <= 17 ? 4 : (K <= 19 ? 2 : 1)) : (K <= 12 ? 8 : (K <= 17 ? 4 : 2));
  extern __shared__ __align__(16) float sk_smem[];
  const int tid = threadIdx.x, nthr = blockDim.x;        // blockDim.x = 32 * (H / 32)
  const long long row0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  const int nrows = static_cast<int>(min(static_cast<long long>(rows_per_cta), M - row0));   // grid never overshoots
  stage_rows<K>(sk_smem, B, row0, nrows, tid, nthr);
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  const int cg = lane & 7, rl = lane >> 3;
  const int c0 = warp * 32 + cg * 4;
  float acc[KP][4];
#pragma unroll
  for (int k = 0; k < KP; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[k][j] = 0.f;
  float4 asum = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* ap = A + row0 * H + c0;
  const float* yp = ACT ? Yact + row0 * H + c0 : nullptr;
  int r = rl;
  for (; r + 4 * (U - 1) < nrows; r += 4 * U) {
    float4 g[U], y[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      g[u] = __ldg(reinterpret_cast<const float4*>(ap + static_cast<long long>(r + 4 * u) * H));
      if (ACT) y[u] = __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r + 4 * u) * H));
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (ACT) act_wgrad_row<K>(acc, asum, g[u], y[u], sk_smem + (r + 4 * u) * KP, act);
      else tn_fma_row<K>(acc, g[u], sk_smem + (r + 4 * u) * KP);
    }
  }
  for (; r < nrows; r += 4) {
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(ap + static_cast<long long>(r) * H));
    if (ACT) act_wgrad_row<K>(acc, asum, a0, __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r) * H)),
                              sk_smem + r * KP, act);
    else tn_fma_row<K>(acc, a0, sk_smem + r * KP);
  }
  // partial layout per CTA: [K + 1][H] (k-major), after the fixed-order combine of the 4 row lanes (skinny_common.cuh)
  float* pp = partial + static_cast<long long>(blockIdx.x) * (K + 1) * H;
  if (ACT) {
    act_wgrad_store<K>(pp, acc, asum, H, c0, rl);
  } else {
    tn_combine_lanes<K>(acc);
    tn_store_rows<K>(pp, acc, H, c0, rl);
  }
  if (!ACT && tid < K) {
    float s = 0.f;
    if (want_colsum)
      for (int rr = 0; rr < nrows; ++rr) s += sk_smem[rr * KP + tid];
    pp[static_cast<long long>(K) * H + tid] = s;          // only the first K entries of row K are meaningful
  }
}

// second stage: e indexes the k-major partial ([K][H] then K column sums).  CTA = 8 elements x 32 groups (256 threads;
// 8 consecutive floats = one 32-byte sector per slab): group g sums partials g, g+32, ... with every load independent
// (a few hundred slabs => one or two rounds of L2 latency instead of a 40-deep dependent chain), then the first 8
// threads add the 32 group sums in order.  Small CTAs on purpose: inside the minibatch graph this kernel starts while
// the other network's kernels still hold most of every SM.
constexpr int kRedGroups = 32;
constexpr int kRedElems = 8;
__device__ __forceinline__ void tn_reduce_block(const float* __restrict__ partial, float* __restrict__ Out,
                                                float* __restrict__ colsum, int n_cs, int nslab, int H, int K,
                                                int out_transposed, int block, float (*red)[kRedElems + 1]) {
  const int el = threadIdx.x & (kRedElems - 1), g = threadIdx.x / kRedElems;
  const int e = block * kRedElems + el;
  const int n_main = K * H;
  const int n_all = n_main + n_cs;                       // n_cs trailing entries of row K go to colsum[]
  const long long stride = static_cast<long long>(K + 1) * H;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (e < n_all) {
    const float* pe = partial + e;
    int sl = g;
    for (; sl + 3 * kRedGroups < nslab; sl += 4 * kRedGroups) {
      const float v0 = __ldcg(pe + static_cast<long long>(sl) * stride);
      const float v1 = __ldcg(pe + static_cast<long long>(sl + kRedGroups) * stride);
      const float v2 = __ldcg(pe + static_cast<long long>(sl + 2 * kRedGroups) * stride);
      const float v3 = __ldcg(pe + static_cast<long long>(sl + 3 * kRedGroups) * stride);
      s0 += v0; s1 += v1; s2 += v2; s3 += v3;
    }
    for (; sl < nslab; sl += kRedGroups) s0 += __ldcg(pe + static_cast<long long>(sl) * stride);
  }
  red[g][el] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (g == 0 && e < n_all) {
    float s = red[0][el];
#pragma unroll
    for (int i = 1; i < kRedGroups; ++i) s += red[i][el];
    if (e < n_main) {
      const int k = e / H, h = e - k * H;
      if (out_transposed) Out[e] = s;                                  // Out is (K, H)
      else Out[static_cast<long long>(h) * K + k] = s;                 // Out is (H, K)
    } else {
      colsum[e - n_main] = s;
    }
  }
}

__global__ void __launch_bounds__(kRedElems * kRedGroups) skinny_tn_reduce_kernel(const float* __restrict__ partial,
                                                                                 float* __restrict__ Out,
                                                                                 float* __restrict__ colsum, int n_cs,
                                                                                 int nslab, int H, int K,
                                                                                 int out_transposed) {
  __shared__ float red[kRedGroups][kRedElems + 1];
  tn_reduce_block(partial, Out, colsum, n_cs, nslab, H, K, out_transposed, blockIdx.x, red);
}

// Several second stages in ONE launch (the slab sums of a whole backward pass: two first-layer, two output-layer weight
// gradients and two bias gradients per PPO minibatch are six launches of a few microseconds of latency each otherwise).
constexpr int kMaxRedJobs = 8;
struct ReduceJobs {
  const float* partial[kMaxRedJobs];
  float* out[kMaxRedJobs];
  float* colsum[kMaxRedJobs];
  int n_cs[kMaxRedJobs], nslab[kMaxRedJobs], H[kMaxRedJobs], K[kMaxRedJobs], out_t[kMaxRedJobs];
  int cta_begin[kMaxRedJobs + 1];
  int njobs;
};
__global__ void __launch_bounds__(kRedElems * kRedGroups) skinny_reduce_jobs_kernel(const ReduceJobs q) {
  __shared__ float red[kRedGroups][kRedElems + 1];
  int j = 0;
#pragma unroll
  for (int i = 1; i < kMaxRedJobs; ++i) j += (i < q.njobs && static_cast<int>(blockIdx.x) >= q.cta_begin[i]) ? 1 : 0;
  tn_reduce_block(q.partial[j], q.out[j], q.colsum[j], q.n_cs[j], q.nslab[j], q.H[j], q.K[j], q.out_t[j],
                  static_cast<int>(blockIdx.x) - q.cta_begin[j], red);
}

// ------------------------------------------------------------------------------------------------- skinny_n_fwd
// Y[m][n] = b[n] + sum_h X[m][h] * W[n][h].  One warp per row; lane holds W[n][its 4*HC columns] for the NB >= N
// outputs of the instantiation in registers (rows n >= N are zero; NB in {1, 2, 4, 8} so that the 1-output value head
// does not carry the registers of an 8-output policy head).  Three or four rows per iteration (that many * HC independent 16-byte loads
// per lane), two CTAs per SM.  The NB per-lane partial sums of a row are reduced with a halving butterfly (9 shuffles
// instead of 40 at NB = 8): each halving stage exchanges half of the live values across one lane bit.
template <int NB>
__device__ __forceinline__ float nb_butterfly(float (&v)[NB], int lane) {
  int off = 16;
#pragma unroll
  for (int cnt = NB; cnt > 1; cnt >>= 1) {
    const int half = cnt >> 1;
    const bool hi = lane & off;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = hi ? v[i] : v[i + half];
      const float keep = hi ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
    off >>= 1;
  }
  for (; off > 0; off >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
  return v[0];       // every lane holds the total of output nb_out_index<NB>(lane)
}
template <int NB>
__device__ __forceinline__ int nb_out_index(int lane) {
  int n = 0, off = 16;
#pragma unroll
  for (int cnt = NB; cnt > 1; cnt >>= 1) {
    if (lane & off) n += cnt >> 1;
    off >>= 1;
  }
  return n;
}

template <int HC, int NB>
__global__ void __launch_bounds__(256, 2) skinny_n_fwd_kernel(const float* __restrict__ X, const float* __restrict__ W,
                                                             const float* __restrict__ bias, float* __restrict__ Y,
                                                             long long M, int H, int N) {
  const int lane = threadIdx.x & 31;
  const long long gw = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const long long nw = static_cast<long long>(gridDim.x) * 8;
  float4 w[NB][HC];
#pragma unroll
  for (int n = 0; n < NB; ++n)
#pragma unroll
    for (int c = 0; c < HC; ++c)
      w[n][c] = (n < N) ? *reinterpret_cast<const float4*>(W + static_cast<long long>(n) * H + c * 128 + lane * 4)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
  const int n_out = nb_out_index<NB>(lane);
  const bool writer = (lane & (32 / NB - 1)) == 0 && n_out < N;
  const float b_out = (n_out < N) ? bias[n_out] : 0.f;
  constexpr int R = (NB == 8 && HC == 2) ? 3 : 4;          // rows per iteration: what fits in 128 registers beside W
  for (long long m0 = gw * R; m0 < M; m0 += nw * R) {
    float4 x[R][HC];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int c = 0; c < HC; ++c)
        x[i][c] = (m0 + i < M) ? __ldg(reinterpret_cast<const float4*>(X + (m0 + i) * H + c * 128 + lane * 4))
                               : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < R; ++i) {
      float v[NB];
#pragma unroll
      for (int n = 0; n < NB; ++n) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < HC; ++c)
          s = fmaf(x[i][c].x, w[n][c].x, fmaf(x[i][c].y, w[n][c].y, fmaf(x[i][c].z, w[n][c].z, fmaf(x[i][c].w, w[n][c].w, s))));
        v[n] = s;
      }
      const float tot = nb_butterfly<NB>(v, lane);
      if (writer && m0 + i < M) Y[(m0 + i) * N + n_out] = tot + b_out;
    }
  }
}

// ------------------------------------------------------------------------------------------------- skinny_n_dgrad
// dX[m][h] = sum_n G[m][n] * W[n][h].  thread = (column group of 4, row lane), W[n][4 cols] in registers, the G slab
// ([rows][8], zero padded) broadcast from shared memory: 2 LDS.128 + 32 FMA + one 16-byte store per row.
// ACT = true: the result is multiplied by act'(Yact) before it is stored (gz of the last hidden layer) and the
// per-column sums of the stored values (that layer's bias gradient) go to colpart[cta][H].
// NW > 0 (with ACT, H = 256, N = NW): the same pass also forms the output layer's weight / bias gradient slab partial
// of skinny_tn_kernel<NW, false>(Yact, G, want_colsum = 1), bit for bit, in wpart[cta][NW + 1][H].  At H = 256 both
// kernels give a thread 4 columns and a row lane rl in 0..3 that runs rows rl, rl + 4, ... in increasing order; each
// thread feeds the Yact float4 it loaded for act'() and the staged G row to tn_fma_row<NW> (skinny_common.cuh), the
// 4 row lanes (here in different warps) are added through shared memory as (v0 + v1) + (v2 + v3), tn_combine_lanes'
// value, and row NW is the sequential sum of the slab's staged G rows.
template <bool ACT, int NW>
__global__ void __launch_bounds__(256, 2) skinny_n_dgrad_kernel(const float* __restrict__ G, const float* __restrict__ W,
                                                               const float* __restrict__ Yact, int act,
                                                               float* __restrict__ dX, float* __restrict__ colpart,
                                                               float* __restrict__ wpart, long long M, int H, int N,
                                                               int rows_per_cta) {
  static_assert(NW == 0 || (ACT && NW <= 8), "the output-layer weight gradient rides on the activation backward");
  extern __shared__ __align__(16) float sk_smem[];       // G slab [rows_per_cta][8]; NW > 0: then [3][NW][H]
  __shared__ __align__(16) float colred[1024];           // [RL][H], RL * H <= 1024
  const int tid = threadIdx.x;
  const long long row0 = static_cast<long long>(blockIdx.x) * rows_per_cta;
  const int nrows = static_cast<int>(min(static_cast<long long>(rows_per_cta), M - row0));   // grid never overshoots
  if (NW > 0) N = NW;
  const int cpg = H >> 2;
  const int RL = 256 / cpg;
  const bool active = tid < RL * cpg;
  const int cg = tid % cpg, rl = tid / cpg;
  // NW in 1..6 (registers to spare): the Yact rows go through a two-batch pipeline, the next four rows requested
  // before the current four are used, and the first four are requested before the G slab is staged, so that only
  // one load latency per CTA is exposed (a slab is 16 rows per row lane at M = 16384).  Same rows, same order.
  constexpr bool kPipe = NW > 0 && NW <= 6;
  const float* yp = ACT ? Yact + row0 * H + 4 * cg : nullptr;
  float4 ya[4], yn[4];
  auto load4 = [&](float4 (&d)[4], int r) {
#pragma unroll
    for (int u = 0; u < 4; ++u)
      d[u] = (r + u * RL < nrows) ? __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r + u * RL) * H))
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  if (kPipe) load4(ya, rl);
  stage_rows_rt<8>(sk_smem, G, row0, nrows, N, tid, 256);
  float4 w[8];
#pragma unroll
  for (int n = 0; n < 8; ++n)
    w[n] = (active && n < N) ? *reinterpret_cast<const float4*>(W + static_cast<long long>(n) * H + 4 * cg)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
  constexpr int NWA = NW > 0 ? NW : 1;
  float wacc[(NWA + 3) & ~3][4];                         // this thread's 4 columns of the NW rows of G^T Yact
  if (NW > 0) {
#pragma unroll
    for (int k = 0; k < NWA; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) wacc[k][j] = 0.f;
  }
  __syncthreads();
  float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
  auto row_out = [&](int r, float4 yv) {
    const float4 g0 = reinterpret_cast<const float4*>(sk_smem + r * 8)[0];
    const float4 g1 = reinterpret_cast<const float4*>(sk_smem + r * 8)[1];
    float4 acc;
    acc.x = g0.x * w[0].x; acc.y = g0.x * w[0].y; acc.z = g0.x * w[0].z; acc.w = g0.x * w[0].w;
    acc.x = fmaf(g0.y, w[1].x, acc.x); acc.y = fmaf(g0.y, w[1].y, acc.y); acc.z = fmaf(g0.y, w[1].z, acc.z); acc.w = fmaf(g0.y, w[1].w, acc.w);
    acc.x = fmaf(g0.z, w[2].x, acc.x); acc.y = fmaf(g0.z, w[2].y, acc.y); acc.z = fmaf(g0.z, w[2].z, acc.z); acc.w = fmaf(g0.z, w[2].w, acc.w);
    acc.x = fmaf(g0.w, w[3].x, acc.x); acc.y = fmaf(g0.w, w[3].y, acc.y); acc.z = fmaf(g0.w, w[3].z, acc.z); acc.w = fmaf(g0.w, w[3].w, acc.w);
    acc.x = fmaf(g1.x, w[4].x, acc.x); acc.y = fmaf(g1.x, w[4].y, acc.y); acc.z = fmaf(g1.x, w[4].z, acc.z); acc.w = fmaf(g1.x, w[4].w, acc.w);
    acc.x = fmaf(g1.y, w[5].x, acc.x); acc.y = fmaf(g1.y, w[5].y, acc.y); acc.z = fmaf(g1.y, w[5].z, acc.z); acc.w = fmaf(g1.y, w[5].w, acc.w);
    acc.x = fmaf(g1.z, w[6].x, acc.x); acc.y = fmaf(g1.z, w[6].y, acc.y); acc.z = fmaf(g1.z, w[6].z, acc.z); acc.w = fmaf(g1.z, w[6].w, acc.w);
    acc.x = fmaf(g1.w, w[7].x, acc.x); acc.y = fmaf(g1.w, w[7].y, acc.y); acc.z = fmaf(g1.w, w[7].z, acc.z); acc.w = fmaf(g1.w, w[7].w, acc.w);
    if (ACT) {
      if (NW > 0) tn_fma_row<NWA>(wacc, yv, sk_smem + r * 8);
      acc = sk_dact4(acc, yv, act);
      cs.x += acc.x; cs.y += acc.y; cs.z += acc.z; cs.w += acc.w;
    }
    *reinterpret_cast<float4*>(dX + (row0 + r) * H + 4 * cg) = acc;
  };
  if (active) {
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    int r = rl;
    if (kPipe) {
      for (; r < nrows; r += 4 * RL) {
        load4(yn, r + 4 * RL);
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (r + u * RL < nrows) row_out(r + u * RL, ya[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u) ya[u] = yn[u];
      }
    } else if (ACT) {
      // the activations of four rows are requested before the first one is used: four 16-byte loads in flight per
      // thread instead of one dependent load per row
      for (; r + 3 * RL < nrows; r += 4 * RL) {
        const float4 y0 = __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r) * H));
        const float4 y1 = __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r + RL) * H));
        const float4 y2 = __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r + 2 * RL) * H));
        const float4 y3 = __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r + 3 * RL) * H));
        row_out(r, y0); row_out(r + RL, y1); row_out(r + 2 * RL, y2); row_out(r + 3 * RL, y3);
      }
      for (; r < nrows; r += RL) row_out(r, __ldg(reinterpret_cast<const float4*>(yp + static_cast<long long>(r) * H)));
    } else {
      for (; r < nrows; r += RL) row_out(r, z4);
    }
  }
  if (ACT) {
    float* cb = sk_smem + rows_per_cta * 8;              // NW > 0: row lanes 1..3 of wacc, [3][NW][H]
    float gs = 0.f;
    if (active) *reinterpret_cast<float4*>(colred + rl * H + 4 * cg) = cs;
    if (NW > 0) {
      if (rl > 0) {
#pragma unroll
        for (int k = 0; k < NW; ++k)
          *reinterpret_cast<float4*>(cb + ((rl - 1) * NW + k) * H + 4 * cg) =
              make_float4(wacc[k][0], wacc[k][1], wacc[k][2], wacc[k][3]);
      }
      if (tid < NW)
        for (int rr = 0; rr < nrows; ++rr) gs += sk_smem[rr * 8 + tid];
    }
    __syncthreads();
    for (int c = tid; c < H; c += blockDim.x) {          // H may exceed the 256 threads (H <= 1024)
      float s = colred[c];
      for (int i = 1; i < RL; ++i) s += colred[i * H + c];
      colpart[static_cast<long long>(blockIdx.x) * H + c] = s;
    }
    if (NW > 0) {
      // skinny_tn_kernel's partial layout, [NW + 1][H] per CTA; only the first NW entries of row NW are meaningful
      float* pp = wpart + static_cast<long long>(blockIdx.x) * (NW + 1) * H;
      if (rl == 0) {
#pragma unroll
        for (int k = 0; k < NW; ++k) {
          const float4 v1 = *reinterpret_cast<const float4*>(cb + k * H + 4 * cg);
          const float4 v2 = *reinterpret_cast<const float4*>(cb + (NW + k) * H + 4 * cg);
          const float4 v3 = *reinterpret_cast<const float4*>(cb + (2 * NW + k) * H + 4 * cg);
          *reinterpret_cast<float4*>(pp + k * H + 4 * cg) =
              make_float4((wacc[k][0] + v1.x) + (v2.x + v3.x), (wacc[k][1] + v1.y) + (v2.y + v3.y),
                          (wacc[k][2] + v1.z) + (v2.z + v3.z), (wacc[k][3] + v1.w) + (v2.w + v3.w));
        }
      }
      if (tid < NW) pp[NW * H + tid] = gs;
    }
  }
}

}  // namespace trl

TRL_API int trl_skinny_k_fwd(const float* X, const float* W, const float* bias, float* Y, int64_t M, int K, int H,
                             int act, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && K >= 1 && K <= 24 && H >= 4 && H % 4 == 0 && H <= 1024,
              "trl_skinny_k_fwd: need 1<=K<=24, H%%4==0, H<=1024 (K=%d H=%d)", K, H);
  TRL_REQUIRE(X && W && bias && Y, "trl_skinny_k_fwd: null pointer");
  TRL_REQUIRE(aligned16(bias) && aligned16(Y), "trl_skinny_k_fwd: bias/Y must be 16-byte aligned");
  const int rows = sk_rows_per_cta(M);
  const unsigned grid = static_cast<unsigned>(ceil_div<long long>(M, rows));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int kp = (K + 3) & ~3;
  const size_t smem = sizeof(float) * (static_cast<size_t>(rows) * kp + static_cast<size_t>(K) * (H + 4));
#define TRL_KF(KK)                                                                                                    \
  case KK: {                                                                                                          \
    if (smem > 48 * 1024) {                                                                                           \
      static bool raised = false;                                                                                     \
      if (!raised) {                                                                                                  \
        cudaError_t e = cudaFuncSetAttribute(skinny_k_fwd_kernel<KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024); \
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return static_cast<int>(e); } \
        raised = true;                                                                                                \
      }                                                                                                               \
    }                                                                                                                 \
    skinny_k_fwd_kernel<KK><<<grid, 256, smem, st>>>(X, W, bias, Y, M, H, act, rows);                                 \
  } break
  switch (K) {
    TRL_KF(1); TRL_KF(2); TRL_KF(3); TRL_KF(4); TRL_KF(5); TRL_KF(6); TRL_KF(7); TRL_KF(8);
    TRL_KF(9); TRL_KF(10); TRL_KF(11); TRL_KF(12); TRL_KF(13); TRL_KF(14); TRL_KF(15); TRL_KF(16);
    TRL_KF(17); TRL_KF(18); TRL_KF(19); TRL_KF(20); TRL_KF(21); TRL_KF(22); TRL_KF(23); TRL_KF(24);
  }
#undef TRL_KF
  return check_launch("skinny_k_fwd_kernel");
}

TRL_API int64_t trl_skinny_tn_scratch_floats(int64_t M, int H, int K) {
  const int rows = trl::sk_rows_per_cta(M);
  return trl::ceil_div<long long>(M, rows) * (K + 1) * H;
}

static int launch_skinny_tn(const float* A, const float* Yact, const float* B, float* Out, float* colsum, int64_t M,
                            int H, int K, int out_transposed, int act, bool fused_act, float* scratch, void* stream,
                            const char* who, bool defer = false) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && K >= 1 && K <= 24 && H >= 32 && H % 32 == 0 && H <= 256,
              "%s: need 1<=K<=24, H%%32==0, H<=256 (K=%d H=%d)", who, K, H);
  TRL_REQUIRE(A && B && Out && scratch, "%s: null pointer", who);
  TRL_REQUIRE(aligned16(A) && aligned16(scratch) && (!Yact || aligned16(Yact)), "%s: A/Y/scratch must be 16-byte aligned", who);
  const int rows = sk_rows_per_cta(M);
  const int nslab = static_cast<int>(ceil_div<long long>(M, rows));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int wc = colsum ? 1 : 0;
  const int kp = (K + 3) & ~3;
  const size_t smem = sizeof(float) * rows * kp;
  const unsigned nthr = static_cast<unsigned>(H);            // 32 threads per 32 columns
#define TRL_TN(KK)                                                                                              \
  case KK:                                                                                                      \
    if (fused_act) skinny_tn_kernel<KK, true><<<nslab, nthr, smem, st>>>(A, Yact, B, wc, act, scratch, M, H, rows);   \
    else skinny_tn_kernel<KK, false><<<nslab, nthr, smem, st>>>(A, nullptr, B, wc, act, scratch, M, H, rows);   \
    break
  switch (K) {
    TRL_TN(1); TRL_TN(2); TRL_TN(3); TRL_TN(4); TRL_TN(5); TRL_TN(6); TRL_TN(7); TRL_TN(8);
    TRL_TN(9); TRL_TN(10); TRL_TN(11); TRL_TN(12); TRL_TN(13); TRL_TN(14); TRL_TN(15); TRL_TN(16);
    TRL_TN(17); TRL_TN(18); TRL_TN(19); TRL_TN(20); TRL_TN(21); TRL_TN(22); TRL_TN(23); TRL_TN(24);
  }
#undef TRL_TN
  int rc = check_launch("skinny_tn_kernel");
  if (rc != TRL_OK || defer) return rc;
  const int n_cs = colsum ? (fused_act ? H : K) : 0;
  const int n_all = K * H + n_cs;
  skinny_tn_reduce_kernel<<<ceil_div(n_all, kRedElems), kRedElems * kRedGroups, 0, st>>>(scratch, Out, colsum, n_cs, nslab, H, K, out_transposed);
  return check_launch("skinny_tn_reduce_kernel");
}

// Out = A^T B: A (M,H), B (M,K<=24).  out_transposed=0: Out (H,K); =1: Out (K,H).  colsum: NULL or (K) = column sums of B.
// scratch: trl_skinny_tn_scratch_floats(M,H,K) floats.
TRL_API int trl_skinny_tn(const float* A, const float* B, float* Out, float* colsum, int64_t M, int H, int K,
                          int out_transposed, float* scratch, void* stream) {
  return launch_skinny_tn(A, nullptr, B, Out, colsum, M, H, K, out_transposed, 0, false, scratch, stream, "trl_skinny_tn");
}

// First-layer backward in one pass: with gz = G * act'(Y) (never stored),  dW (H,K) = gz^T X  and  db (H) = colsum(gz).
TRL_API int trl_skinny_act_wgrad(const float* G, const float* Y, const float* X, float* dW, float* db, int64_t M, int H,
                                 int K, int act, float* scratch, void* stream) {
  using namespace trl;
  TRL_REQUIRE(Y && db, "trl_skinny_act_wgrad: null pointer");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_skinny_act_wgrad: unknown activation %d", act);
  return launch_skinny_tn(G, Y, X, dW, db, M, H, K, 0, act, true, scratch, stream, "trl_skinny_act_wgrad");
}

TRL_API int trl_skinny_n_fwd(const float* X, const float* W, const float* bias, float* Y, int64_t M, int H, int N,
                             void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && N >= 1 && N <= 8 && (H == 128 || H == 256),
              "trl_skinny_n_fwd: need N<=8 and H in {128, 256} (N=%d H=%d)", N, H);
  TRL_REQUIRE(X && W && bias && Y, "trl_skinny_n_fwd: null pointer");
  TRL_REQUIRE(aligned16(X) && aligned16(W), "trl_skinny_n_fwd: X/W must be 16-byte aligned");
  long long blocks = ceil_div<long long>(M, 8 * 3);          // 8 warps x 3-4 rows per iteration
  if (blocks > 2 * kNumSM) blocks = 2 * kNumSM;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>(blocks);
#define TRL_NF(HC, NB) skinny_n_fwd_kernel<HC, NB><<<grid, 256, 0, st>>>(X, W, bias, Y, M, H, N)
#define TRL_NF_H(HC)                  \
  do {                                \
    if (N == 1) TRL_NF(HC, 1);        \
    else if (N == 2) TRL_NF(HC, 2);   \
    else if (N <= 4) TRL_NF(HC, 4);   \
    else TRL_NF(HC, 8);               \
  } while (0)
  if (H == 128) TRL_NF_H(1);
  else TRL_NF_H(2);
#undef TRL_NF_H
#undef TRL_NF
  return check_launch("skinny_n_fwd_kernel");
}

TRL_API int trl_skinny_n_dgrad(const float* G, const float* W, float* dX, int64_t M, int H, int N, void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && N >= 1 && N <= 8 && H >= 4 && H % 4 == 0 && H <= 1024,
              "trl_skinny_n_dgrad: need N<=8, H%%4==0, H<=1024");
  TRL_REQUIRE(G && W && dX, "trl_skinny_n_dgrad: null pointer");
  TRL_REQUIRE(aligned16(W) && aligned16(dX), "trl_skinny_n_dgrad: W/dX must be 16-byte aligned");
  const int rows = sk_rows_per_cta(M);
  const unsigned grid = static_cast<unsigned>(ceil_div<long long>(M, rows));
  skinny_n_dgrad_kernel<false, 0><<<grid, 256, sizeof(float) * rows * 8, static_cast<cudaStream_t>(stream)>>>(
      G, W, nullptr, 0, dX, nullptr, nullptr, M, H, N, rows);
  return check_launch("skinny_n_dgrad_kernel");
}

TRL_API int64_t trl_skinny_dgrad_act_scratch_floats(int64_t M, int H) {
  return trl::ceil_div<long long>(M, trl::sk_rows_per_cta(M)) * H;
}

// Output-layer dgrad fused with the previous layer's activation backward:
//   gz (M,H) = (G (M,N) . W (N,H)) * act'(Y (M,H)),   db (H) = colsum(gz).   scratch: ..._scratch_floats(M,H) floats.
static int launch_n_dgrad_act(const float* G, const float* W, const float* Y, float* gz, float* db, int64_t M, int H, int N,
                              int act, float* scratch, void* stream, bool defer) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && N >= 1 && N <= 8 && H >= 4 && H % 4 == 0 && H <= 1024,
              "trl_skinny_n_dgrad_act: need N<=8, H%%4==0, H<=1024");
  TRL_REQUIRE(G && W && Y && gz && (db || defer) && scratch, "trl_skinny_n_dgrad_act: null pointer");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_skinny_n_dgrad_act: unknown activation %d", act);
  TRL_REQUIRE(aligned16(W) && aligned16(gz) && aligned16(Y), "trl_skinny_n_dgrad_act: W/Y/gz must be 16-byte aligned");
  const int rows = sk_rows_per_cta(M);
  const int nslab = static_cast<int>(ceil_div<long long>(M, rows));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  skinny_n_dgrad_kernel<true, 0><<<nslab, 256, sizeof(float) * rows * 8, st>>>(G, W, Y, act, gz, scratch, nullptr, M, H,
                                                                               N, rows);
  int rc = check_launch("skinny_n_dgrad_kernel");
  if (rc != TRL_OK || defer) return rc;
  // column sums: partial [nslab][H] viewed as a K = 0 "tn" partial (stride H, all H entries are colsum entries)
  skinny_tn_reduce_kernel<<<ceil_div(H, kRedElems), kRedElems * kRedGroups, 0, st>>>(scratch, db, db, H, nslab, H, 0, 0);
  return check_launch("skinny_tn_reduce_kernel");
}

TRL_API int trl_skinny_n_dgrad_act(const float* G, const float* W, const float* Y, float* gz, float* db, int64_t M,
                                   int H, int N, int act, float* scratch, void* stream) {
  return launch_n_dgrad_act(G, W, Y, gz, db, M, H, N, act, scratch, stream, false);
}

// ---- first stages alone + ONE launch for all the second stages of a backward pass -------------------------------------
// The *_partial entry points run only the pass over the (M x H) matrix and leave the per-CTA slabs in `scratch` (which
// must then stay untouched, one scratch buffer per pending job); trl_skinny_reduce_jobs finishes up to 8 such jobs in one
// launch.  kind: 0 = trl_skinny_tn (colsum NULL or (K)), 1 = trl_skinny_act_wgrad (colsum = db (H)), 2 =
// trl_skinny_n_dgrad_act (colsum = db (H); out / K / out_transposed unused).
TRL_API int trl_skinny_tn_partial(const float* A, const float* B, int64_t M, int H, int K, int want_colsum, float* scratch,
                                  void* stream) {
  float dummy;
  return launch_skinny_tn(A, nullptr, B, &dummy, want_colsum ? &dummy : nullptr, M, H, K, 0, 0, false, scratch, stream,
                          "trl_skinny_tn_partial", true);
}

TRL_API int trl_skinny_act_wgrad_partial(const float* G, const float* Y, const float* X, int64_t M, int H, int K, int act,
                                         float* scratch, void* stream) {
  using namespace trl;
  TRL_REQUIRE(Y, "trl_skinny_act_wgrad_partial: null pointer");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_skinny_act_wgrad_partial: unknown activation %d", act);
  float dummy;
  return launch_skinny_tn(G, Y, X, &dummy, &dummy, M, H, K, 0, act, true, scratch, stream, "trl_skinny_act_wgrad_partial", true);
}

TRL_API int trl_skinny_n_dgrad_act_partial(const float* G, const float* W, const float* Y, float* gz, int64_t M, int H, int N,
                                           int act, float* scratch, void* stream) {
  return launch_n_dgrad_act(G, W, Y, gz, nullptr, M, H, N, act, scratch, stream, true);
}

TRL_API int trl_skinny_reduce_jobs(int njobs, const int* kind, const float* const* scratch, float* const* out,
                                   float* const* colsum, const int64_t* M, const int* H, const int* K,
                                   const int* out_transposed, void* stream) {
  using namespace trl;
  TRL_REQUIRE(njobs >= 0 && njobs <= kMaxRedJobs, "trl_skinny_reduce_jobs: njobs %d not in 0..%d", njobs, kMaxRedJobs);
  if (njobs == 0) return TRL_OK;
  TRL_REQUIRE(kind && scratch && out && colsum && M && H && K && out_transposed, "trl_skinny_reduce_jobs: null table");
  ReduceJobs q;
  int ctas = 0;
  for (int j = 0; j < kMaxRedJobs; ++j) {
    q.cta_begin[j] = ctas;
    if (j >= njobs) { q.partial[j] = nullptr; q.out[j] = nullptr; q.colsum[j] = nullptr; q.n_cs[j] = q.nslab[j] = q.H[j] = q.K[j] = q.out_t[j] = 0; continue; }
    TRL_REQUIRE(kind[j] >= 0 && kind[j] <= 2 && scratch[j] && M[j] >= 1 && H[j] >= 1, "trl_skinny_reduce_jobs: bad job %d", j);
    const int rows = sk_rows_per_cta(M[j]);
    q.partial[j] = scratch[j];
    q.nslab[j] = static_cast<int>(ceil_div<long long>(M[j], rows));
    q.H[j] = H[j];
    if (kind[j] == 2) {
      TRL_REQUIRE(colsum[j], "trl_skinny_reduce_jobs: job %d needs colsum", j);
      q.out[j] = colsum[j]; q.colsum[j] = colsum[j]; q.K[j] = 0; q.n_cs[j] = H[j]; q.out_t[j] = 0;
    } else {
      TRL_REQUIRE(out[j] && K[j] >= 1 && K[j] <= 24 && (kind[j] == 0 || colsum[j]), "trl_skinny_reduce_jobs: bad job %d", j);
      q.out[j] = out[j]; q.colsum[j] = colsum[j]; q.K[j] = K[j]; q.out_t[j] = out_transposed[j];
      q.n_cs[j] = colsum[j] ? (kind[j] == 1 ? H[j] : K[j]) : 0;
    }
    ctas += ceil_div(q.K[j] * q.H[j] + q.n_cs[j], kRedElems);
  }
  q.cta_begin[kMaxRedJobs] = ctas;
  q.njobs = njobs;
  skinny_reduce_jobs_kernel<<<ctas, kRedElems * kRedGroups, 0, static_cast<cudaStream_t>(stream)>>>(q);
  return check_launch("skinny_reduce_jobs_kernel");
}

// ---- the output layer's whole backward in one pass over Y (H = 256) ------------------------------------------------
// trl_skinny_n_dgrad_act_partial(G, W, Y, gz, M, 256, N, act, db_scratch) and trl_skinny_tn_partial(Y, G, M, 256, N, 1,
// w_scratch) in one launch, the same bits: gz, the db slabs (reduce kind 2) and the dW (N,H) / dbias (N) slabs (kind 0,
// out_transposed = 1).  db_scratch: trl_skinny_dgrad_act_scratch_floats(M, 256); w_scratch:
// trl_skinny_tn_scratch_floats(M, 256, N).
TRL_API int trl_skinny_n_dgrad_act_wgrad_partial(const float* G, const float* W, const float* Y, float* gz, int64_t M,
                                                 int H, int N, int act, float* db_scratch, float* w_scratch,
                                                 void* stream) {
  using namespace trl;
  TRL_REQUIRE(M >= 1 && N >= 1 && N <= 8 && H == 256,
              "trl_skinny_n_dgrad_act_wgrad: need M>=1, 1<=N<=8, H==256 (M=%lld N=%d H=%d)", static_cast<long long>(M),
              N, H);
  TRL_REQUIRE(G && W && Y && gz && db_scratch && w_scratch, "trl_skinny_n_dgrad_act_wgrad: null pointer");
  TRL_REQUIRE(act >= 0 && act <= 2, "trl_skinny_n_dgrad_act_wgrad: unknown activation %d", act);
  TRL_REQUIRE(aligned16(W) && aligned16(Y) && aligned16(gz) && aligned16(w_scratch),
              "trl_skinny_n_dgrad_act_wgrad: W/Y/gz/w_scratch must be 16-byte aligned");
  const int rows = sk_rows_per_cta(M);
  const int nslab = static_cast<int>(ceil_div<long long>(M, rows));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = sizeof(float) * (static_cast<size_t>(rows) * 8 + 3 * static_cast<size_t>(N) * H);   // <= 28 KB
#define TRL_NDW(NN)                                                                                              \
  case NN:                                                                                                       \
    skinny_n_dgrad_kernel<true, NN><<<nslab, 256, smem, st>>>(G, W, Y, act, gz, db_scratch, w_scratch, M, H, N, rows); \
    break
  switch (N) {
    TRL_NDW(1); TRL_NDW(2); TRL_NDW(3); TRL_NDW(4); TRL_NDW(5); TRL_NDW(6); TRL_NDW(7); TRL_NDW(8);
  }
#undef TRL_NDW
  return check_launch("skinny_n_dgrad_kernel");
}

// ... and both second stages in one trl_skinny_reduce_jobs launch: db (H) = colsum(gz), dW (N,H) = G^T Y, dbias (N) =
// colsum(G).
TRL_API int trl_skinny_n_dgrad_act_wgrad(const float* G, const float* W, const float* Y, float* gz, float* db, float* dW,
                                         float* dbias, int64_t M, int H, int N, int act, float* db_scratch,
                                         float* w_scratch, void* stream) {
  TRL_REQUIRE(db && dW && dbias, "trl_skinny_n_dgrad_act_wgrad: null pointer");
  const int rc = trl_skinny_n_dgrad_act_wgrad_partial(G, W, Y, gz, M, H, N, act, db_scratch, w_scratch, stream);
  if (rc != TRL_OK) return rc;
  const int kind[2] = {2, 0}, Hs[2] = {H, H}, Ks[2] = {0, N}, out_t[2] = {0, 1};
  const float* scratch[2] = {db_scratch, w_scratch};
  float* out[2] = {nullptr, dW};
  float* colsum[2] = {db, dbias};
  const int64_t Ms[2] = {M, M};
  return trl_skinny_reduce_jobs(2, kind, scratch, out, colsum, Ms, Hs, Ks, out_t, stream);
}
