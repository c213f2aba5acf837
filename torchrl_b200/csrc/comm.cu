// comm.cu -- K12: one-shot all-reduce over NVLink peer memory, fused with the gradient-norm reduction.
//
// The reference is single-process (no collective anywhere, SURVEY.md section 2.1 / 8(e)); data-parallel PPO needs, per
// minibatch, the SUM over ranks of the flat pf|vf gradient (570 KB at MLP(256,256)) followed by the per-network
// global norm that clip_grad_norm_ uses (/root/reference/torchrl/algo/on_policy/ppo.py:72,117), and per collector
// step / per epoch a few hundred bytes of fp64 moments.  All of these are LATENCY-bound: NCCL's ring / tree launch
// costs ~25-40 us per call on 8 GPUs, more than the 6 us the bytes need on NVLink 5.
//
// One kernel does the exchange AND the reduction that follows it:
//   * every rank keeps its operand in a buffer that all peers have mapped (cudaIpc handles, exchanged once);
//   * block b of every rank raises flag[ready][b][rank] in all peers' flag pads and waits for the W flags in its
//     own pad: "everybody's operand is complete";
//   * each thread sums its float4 / double slice over the W peer buffers IN RANK ORDER (so every rank computes the
//     bit-identical result -- parameters never drift apart, no broadcast needed), writes the sum to a local output
//     buffer and, for the gradient, accumulates the per-segment sum of squares in fp64 (two-level, fixed order: the
//     role of csrc/optim.cu's grad_sumsq_kernel, with the same last-block tail: reduce.cuh's sumsq_segment_tail);
//   * block b raises flag[done][b][rank] everywhere and waits: "everybody has finished reading my operand", then
//     zeroes its slice of the local operand (the gradient buffer is accumulated into by the next backward).
// Flags carry a sequence number that only grows (kept in device memory, bumped by the last block), so nothing is
// ever reset.  grid <= 148 blocks (one per SM): all co-resident, the peer waits cannot deadlock on scheduling.
// Evidence in SASS: LDG / STG with .SYS scope on peer (IPC-mapped) addresses in the same kernel as the reduction.
// Measured alone (scripts/comm_probe.py, 141 k floats, launch included): 14 us at W = 2, 20 us at W = 8 (NCCL all-reduce
// of the same buffer, without the norms: 19 / 36 us).  Two variants were built and dropped: a reduce-scatter + all-gather
// in two PUSH rounds of flag-carrying 16-byte packets (22 us at W = 2: NVLink sees 70 k small volatile stores per round),
// and a deferred second phase on a side stream beside the Adam launch (no measurable gain).  The flag-in-payload push IS
// the better scheme for the few-hundred-byte fp64 vectors (allreduce_f64_ll_kernel below: 3.5 us against 5.7 us).
#include "reduce.cuh"

namespace trl {
namespace comm {

constexpr int kMaxWorld = 8;
constexpr int kMaxBlocks = 148;                          // one block per SM at most: co-resident
constexpr int kThreads = 256;
constexpr int kMaxSeg = 8;
constexpr int kFlagWords = 2 * kMaxBlocks * kMaxWorld;    // [phase][block][source rank] uint32

__device__ __forceinline__ void st_flag(unsigned* p, unsigned v) {
  asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_flag(const unsigned* p) {
  unsigned v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ double ld_peer_f64(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

struct Peers {
  const void* data[kMaxWorld];     // operand buffer of every rank (own entry = local pointer)
  unsigned* flags[kMaxWorld];      // flag pad of every rank (kFlagWords uint32)
};

// All blocks of all ranks: raise my flag of `phase` in every pad, wait for every rank's flag in my pad.
// No fences and no release / acquire qualifiers (measured: `__threadfence_system` + st.release.sys + ld.acquire.sys
// cost two MEMBAR.SYS per phase, ~14 us per collective on 2 GPUs -- slower than NCCL):
//   * phase 0 publishes data written by EARLIER kernels of this stream: complete in this GPU's L2 -- the coherence
//     point peers read through -- before this kernel started;
//   * phase 1 publishes "my reads are done": every thread has consumed its loaded values (they were summed and
//     stored) before the __syncthreads() that precedes the flag store;
//   * flags and peer data are accessed with .volatile (strong, system-scope: never served from a stale L1 line);
//     the bar.sync orders the polling threads' loads before the other threads' data loads.
__device__ __forceinline__ void cross_rank_barrier(const Peers& pe, int rank, int world, int phase, unsigned seq) {
  const int slot = (phase * kMaxBlocks + blockIdx.x) * kMaxWorld;
  __syncthreads();                                     // every thread of this block is done with the previous stage
  if (threadIdx.x < world) {
    st_flag(pe.flags[threadIdx.x] + slot + rank, seq);
    const unsigned* mine = pe.flags[rank] + slot + threadIdx.x;
    while (static_cast<int>(ld_flag(mine) - seq) < 0) { }
  }
  __syncthreads();
}

struct SegTable {
  long long begin[kMaxSeg + 1];
  int nseg;
};

struct GradParams {
  Peers pe;
  int rank, world;
  float* __restrict__ local;       // this rank's operand (= pe.data[rank]), zeroed at the end when zero_local
  float* __restrict__ out;         // (n) reduced gradient (SUM over ranks)
  long long n;                     // floats, a multiple of 4
  SegTable seg;
  unsigned active_mask;
  double* __restrict__ partial;    // (gridDim.x * nseg) scratch
  double* __restrict__ sumsq3;     // (3 nseg): sum of squares, then (1 - b1^t, sqrt(1 - b2^t)) per segment
  int* __restrict__ step;          // (nseg) Adam step counts (bumped here), may be null
  double beta1, beta2;
  unsigned* __restrict__ ticket;
  unsigned* __restrict__ seq;      // device sequence number of this communicator
  int zero_local;
};

__global__ void __launch_bounds__(kThreads) allreduce_grad_kernel(const GradParams p) {
  __shared__ double sh[kThreads / 32][kMaxSeg];
  const unsigned seq = *p.seq + 1u;
  cross_rank_barrier(p.pe, p.rank, p.world, 0, seq);
  // ---- reduce my slice over the ranks, in rank order -------------------------------------------------------------
  const long long n4 = p.n >> 2;
  const long long per = ceil_div<long long>(n4, gridDim.x);
  const long long lo = per * blockIdx.x, hi = (lo + per < n4) ? lo + per : n4;
  double acc[kMaxSeg];
#pragma unroll
  for (int s = 0; s < kMaxSeg; ++s) acc[s] = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += kThreads) {
    // all W peer loads are issued before the first add (a load-add-load chain costs W NVLink round trips of ~2 us
    // each: measured 39 us per minibatch at W = 8), then summed in rank order
    float4 w[kMaxWorld];
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < p.world) w[r] = ld_peer_f4(static_cast<const float*>(p.pe.data[r]) + 4 * i);
    float4 v = w[0];
#pragma unroll
    for (int r = 1; r < kMaxWorld; ++r)
      if (r < p.world) { v.x += w[r].x; v.y += w[r].y; v.z += w[r].z; v.w += w[r].w; }
    *reinterpret_cast<float4*>(p.out + 4 * i) = v;
    // segments start on 16-byte boundaries (flat.py), so a float4 never straddles two of them
    int s = 0;
#pragma unroll
    for (int k = 1; k < kMaxSeg; ++k) s += (k < p.seg.nseg && 4 * i >= p.seg.begin[k]) ? 1 : 0;
    const double q = static_cast<double>(v.x) * v.x + static_cast<double>(v.y) * v.y + static_cast<double>(v.z) * v.z +
                     static_cast<double>(v.w) * v.w;
#pragma unroll
    for (int k = 0; k < kMaxSeg; ++k) acc[k] += (k == s) ? q : 0.0;
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kMaxSeg; ++k) {
    const double t = warp_sum(acc[k]);
    if (lane == 0) sh[wid][k] = t;
  }
  __syncthreads();
  if (threadIdx.x < p.seg.nseg) {
    double t = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) t += sh[w][threadIdx.x];
    p.partial[blockIdx.x * p.seg.nseg + threadIdx.x] = t;
  }
  // ---- last block to get here: per-segment totals, Adam step counts, bias corrections, sequence number.  Done BEFORE
  // the second cross-rank phase so that this serial tail runs in the shadow of that phase's NVLink round trip.
  if (last_cta(p.ticket, gridDim.x)) {
    const int k = threadIdx.x;
    if (k < p.seg.nseg && ((p.active_mask >> k) & 1u))
      sumsq_segment_tail(p.partial + k, gridDim.x, p.seg.nseg, k, p.seg.nseg, p.sumsq3, p.step, p.beta1, p.beta2);
    if (threadIdx.x == 0) *p.seq = seq;  // every block read the old value at its start (they all passed the ticket above)
  }
  // ---- everybody has read my operand: it may be overwritten ------------------------------------------------------------
  cross_rank_barrier(p.pe, p.rank, p.world, 1, seq);
  if (p.zero_local)
    for (long long i = lo + threadIdx.x; i < hi; i += kThreads)
      *reinterpret_cast<float4*>(p.local + 4 * i) = make_float4(0.f, 0.f, 0.f, 0.f);
}

struct VecParams {
  Peers pe;
  int rank, world;
  double* __restrict__ out;        // mode 0: (n) sum over ranks; mode 1: (world, n) every rank's vector, rank order
  int n;                           // doubles per rank (small: moments)
  int gather;
  unsigned* __restrict__ seq;
};

// one block: moments are a few hundred bytes
__global__ void __launch_bounds__(kThreads) allreduce_f64_kernel(const VecParams p) {
  const unsigned seq = *p.seq + 1u;
  cross_rank_barrier(p.pe, p.rank, p.world, 0, seq);
  for (int i = threadIdx.x; i < p.n; i += kThreads) {
    double w[kMaxWorld];                                 // every peer's value requested before the first use
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < p.world) w[r] = ld_peer_f64(static_cast<const double*>(p.pe.data[r]) + i);
    if (p.gather) {
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r)
        if (r < p.world) p.out[r * p.n + i] = w[r];
    } else {
      double v = 0.0;
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r)
        if (r < p.world) v += w[r];
      p.out[i] = v;
    }
  }
  cross_rank_barrier(p.pe, p.rank, p.world, 1, seq);
  if (threadIdx.x == 0) *p.seq = seq;
}

// ---- small vectors: PUSH with the flag inside the payload (the "LL" scheme NCCL uses for latency-bound sizes) ----------
// Every double travels as one 16-byte store {lo32, seq, hi32, seq}: each 8-byte half carries its own flag, so a reader
// that sees both flags equal to this exchange's sequence number holds valid data -- no fence between data and flag, no
// separate barrier.  A rank WRITES its vector into slot [parity][rank] of every peer's receive area (remote stores are
// fire-and-forget: one NVLink traversal) and then polls its OWN receive area (local memory) for the W contributions.
// Two parities: a rank starts exchange k+2 only after it has finished k+1, which needed every peer's k+1 data, which a
// peer sends only after it has finished reading exchange k (stream order on that peer) -- so slot k%2 is free again.
struct LLParams {
  void* recv[kMaxWorld];           // receive area of every rank: [2][world][nmax] x 16 bytes
  const double* __restrict__ local;
  double* __restrict__ out;        // gather == 0: (n) sum in rank order; gather != 0: (world, n)
  int n, nmax, rank, world, gather;
  unsigned* __restrict__ ll_seq;   // device counter of LL exchanges of this communicator
};

constexpr int kLLThreads = 512;

__global__ void __launch_bounds__(kLLThreads) allreduce_f64_ll_kernel(const LLParams p) {
  const unsigned seq = *p.ll_seq + 1u;
  const long long slot0 = static_cast<long long>(seq & 1u) * p.world;
  for (int i = threadIdx.x; i < p.n; i += kLLThreads) {
    const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(p.local[i]));
    const unsigned lo = static_cast<unsigned>(bits), hi = static_cast<unsigned>(bits >> 32);
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < p.world) {
        char* dst = static_cast<char*>(p.recv[r]) + ((slot0 + p.rank) * p.nmax + i) * 16;
        asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(lo), "r"(seq), "r"(hi), "r"(seq) : "memory");
      }
  }
  const char* mine = static_cast<const char*>(p.recv[p.rank]);
  for (int i = threadIdx.x; i < p.n; i += kLLThreads) {
    double w[kMaxWorld];
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r)
      if (r < p.world) {
        const char* src = mine + ((slot0 + r) * p.nmax + i) * 16;
        unsigned a, fa, b, fb;
        do {
          asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(fa), "=r"(b), "=r"(fb) : "l"(src) : "memory");
        } while (fa != seq || fb != seq);
        w[r] = __longlong_as_double(static_cast<long long>((static_cast<unsigned long long>(b) << 32) | a));
      }
    if (p.gather) {
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r)
        if (r < p.world) p.out[r * p.n + i] = w[r];
    } else {
      double v = 0.0;
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r)
        if (r < p.world) v += w[r];
      p.out[i] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *p.ll_seq = seq;
}

static bool fill_peers(Peers& pe, const void* const* data, void* const* flags, int world) {
  if (world < 1 || world > kMaxWorld || !data || !flags) return false;
  for (int r = 0; r < kMaxWorld; ++r) {
    pe.data[r] = r < world ? data[r] : nullptr;
    pe.flags[r] = r < world ? static_cast<unsigned*>(flags[r]) : nullptr;
    if (r < world && (!pe.data[r] || !pe.flags[r])) return false;
  }
  return true;
}

}  // namespace comm
}  // namespace trl

// ---- peer-mappable memory (the only allocations this library makes: communication buffers must be cudaMalloc blocks
// of their own for cudaIpc; everything else stays in the caller's allocator) ------------------------------------------
TRL_API int trl_comm_flag_bytes(void) { return trl::comm::kFlagWords * 4; }
TRL_API int trl_comm_ipc_handle_bytes(void) { return static_cast<int>(sizeof(cudaIpcMemHandle_t)); }

TRL_API int trl_comm_alloc(int64_t bytes, void** ptr_out) {
  using namespace trl;
  TRL_REQUIRE(bytes > 0 && ptr_out, "trl_comm_alloc: bad arguments");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, static_cast<size_t>(bytes));
  if (e == cudaSuccess) e = cudaMemset(p, 0, static_cast<size_t>(bytes));
  if (e != cudaSuccess) { set_error("trl_comm_alloc: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
  *ptr_out = p;
  return TRL_OK;
}

TRL_API int trl_comm_free(void* ptr) {
  using namespace trl;
  cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) { set_error("trl_comm_free: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
  return TRL_OK;
}

TRL_API int trl_comm_ipc_get(void* ptr, void* handle_out) {
  using namespace trl;
  TRL_REQUIRE(ptr && handle_out, "trl_comm_ipc_get: null pointer");
  cudaError_t e = cudaIpcGetMemHandle(static_cast<cudaIpcMemHandle_t*>(handle_out), ptr);
  if (e != cudaSuccess) { set_error("cudaIpcGetMemHandle: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
  return TRL_OK;
}

TRL_API int trl_comm_ipc_open(const void* handle, void** ptr_out) {
  using namespace trl;
  TRL_REQUIRE(handle && ptr_out, "trl_comm_ipc_open: null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  cudaError_t e = cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) { set_error("cudaIpcOpenMemHandle: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
  return TRL_OK;
}

TRL_API int trl_comm_ipc_close(void* ptr) {
  using namespace trl;
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  if (e != cudaSuccess) { set_error("cudaIpcCloseMemHandle: %s", cudaGetErrorString(e)); return static_cast<int>(e); }
  return TRL_OK;
}

static unsigned grad_blocks(long long n) {
  long long blocks = trl::ceil_div<long long>(n / 4, 1LL * trl::comm::kThreads);   // one float4 per thread while the SMs last
  if (blocks > trl::comm::kMaxBlocks) blocks = trl::comm::kMaxBlocks;
  if (blocks < 1) blocks = 1;
  return static_cast<unsigned>(blocks);
}

TRL_API int trl_comm_scratch_doubles(int nseg) { return trl::comm::kMaxBlocks * (nseg > 0 ? nseg : 1); }

// out (n floats) = sum over ranks of peer_data[r] (rank order), sumsq3 as trl_grad_sumsq computes it for `out`; this
// rank's operand (peer_data[rank]) is zeroed afterwards when zero_local.  peer_data / peer_flags: host arrays of `world`
// device pointers (own entries included).  n % 4 == 0.  `seq`: device uint32 owned by the communicator (starts at 0).
TRL_API int trl_allreduce_grad(const void* const* peer_data, void* const* peer_flags, int rank, int world, float* out,
                               int64_t n, const int64_t* seg_begin_host, int nseg, unsigned active_mask,
                               double* sumsq3_out, int* step_counts, double beta1, double beta2, double* scratch,
                               unsigned* ticket, unsigned* seq, int zero_local, void* stream) {
  using namespace trl;
  using namespace trl::comm;
  GradParams p;
  TRL_REQUIRE(fill_peers(p.pe, peer_data, peer_flags, world), "trl_allreduce_grad: bad peer table (world %d)", world);
  TRL_REQUIRE(rank >= 0 && rank < world, "trl_allreduce_grad: rank %d not in [0, %d)", rank, world);
  TRL_REQUIRE(n > 0 && n % 4 == 0, "trl_allreduce_grad: n = %lld must be a positive multiple of 4", (long long)n);
  TRL_REQUIRE(nseg >= 1 && nseg <= kMaxSeg && seg_begin_host, "trl_allreduce_grad: bad segment table");
  TRL_REQUIRE(out && sumsq3_out && scratch && ticket && seq, "trl_allreduce_grad: null pointer");
  for (int i = 0; i <= nseg; ++i) p.seg.begin[i] = seg_begin_host[i];
  for (int i = nseg + 1; i <= kMaxSeg; ++i) p.seg.begin[i] = seg_begin_host[nseg];
  for (int i = 0; i <= nseg; ++i) TRL_REQUIRE(p.seg.begin[i] % 4 == 0, "trl_allreduce_grad: segments must start on 16-byte boundaries");
  p.seg.nseg = nseg;
  p.rank = rank; p.world = world;
  p.local = static_cast<float*>(const_cast<void*>(peer_data[rank]));
  p.out = out; p.n = n; p.active_mask = active_mask; p.partial = scratch; p.sumsq3 = sumsq3_out; p.step = step_counts;
  p.beta1 = beta1; p.beta2 = beta2; p.ticket = ticket; p.seq = seq; p.zero_local = zero_local;
  allreduce_grad_kernel<<<grad_blocks(n), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("allreduce_grad_kernel");
}

// fp64 vectors of n elements per rank (moments): gather == 0: out (n) = sum over ranks; gather != 0: out (world, n).
TRL_API int trl_allreduce_f64(const void* const* peer_data, void* const* peer_flags, int rank, int world, double* out,
                              int n, int gather, unsigned* seq, void* stream) {
  using namespace trl;
  using namespace trl::comm;
  VecParams p;
  TRL_REQUIRE(fill_peers(p.pe, peer_data, peer_flags, world), "trl_allreduce_f64: bad peer table (world %d)", world);
  TRL_REQUIRE(rank >= 0 && rank < world && n >= 1 && out && seq, "trl_allreduce_f64: bad arguments");
  p.rank = rank; p.world = world; p.out = out; p.n = n; p.gather = gather; p.seq = seq;
  allreduce_f64_kernel<<<1, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("allreduce_f64_kernel");
}

// The same exchange for SMALL vectors (n <= nmax) with the flag carried inside every 16-byte packet: one NVLink traversal,
// no barrier phases (see allreduce_f64_ll_kernel).  peer_recv: host array of `world` device pointers to the ranks' receive
// areas of trl_comm_ll_recv_bytes(world, nmax) bytes each (zero-initialised); ll_seq: device uint32 of the communicator
// (starts at 0, counts LL exchanges only).
TRL_API int64_t trl_comm_ll_recv_bytes(int world, int nmax) { return 2LL * world * nmax * 16; }

TRL_API int trl_allreduce_f64_ll(const double* local, void* const* peer_recv, int rank, int world, double* out, int n,
                                 int nmax, int gather, unsigned* ll_seq, void* stream) {
  using namespace trl;
  using namespace trl::comm;
  TRL_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world, "trl_allreduce_f64_ll: bad rank / world");
  TRL_REQUIRE(n >= 1 && n <= nmax && local && peer_recv && out && ll_seq, "trl_allreduce_f64_ll: bad arguments (n=%d nmax=%d)", n, nmax);
  LLParams p;
  for (int r = 0; r < kMaxWorld; ++r) {
    p.recv[r] = r < world ? peer_recv[r] : nullptr;
    TRL_REQUIRE(r >= world || (p.recv[r] && aligned16(p.recv[r])), "trl_allreduce_f64_ll: receive areas must be 16-byte aligned");
  }
  p.local = local; p.out = out; p.n = n; p.nmax = nmax; p.rank = rank; p.world = world; p.gather = gather; p.ll_seq = ll_seq;
  allreduce_f64_ll_kernel<<<1, kLLThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("allreduce_f64_ll_kernel");
}
