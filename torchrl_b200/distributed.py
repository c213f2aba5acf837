"""K12 -- one process per GPU, envs sharded across ranks, NCCL all-reduce of the flat gradient.

The reference is single-process (no torch.distributed / NCCL anywhere, SURVEY.md section 2.1);
this is the data-parallel form of its PPO path that keeps single-process semantics:
  * rank g owns envs [g*N/G, (g+1)*N/G) -- seeds follow VecEnv.seed with the GLOBAL env index;
  * every rank draws the SAME minibatch row order (same host seed), so a global minibatch is the
    same b time-rows x all N envs as in the single-process reference;
  * the flat pf|vf gradient is summed with ONE all-reduce per minibatch and scaled by 1/G inside
    the Adam kernel, *before* global-norm clipping (clip what a single process would clip);
  * advantage-normalisation moments (ppo.py:147) and observation-normaliser batch moments
    (base_wrapper.py:75-82) are all-reduced too, so the statistics span all N envs.
Messages are tiny (570 KB gradient, < 1 KB of moments), i.e. latency-bound.  On CUDA the exchange runs through
csrc/comm.cu: one hand-written kernel per collective that reads every peer's buffer over NVLink (cudaIpc-mapped),
sums in rank order and -- for the gradient -- also produces the per-network gradient norms (a fused compute +
collective; `PeerComm` below).  torch.distributed (NCCL / gloo) remains the bootstrap (rendezvous, handle exchange,
barriers), the fallback (`TORCHRL_B200_COMM=nccl`) and the CPU test path.
"""
import ctypes
import os

import torch
import torch.distributed as dist

from . import ops


class _RawDeviceMemory:
    """__cuda_array_interface__ view of raw device memory (zero-copy into a torch tensor)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


class PeerComm:
    """Peer-mapped communication buffers of this rank and all its peers (csrc/comm.cu).

    One cudaMalloc block per rank: [flag pad | named regions ...].  Regions are carved in call order, which is the
    same on every rank, so a region has the same offset everywhere; peers' blocks are mapped once through cudaIpc
    handles exchanged with torch.distributed."""

    BLOCK_BYTES = 8 << 20

    def __init__(self, ctx):
        self.ctx = ctx
        self.rank, self.world = ctx.rank, ctx.world_size
        dev = ctx.device
        self.base = ops.comm_alloc(self.BLOCK_BYTES)
        mine = torch.tensor(list(ops.comm_ipc_get(self.base)), dtype=torch.uint8, device=dev)
        everyone = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(everyone, mine)
        self.bases = [self.base if r == self.rank else ops.comm_ipc_open(bytes(h.cpu().tolist()))
                      for r, h in enumerate(everyone)]
        self._whole = torch.as_tensor(_RawDeviceMemory(self.base, self.BLOCK_BYTES), device=dev)
        self.flag_bytes = (ops.comm_sizes()[0] + 255) // 256 * 256
        self._top = self.flag_bytes
        self.flag_ptrs = (ctypes.c_void_p * self.world)(*self.bases)
        self.seq = torch.zeros(1, dtype=torch.int32, device=dev)
        self.regions = {}
        # receive area of the flag-in-payload exchange of small fp64 vectors (all_reduce_f64), zero from trl_comm_alloc
        self._ll_recv = self.region("__ll_recv__", ops.comm_ll_recv_bytes(self.world, self.LL_NMAX), torch.uint8)[1]
        self._ll_seq = torch.zeros(1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize(dev)
        dist.barrier()                      # every rank has mapped every block before anyone launches on them

    def region(self, name, nbytes, dtype):
        """(local tensor view, ctypes array of the W peer pointers) of a named region; created on first use."""
        if name in self.regions:
            return self.regions[name]
        nbytes = (int(nbytes) + 255) // 256 * 256
        off = self._top
        if off + nbytes > self.BLOCK_BYTES:
            raise MemoryError("PeerComm block exhausted (%d + %d > %d bytes)" % (off, nbytes, self.BLOCK_BYTES))
        self._top = off + nbytes
        local = self._whole[off:off + nbytes].view(dtype)
        ptrs = (ctypes.c_void_p * self.world)(*[b + off for b in self.bases])
        self.regions[name] = (local, ptrs)
        return self.regions[name]

    LL_NMAX = 2048

    def all_reduce_f64(self, name, n, out, gather=False):
        """out = sum over ranks (or the (W, n) stack when gather) of the first n doubles of region `name`.  Up to
        LL_NMAX doubles travel as flag-carrying 16-byte packets pushed into the peers' receive areas (one NVLink
        traversal, no barrier phases: trl_allreduce_f64_ll); longer vectors take the two-phase pull kernel."""
        local, ptrs = self.regions[name]
        if int(n) <= self.LL_NMAX:
            return ops.allreduce_f64_ll(local, self._ll_recv, self.rank, self.world, out, n, self.LL_NMAX, gather,
                                        self._ll_seq)
        return ops.allreduce_f64(ptrs, self.flag_ptrs, self.rank, self.world, out, n, gather, self.seq)


def shard_range(total, world_size, rank):
    """[first, first+count) of a contiguous, equal-size shard; total must divide evenly."""
    if total % world_size != 0:
        raise ValueError("env count %d is not divisible by world size %d" % (total, world_size))
    per = total // world_size
    return rank * per, per


def combine_moments(sum_x, sum_x2, count):
    """(mean, unbiased std) from globally summed moments -- what torch.std() of the concatenated
    minibatch returns."""
    mean = sum_x / count
    var = (sum_x2 - sum_x * mean) / (count - 1.0)
    return mean, torch.sqrt(torch.clamp(var, min=0.0))


class DataParallelContext:
    def __init__(self, backend=None, device=None):
        self.world_size = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank = int(os.environ.get("RANK", "0"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        self.backend = backend
        if device is None:
            device = torch.device("cuda", self.local_rank) if backend == "nccl" else torch.device("cpu")
        self.device = torch.device(device)
        if self.device.type == "cuda":
            torch.cuda.set_device(self.device)
        if self.world_size > 1 and not dist.is_initialized():
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29500")
            kw = {"device_id": self.device} if backend == "nccl" else {}
            dist.init_process_group(backend=backend, rank=self.rank, world_size=self.world_size, **kw)
        self._peer = None
        self._peer_tried = False

    @property
    def peer(self):
        """The PeerComm of this job (CUDA, world > 1, not disabled by TORCHRL_B200_COMM=nccl), else None."""
        if not self._peer_tried:
            self._peer_tried = True
            if (self.world_size > 1 and self.device.type == "cuda" and self.world_size <= 8
                    and os.environ.get("TORCHRL_B200_COMM", "peer") == "peer"):
                self._peer = PeerComm(self)
        return self._peer

    @property
    def active(self):
        return self.world_size > 1

    def shard(self, total_envs):
        return shard_range(total_envs, self.world_size, self.rank)

    def barrier(self):
        if self.active:
            dist.barrier()

    # ------------------------------------------------------------------ collectives
    def all_reduce_grads(self, flat_grad):
        """SUM the flat gradient over ranks in place (NCCL); returns the scale (1/G) the optimizer must apply."""
        if not self.active:
            return 1.0
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)
        return 1.0 / self.world_size

    def grad_buffer(self, n_floats):
        """Where an optimizer should keep its flat gradient: a peer-mapped region when PeerComm is in use (so that
        `reduce_grads` needs no staging copy), else None (ordinary allocation)."""
        if self.peer is None:
            return None
        local, _ = self.peer.region("flat_grad", 4 * int(n_floats), torch.float32)
        return local[:n_floats]

    def reduce_grads(self, opt, active_mask=None):
        """Gradient exchange of one optimizer step.  PeerComm: ONE kernel sums the peers' flat gradients into
        `opt.reduced`, computes the per-segment sums of squares / Adam step counts / bias corrections of the summed
        gradient (what trl_grad_sumsq would) and zeroes the local gradient once every peer has read it; returns
        (scale, True).  Otherwise NCCL all-reduce in place; returns (scale, False)."""
        if not self.active:
            return 1.0, False
        if self.peer is None or getattr(opt, "_grad_region", None) is None:
            return self.all_reduce_grads(opt.grad), False
        pc = self.peer
        _, ptrs = pc.regions["flat_grad"]
        mask = opt.all_mask if active_mask is None else int(active_mask)
        ops.allreduce_grad(ptrs, pc.flag_ptrs, pc.rank, pc.world, opt.reduced, opt._seg_c, opt.nseg, mask, opt.sumsq3,
                           opt.step_counts, opt.betas, opt._comm_scratch, opt._ticket, pc.seq)
        return 1.0 / self.world_size, True

    def all_reduce_sum_(self, t):
        if self.active:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return t

    def all_reduce_max_(self, t):
        if self.active:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t

    def global_vec_stats(self, x, out):
        """out[0..3] = mean, unbiased std, max, min of the concatenation of `x` over all ranks (every rank holds
        the same number of elements).  CUDA: one raw-moments launch, ONE all-gather of 4 doubles per rank, one
        combine launch (capturable).  CPU tensors (gloo tests): the same arithmetic in torch ops."""
        if x.is_cuda:
            if not hasattr(self, "_mom"):
                self._mom = torch.zeros(4, dtype=torch.float64, device=x.device)
                self._mom_all = torch.zeros(4 * self.world_size, dtype=torch.float64, device=x.device)
            peer = self.peer if self.active else None
            mom = peer.region("vec_moments", 32, torch.float64)[0] if peer is not None else self._mom
            ops.vec_moments(x, mom)
            if peer is not None:
                peer.all_reduce_f64("vec_moments", 4, self._mom_all, gather=True)
            elif self.active:
                dist.all_gather_into_tensor(self._mom_all, self._mom)
            else:
                self._mom_all.copy_(self._mom)
            return ops.vec_stats_from_moments(self._mom_all, self.world_size, x.numel() * self.world_size, out)
        xd = x.double()
        mom = torch.stack([xd.sum(), (xd * xd).sum()])
        ext = torch.stack([x.max(), -x.min()]).double()
        self.all_reduce_sum_(mom)
        self.all_reduce_max_(ext)
        n = float(x.numel() * self.world_size)
        mean = mom[0] / n
        var = (mom[1] - mom[0] * mean) / (n - 1.0)
        std = torch.sqrt(torch.clamp(var, min=0.0))
        out.copy_(torch.stack([mean, std, ext[0], -ext[1]]).to(out.dtype))
        return out

    def max_over_ranks(self, value):
        t = torch.tensor([float(value)], dtype=torch.float64, device=self.device)
        self.all_reduce_max_(t)
        return float(t.item())

    def destroy(self):
        if self.active and dist.is_initialized():
            dist.destroy_process_group()
