"""Latency of the peer-memory collectives (csrc/comm.cu) with nothing else running: REPS launches inside one CUDA graph
per rank, CUDA events around the replay.  Run under torchrun (2..8 ranks):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 scripts/comm_probe.py
"""
import ctypes
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torchrl_b200 import _lib, ops  # noqa: E402
from torchrl_b200.distributed import DataParallelContext  # noqa: E402


def timed(fn, reps, dev):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _ in range(reps):
                fn()
    g.replay()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(5):
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    t = torch.tensor([best], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def main():
    ctx = DataParallelContext()
    pc = ctx.peer
    assert pc is not None, "needs 2..8 CUDA ranks"
    dev = ctx.device
    reps = 50
    W = ctx.world_size
    # small fp64 vectors: the flag-in-payload push against the two-phase pull
    for n in (40, 1280):
        local, ptrs = pc.region("probe_%d" % n, 8 * n, torch.float64)
        local[:n] = torch.arange(n, device=dev, dtype=torch.float64) + ctx.rank
        out = torch.zeros(n, dtype=torch.float64, device=dev)
        t_ll = timed(lambda: pc.all_reduce_f64("probe_%d" % n, n, out), reps, dev)
        exp = W * torch.arange(n, device=dev, dtype=torch.float64) + W * (W - 1) / 2
        assert torch.equal(out, exp), "LL sum wrong"
        t_pull = timed(lambda: _lib.call("trl_allreduce_f64", ptrs, pc.flag_ptrs, pc.rank, pc.world, out.data_ptr(), n, 0,
                                         pc.seq.data_ptr(), ops._stream()), reps, dev)
        assert torch.equal(out, exp), "pull sum wrong"
        if ctx.rank == 0:
            print(f"W={W} fp64 x {n}: LL push {t_ll:.2f} us   two-phase pull {t_pull:.2f} us", flush=True)
    # the flat PPO gradient (141318 floats, 3 segments) with the fused norm
    total = 141320
    seg = [0, 70656, 70664, total]
    g, gp = pc.region("probe_grad", 4 * total, torch.float32)
    red = torch.zeros(total, device=dev)
    s3 = torch.zeros(9, dtype=torch.float64, device=dev)
    step = torch.zeros(3, dtype=torch.int32, device=dev)
    scr = torch.zeros(int(_lib.load().trl_comm_scratch_doubles(3)), dtype=torch.float64, device=dev)
    tick = torch.zeros(1, dtype=torch.int32, device=dev)
    seg_c = (ctypes.c_int64 * 4)(*seg)
    g[:total] = 1.0 + ctx.rank

    def grad():
        _lib.call("trl_allreduce_grad", gp, pc.flag_ptrs, pc.rank, pc.world, red.data_ptr(), total, seg_c, 3, 7,
                  s3.data_ptr(), step.data_ptr(), 0.9, 0.999, scr.data_ptr(), tick.data_ptr(), pc.seq.data_ptr(), 0,
                  ops._stream())
    t_g = timed(grad, reps, dev)
    assert float(red[0]) == W * (W + 1) / 2
    # NCCL on the same buffer for reference
    t_n = timed(lambda: dist.all_reduce(red), reps, dev) if os.environ.get("PROBE_NCCL", "1") == "1" else float("nan")
    if ctx.rank == 0:
        print(f"W={W} gradient 141 k floats: peer all-reduce + norm {t_g:.2f} us   NCCL all-reduce {t_n:.2f} us", flush=True)
    dist.barrier()


if __name__ == "__main__":
    main()
