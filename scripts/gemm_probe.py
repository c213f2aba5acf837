"""Hardware check of the hot-path 3xTF32 GEMM (csrc/gemm_pair.cu) against fp64 and against csrc/gemm_tf32x3.cu.

    python scripts/gemm_probe.py            # every case in its own subprocess under a 90 s timeout
    python scripts/gemm_probe.py case nt    # one case in this process

A wrong barrier protocol hangs the kernel: never run a case without a timeout around it.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = ("nt", "nt_split", "nn", "nn_split", "tn", "time", "dgrad_first")


def timeit(fn, n=50):
    import torch
    for _ in range(5):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / n


def planes(w):
    from torchrl_b200.networks import fused
    return fused.split_tf32(w)


def run_case(name):
    import torch
    from torchrl_b200 import ops
    torch.manual_seed(0)
    dev = "cuda"
    if name in ("nt", "nt_split", "nn", "nn_split"):
        nmajor = name.startswith("nn")
        for M, K in ((256, 32), (256, 256), (1000, 256), (4096, 256), (16384, 256), (16384, 512)):
            a = torch.randn(M, K, device=dev)
            w = torch.randn(256, K, device=dev) / K ** 0.5          # forward weight (256 out, K in)
            b = w.t().contiguous() if nmajor else w                   # nn: (K, 256) row-major
            bias = torch.randn(256, device=dev) * 0.1
            ref = a.double() @ w.double().t()
            pl = planes(b) if name.endswith("split") else None
            got = ops.gemm3_pair(a, b, planes=pl, b_nmajor=nmajor)
            torch.cuda.synchronize()
            scale = ref.abs().max().item()
            err = (got.double() - ref).abs().max().item() / scale
            got_t = ops.gemm3_pair(a, b, planes=pl, b_nmajor=nmajor, bias=bias, act=1)
            err_t = (got_t.double() - torch.tanh(ref + bias.double())).abs().max().item()
            got_r = ops.gemm3_pair(a, b, planes=pl, b_nmajor=nmajor, bias=bias, act=2)
            err_r = (got_r.double() - torch.relu(ref + bias.double())).abs().max().item() / scale
            print("%-9s M=%6d K=%4d  rel err %.2e  tanh abs err %.2e  relu rel err %.2e" % (name, M, K, err, err_t, err_r),
                  flush=True)
            # 3xTF32 with the tensor core's fp32 accumulation: ~2e-6 of max|C| at K = 256, growing linearly with K
            tol = 5e-6 * max(1, K // 256)
            assert err < tol and err_t < tol * max(1.0, scale) and err_r < tol, "accuracy"
    elif name == "tn":
        for M, K, S in ((256, 32, 1), (256, 2048, 8), (256, 16384, 64), (512, 16384, 64)):
            g = torch.randn(K, M, device=dev)
            x = torch.randn(K, 256, device=dev)
            ref = g.double().t() @ x.double()
            got = ops.gemm3_pair_tn(g, x, splits=S)
            torch.cuda.synchronize()
            err = (got.double() - ref).abs().max().item() / ref.abs().max().item()
            print("tn        M=%6d K=%6d splits=%2d rel err %.2e" % (M, K, S, err), flush=True)
            assert err < 5e-6, "accuracy"
    elif name == "time":
        for M in (4096, 16384, 65536):
            K = 256
            a = torch.randn(M, K, device=dev)
            w = torch.randn(256, K, device=dev) / 16
            wt = w.t().contiguous()
            bias = torch.randn(256, device=dev) * 0.1
            pl, plt = planes(w), planes(wt)
            t = {}
            t["pair nt raw+tanh"] = timeit(lambda: ops.gemm3_pair(a, w, bias=bias, act=1))
            t["pair nt split+tanh"] = timeit(lambda: ops.gemm3_pair(a, w, planes=pl, bias=bias, act=1))
            t["pair nt split"] = timeit(lambda: ops.gemm3_pair(a, w, planes=pl))
            t["pair nn split"] = timeit(lambda: ops.gemm3_pair(a, w, planes=pl, b_nmajor=True))
            t["single nt+tanh"] = timeit(lambda: ops.gemm_tf32x3_nt(a, w, bias=bias, act=1))
            t["single nt"] = timeit(lambda: ops.gemm_tf32x3_nt(a, w))
            t["cublas fp32"] = timeit(lambda: torch.mm(a, wt))
            print("M=%6d K=256: " % M + "  ".join("%s %.1f us" % kv for kv in t.items()), flush=True)
        K = 16384
        g = torch.randn(K, 256, device=dev)
        x = torch.randn(K, 256, device=dev)
        ws = torch.empty(64 * 256 * 256, device=dev)
        t1 = timeit(lambda: ops.gemm3_pair_tn(g, x, splits=64, workspace=ws))
        t2 = timeit(lambda: ops.gemm_tf32x3_tn(g, x, splits=64, workspace=ws))
        t3 = timeit(lambda: torch.mm(g.t(), x))
        print("wgrad 256x256, K=16384, 64 splits (incl. reduce): pair %.1f us  single %.1f us  cublas %.1f us" % (t1, t2, t3),
              flush=True)
    elif name == "dgrad_first":
        # the dgrad dH1 = gz2 W2 with the first layer's backward in its epilogue, against the dgrad (transposed
        # pre-split planes) followed by trl_skinny_act_wgrad_partial: same slab partials, one launch instead of two
        from torchrl_b200 import _lib
        M, K = 16384, 17
        gz = torch.randn(M, 256, device=dev)
        w = torch.randn(256, 256, device=dev) / 16
        hi, lo = planes(w)
        plt = (hi.t().contiguous(), lo.t().contiguous())
        h1 = torch.tanh(torch.randn(M, 256, device=dev))
        x = torch.randn(M, K, device=dev)
        n = int(_lib.load().trl_skinny_tn_scratch_floats(M, 256, K))
        ws_f, ws_u = torch.empty(n, device=dev), torch.empty(n, device=dev)
        dh1 = torch.empty(M, 256, device=dev)

        def unfused():
            ops.gemm3_pair(gz, w, out=dh1, planes=plt)
            _lib.call("trl_skinny_act_wgrad_partial", dh1.data_ptr(), h1.data_ptr(), x.data_ptr(), M, 256, K, 1,
                      ws_u.data_ptr(), ops._stream())

        def fused_():
            ops.gemm3_pair_dgrad_act_wgrad(gz, plt, h1, x, 1, ws_f)

        unfused()
        fused_()
        torch.cuda.synchronize()
        assert torch.equal(ws_f.view(torch.int32), ws_u.view(torch.int32)), "slab partials differ"
        t_d = timeit(lambda: ops.gemm3_pair(gz, w, out=dh1, planes=plt))
        t_u = timeit(unfused)
        t_f = timeit(fused_)
        print("M=%d K=%d: dgrad %.1f us, dgrad + act_wgrad %.1f us, fused %.1f us (50 calls each)" % (M, K, t_d, t_u, t_f),
              flush=True)
    else:
        raise SystemExit("unknown case " + name)
    print("CASE %s OK" % name, flush=True)


def main():
    if len(sys.argv) >= 3 and sys.argv[1] == "case":
        return run_case(sys.argv[2])
    failed = []
    for c in CASES:
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "case", c], timeout=90)
            if r.returncode != 0:
                failed.append(c)
                print("CASE %s FAILED rc=%d" % (c, r.returncode), flush=True)
        except subprocess.TimeoutExpired:
            failed.append(c)
            print("CASE %s TIMED OUT (hang)" % c, flush=True)
    print("gemm_probe: failed = %s" % failed, flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
