"""Correctness + timing of the four csrc/skinny.cu kernels against the cuBLAS route they replace (M = minibatch)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torchrl_b200 import _lib, ops
from torchrl_b200.networks import fused

M = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
H = 256
dev = "cuda"
torch.manual_seed(0)


def timeit(fn, n=50):
    for _ in range(5):
        fn()
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)   # 256 MB > L2
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30)).item()


st = ops._stream
for K, N in ((17, 6), (17, 1), (23, 8)):
    x = torch.randn(M, K, device=dev)
    w1 = torch.randn(H, K, device=dev) / K ** 0.5
    b1 = torch.randn(H, device=dev) * 0.1
    y = torch.empty(M, H, device=dev)
    for act, name in ((1, "tanh"), (2, "relu")):
        f = lambda: _lib.call("trl_skinny_k_fwd", x.data_ptr(), w1.data_ptr(), b1.data_ptr(), y.data_ptr(), M, K, H, act, st())
        f(); torch.cuda.synchronize()
        ref = (x.double() @ w1.double().t() + b1.double())
        ref = torch.tanh(ref) if act == 1 else torch.relu(ref)

        def cub():
            z = torch.mm(x, w1.t())
            _lib.call("trl_bias_act_fwd", z.data_ptr(), b1.data_ptr(), M, H, act, st())
        print("k_fwd   K=%2d %s  err %.2e   skinny %6.1f us   cuBLAS+epilogue %6.1f us" % (K, name, rel(y, ref), timeit(f), timeit(cub)))
    gz = torch.randn(M, H, device=dev)
    out = fused.skinny_tn(gz, x)
    ref = gz.double().t() @ x.double()
    f = lambda: fused.skinny_tn(gz, x, out=out)
    print("tn(wg1) K=%2d       err %.2e   skinny %6.1f us   wgrad() %6.1f us" % (K, rel(out, ref), timeit(f), timeit(lambda: fused.wgrad(gz, x))))
    h = torch.randn(M, H, device=dev)
    w2 = torch.randn(N, H, device=dev) / 16
    b2 = torch.randn(N, device=dev)
    y2 = torch.empty(M, N, device=dev)
    f = lambda: _lib.call("trl_skinny_n_fwd", h.data_ptr(), w2.data_ptr(), b2.data_ptr(), y2.data_ptr(), M, H, N, st())
    f(); torch.cuda.synchronize()
    ref = h.double() @ w2.double().t() + b2.double()
    print("n_fwd   N=%d        err %.2e   skinny %6.1f us   addmm %6.1f us" % (N, rel(y2, ref), timeit(f), timeit(lambda: torch.addmm(b2, h, w2.t()))))
    g = torch.randn(M, N, device=dev)
    dx = torch.empty(M, H, device=dev)
    f = lambda: _lib.call("trl_skinny_n_dgrad", g.data_ptr(), w2.data_ptr(), dx.data_ptr(), M, H, N, st())
    f(); torch.cuda.synchronize()
    ref = g.double() @ w2.double()
    print("n_dgrad N=%d        err %.2e   skinny %6.1f us   mm %6.1f us" % (N, rel(dx, ref), timeit(f), timeit(lambda: torch.mm(g, w2))))
    db = torch.empty(N, device=dev)
    dw = fused.skinny_tn(h, g, colsum=db, out_transposed=True)
    ref = g.double().t() @ h.double()
    f = lambda: fused.skinny_tn(h, g, out=dw, colsum=db, out_transposed=True)

    def cub2():
        fused.wgrad(g, h)
        g.sum(0)
    print("tn(wgN) N=%d        err %.2e / db %.2e   skinny %6.1f us   wgrad()+sum %6.1f us" % (
        N, rel(dw, ref), rel(db, g.double().sum(0)), timeit(f), timeit(cub2)))

    # backward fusions
    gup = torch.randn(M, H, device=dev)
    yact = torch.tanh(torch.randn(M, H, device=dev))
    dW = torch.empty(H, K, device=dev); dbh = torch.empty(H, device=dev)
    ws = fused._scratch("tn", torch.device(dev), M, H, K)
    f = lambda: _lib.call("trl_skinny_act_wgrad", gup.data_ptr(), yact.data_ptr(), x.data_ptr(), dW.data_ptr(), dbh.data_ptr(), M, H, K, 1, ws.data_ptr(), st())
    f(); torch.cuda.synchronize()
    gzr = gup.double() * (1 - yact.double() ** 2)

    def sep():
        gz_ = torch.empty_like(gup); db_ = torch.empty(H, device=dev)
        sc, tk = fused._scratch("bias_act", torch.device(dev), M, H)
        _lib.call("trl_bias_act_bwd", gup.data_ptr(), yact.data_ptr(), gz_.data_ptr(), db_.data_ptr(), M, H, 1, sc.data_ptr(), tk.data_ptr(), st())
        fused.wgrad(gz_, x)
    print("act_wgrad K=%2d     err %.2e / db %.2e   fused %6.1f us   bias_act_bwd + wgrad %6.1f us" % (
        K, rel(dW, gzr.t() @ x.double()), rel(dbh, gzr.sum(0)), timeit(f), timeit(sep)))
    gzo = torch.empty(M, H, device=dev)
    n = int(_lib.load().trl_skinny_dgrad_act_scratch_floats(M, H))
    ws2 = torch.empty(n, device=dev)
    f = lambda: _lib.call("trl_skinny_n_dgrad_act", g.data_ptr(), w2.data_ptr(), yact.data_ptr(), gzo.data_ptr(), dbh.data_ptr(), M, H, N, 1, ws2.data_ptr(), st())
    f(); torch.cuda.synchronize()
    refz = (g.double() @ w2.double()) * (1 - yact.double() ** 2)

    def sep2():
        dx_ = torch.mm(g, w2)
        gz_ = torch.empty_like(dx_); db_ = torch.empty(H, device=dev)
        sc, tk = fused._scratch("bias_act", torch.device(dev), M, H)
        _lib.call("trl_bias_act_bwd", dx_.data_ptr(), yact.data_ptr(), gz_.data_ptr(), db_.data_ptr(), M, H, 1, sc.data_ptr(), tk.data_ptr(), st())
    print("dgrad_act N=%d      err %.2e / db %.2e   fused %6.1f us   mm + bias_act_bwd %6.1f us" % (
        N, rel(gzo, refz), rel(dbh, refz.sum(0)), timeit(f), timeit(sep2)))
