"""The backward GEMMs of the 256-wide MLP layers: the weight gradient with its split-K sum inside one clustered launch
(trl_gemm3_pair_tn_cluster) against the two-launch slab route it replaces (trl_gemm3_pair_tn), bit for bit; the
transposed weight planes of fused.transposed_planes() and the dgrad that reads them K-major against the N-major route.

Workspaces are NaN-filled (a partial no CTA wrote shows up), outputs sit inside NaN guards, every call runs twice and
again from a replayed CUDA graph (a ticket left non-zero would pick the wrong last CTA), and the tickets must come back
zero.  The argument checks need no GPU.
"""
import ctypes

import pytest
import torch

GUARD = 256


def guarded(M):
    buf = torch.full((M * 256 + 2 * GUARD,), float("nan"), device="cuda")
    return buf, buf[GUARD:GUARD + M * 256].view(M, 256)


def guards_intact(buf):
    return torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all()


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def two_launch(g, x, splits):
    from torchrl_b200 import ops
    ws = torch.full((splits * g.shape[1] * 256,), float("nan"), device="cuda")
    return ops.gemm3_pair_tn(g, x, splits=splits, workspace=ws)


def cluster_runs(g, x, splits):
    """two direct calls and two graph replays of the clustered wgrad, each into a fresh guarded output"""
    from torchrl_b200 import ops
    M = g.shape[1]
    ws = torch.full((8 * M * 256,), float("nan"), device="cuda")
    tickets = torch.zeros(M // 8, dtype=torch.int32, device="cuda")
    outs = []
    for _ in range(2):
        buf, out = guarded(M)
        ops.gemm3_pair_tn_cluster(g, x, ws, tickets, out=out, splits=splits)
        torch.cuda.synchronize()
        assert guards_intact(buf)
        outs.append(out.clone())
    buf, out = guarded(M)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gemm3_pair_tn_cluster(g, x, ws, tickets, out=out, splits=splits)
    for _ in range(2):
        out.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert guards_intact(buf)
        outs.append(out.clone())
    assert int(tickets.abs().sum()) == 0, "a ticket was left non-zero"
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("M", [256, 512])
@pytest.mark.parametrize("splits", [8, 16, 24, 32, 64])
def test_cluster_wgrad_matches_two_launch(M, splits):
    torch.manual_seed(10 * M + splits)
    K = 16384 if 16384 % (32 * splits) == 0 else 21 * 32 * splits      # 3-CTA clusters: 16128
    g = torch.randn(K, M, device="cuda")
    x = torch.randn(K, 256, device="cuda")
    ref = two_launch(g, x, splits)
    for i, o in enumerate(cluster_runs(g, x, splits)):
        assert same_bits(o, ref), "run %d differs from the two-launch route in %d entries" % (i, int((o != ref).sum()))
    exact = g.double().t() @ x.double()
    err = ((ref.double() - exact).abs().max() / exact.abs().max()).item()
    assert torch.isfinite(ref).all() and err < 5e-6, "rel err %.3g" % err


@pytest.mark.gpu
@pytest.mark.parametrize("M", [256, 512])
@pytest.mark.parametrize("splits", [8, 64])
def test_cluster_wgrad_integers_exact(M, splits):
    torch.manual_seed(20 * M + splits)
    K = 16384
    g = torch.randint(-4, 5, (K, M), device="cuda").float()
    x = torch.randint(-4, 5, (K, 256), device="cuda").float()
    exact = g.double().t() @ x.double()
    for o in cluster_runs(g, x, splits):
        assert torch.equal(o.double(), exact)


def _transposed_planes_current(scope, weights):
    from torchrl_b200.networks import fused
    torch.cuda.synchronize()
    for w in weights:
        hi, lo = fused._PLANES[w.data_ptr()]
        hi_t, lo_t = scope.planes(w)
        assert same_bits(hi_t, hi.t()) and same_bits(lo_t, lo.t())
        assert same_bits(hi + lo, w.detach())


@pytest.mark.gpu
def test_transposed_planes_follow_refresh_and_adam():
    from torchrl_b200 import flat
    from torchrl_b200.networks import fused
    torch.manual_seed(5)
    net = torch.nn.Sequential(torch.nn.Linear(17, 256), torch.nn.Tanh(), torch.nn.Linear(256, 256), torch.nn.Tanh(),
                              torch.nn.Linear(256, 256)).cuda()
    opt = flat.FlatAdam([net], lrs=1e-2)
    square = [net[2].weight, net[4].weight]
    assert opt.hi_t.shape == (2, 256, 256)
    with fused.presplit():
        with fused.transposed_planes(opt) as tp:
            _transposed_planes_current(tp, square)
        before = opt.hi_t.clone()
        for p in net.parameters():
            p.grad.copy_(torch.randn_like(p))
        opt.step()
        with fused.transposed_planes(opt) as tp:
            _transposed_planes_current(tp, square)
        assert not torch.equal(before, opt.hi_t), "the Adam step did not reach the transposed planes"
        with fused.transposed_planes() as tp:
            assert tp.planes(square[0]) is None, "a buffer outside the scope was served"


@pytest.mark.gpu
@pytest.mark.parametrize("M", [4096, 16384, 16384 + 37])
def test_dgrad_on_transposed_planes_matches_nmajor(M):
    """mm_dgrad inside transposed_planes() (K-major planes, the forward's route) against the N-major pre-split route,
    on the calling stream and on a second one"""
    from torchrl_b200 import flat
    from torchrl_b200.networks import fused
    torch.manual_seed(6 + M)
    lin = torch.nn.Linear(256, 256).cuda()
    fp = flat.FlatParams([lin])
    w = lin.weight
    gz = torch.randn(M, 256, device="cuda")
    with fused.presplit():
        ref = fused.mm_dgrad(gz, w)
        with fused.transposed_planes(fp) as tp:
            assert tp.planes(w) is not None
            got = [fused.mm_dgrad(gz, w) for _ in range(2)]
            other = torch.cuda.Stream()
            other.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(other):
                got.append(fused.mm_dgrad(gz, w))
            torch.cuda.current_stream().wait_stream(other)
    torch.cuda.synchronize()
    for i, o in enumerate(got):
        assert same_bits(o, ref), "call %d differs from the N-major route in %d entries" % (i, int((o != ref).sum()))
    exact = gz.double() @ w.detach().double()
    assert ((ref.double() - exact).abs().max() / exact.abs().max()).item() < 5e-6


def _rejects(native_lib, rc, needle):
    assert rc == -1
    msg = native_lib.trl_last_error().decode()
    assert needle in msg, msg


def test_cluster_wgrad_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    p16 = p + (-p % 16)
    fn = native_lib.trl_gemm3_pair_tn_cluster
    for splits in (0, 1, 4, 12, 72, 128):
        _rejects(native_lib, fn(p16, p16, p16, 256, 16384, splits, p16, p16, None), "multiple of 8 in [8, 64]")
    _rejects(native_lib, fn(p16, p16, p16, 256, 16384, 64, p16, None, None), "null pointer")
    _rejects(native_lib, fn(p16, p16, p16, 256, 16384, 64, None, p16, None), "null pointer")
    _rejects(native_lib, fn(p16, p16, p16, 384, 16384, 64, p16, p16, None), "multiple of 256")
    _rejects(native_lib, fn(p16, p16, p16, 256, 16384 + 32 * 8, 64, p16, p16, None), "32*splits")
    _rejects(native_lib, fn(p16 + 4, p16, p16, 256, 16384, 64, p16, p16, None), "aligned")
