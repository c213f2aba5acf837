"""The wgmma 3xTF32 GEMM (csrc/gemm_wgmma.cuh) across its pipeline boundaries: grids below, at and several times the
SM count with ragged tails, the hot-path shapes of the MLP forward / dgrad on all four routes (nt / nn layout x raw /
pre-split B), the split-K weight-gradient shape, and small-integer inputs that must come out exact.

Outputs live inside NaN-filled buffers whose guards must survive (ragged-row masks), split-K workspaces are NaN-filled
(a slab no CTA wrote shows up), and every call is repeated once and must reproduce every bit.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 256                        # one output row on each side
SMS = 132
M_GRID = [128, SMS * 128, 2 * SMS * 128 + 37, 65536 + 37]
M_HOT = [4096, 16384]


def guarded(M):
    buf = torch.full((M * 256 + 2 * GUARD,), float("nan"), device="cuda")
    return buf, buf[GUARD:GUARD + M * 256].view(M, 256)


def guards_intact(buf):
    return torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all()


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def ints(lo, hi, *shape):
    return torch.randint(lo, hi + 1, shape, device="cuda").float()


def four_routes(a, w, bias, act):
    """C = act(a w^T + bias) from nt / nn x raw / pre-split B, each called twice; returns the four outputs"""
    from torchrl_b200 import ops
    from torchrl_b200.networks import fused
    M = a.shape[0]
    wt = w.t().contiguous()
    outs = []
    for b, nmajor in ((w, False), (wt, True)):
        planes = fused.split_tf32(b)
        for pl in (None, planes):
            got = []
            for _ in range(2):
                buf, out = guarded(M)
                ops.gemm3_pair(a, b, out=out, planes=pl, b_nmajor=nmajor, bias=bias, act=act)
                torch.cuda.synchronize()
                assert guards_intact(buf), "nmajor=%s presplit=%s: a write landed outside C" % (nmajor, pl is not None)
                got.append(out.clone())
            assert same_bits(got[0], got[1]), "nmajor=%s presplit=%s: two calls differ" % (nmajor, pl is not None)
            outs.append(got[0])
    return outs


def assert_routes_agree(outs):
    for i, o in enumerate(outs[1:], 1):
        assert same_bits(outs[0], o), "route %d differs from nt/raw in %d entries" % (i, int((o != outs[0]).sum()))


@pytest.mark.parametrize("M", M_GRID + M_HOT)
def test_forward_routes_bias_tanh(M):
    torch.manual_seed(M)
    K = 256
    a = torch.randn(M, K, device="cuda")
    w = torch.randn(256, K, device="cuda") / math.sqrt(K)
    bias = torch.randn(256, device="cuda") * 0.1
    outs = four_routes(a, w, bias, 1)
    assert_routes_agree(outs)
    z = a.double() @ w.double().t()
    err = (outs[0].double() - torch.tanh(z + bias.double())).abs().max().item()
    bound = 5e-6 * z.abs().max().item() + 2.5e-7        # 3xTF32 at K = 256, plus the MUFU tanh
    assert torch.isfinite(outs[0]).all() and err < bound, "max abs err %.3g (bound %.3g)" % (err, bound)


@pytest.mark.parametrize("M", M_GRID)
def test_plain_matches_tf32x3_entry(M):
    """without an epilogue the hot-path entry point and gemm_tf32x3_nt run the same arithmetic"""
    from torchrl_b200 import ops
    torch.manual_seed(1 + M)
    a = torch.randn(M, 256, device="cuda")
    w = torch.randn(256, 256, device="cuda") / 16
    outs = four_routes(a, w, None, 0)
    assert_routes_agree(outs)
    single = ops.gemm_tf32x3_nt(a, w)
    assert same_bits(outs[0], single)
    ref = a.double() @ w.double().t()
    assert ((outs[0].double() - ref).abs().max() / ref.abs().max()).item() < 5e-6


@pytest.mark.parametrize("M", [128, 2 * SMS * 128 + 37])
def test_integers_exact(M):
    torch.manual_seed(2 + M)
    a = ints(-8, 8, M, 256)
    w = ints(-8, 8, 256, 256)
    outs = four_routes(a, w, None, 0)
    ref = a.double() @ w.double().t()
    for o in outs:
        assert torch.equal(o.double(), ref)


@pytest.mark.parametrize("M", [256, 512])
def test_wgrad_split_k(M):
    from torchrl_b200 import ops
    torch.manual_seed(3 + M)
    K, S = 16384, 64
    g = torch.randn(K, M, device="cuda")
    x = torch.randn(K, 256, device="cuda")
    ref = g.double().t() @ x.double()
    for fn in (ops.gemm3_pair_tn, ops.gemm_tf32x3_tn):
        got = []
        for _ in range(2):
            ws = torch.full((S * M * 256,), float("nan"), device="cuda")
            buf, out = guarded(M)
            fn(g, x, out=out, splits=S, workspace=ws)
            torch.cuda.synchronize()
            assert guards_intact(buf)
            got.append(out.clone())
        assert same_bits(got[0], got[1]), "%s: two calls differ" % fn.__name__
        err = ((got[0].double() - ref).abs().max() / ref.abs().max()).item()
        assert torch.isfinite(got[0]).all() and err < 5e-6, "%s: rel err %.3g" % (fn.__name__, err)


@pytest.mark.parametrize("M", [256, 512])
def test_wgrad_integers_exact(M):
    from torchrl_b200 import ops
    torch.manual_seed(4 + M)
    K, S = 16384, 64
    g = ints(-4, 4, K, M)
    x = ints(-4, 4, K, 256)
    ref = g.double().t() @ x.double()
    for fn in (ops.gemm3_pair_tn, ops.gemm_tf32x3_tn):
        ws = torch.full((S * M * 256,), float("nan"), device="cuda")
        assert torch.equal(fn(g, x, splits=S, workspace=ws).double(), ref), fn.__name__
