"""The MLP layer kernels called straight through the C ABI and compared with float64 restatements of the same operation:
the wgmma 3xTF32 pair GEMM (csrc/gemm_pair.cu), the skinny first / output layer kernels (csrc/skinny.cu), the bias +
activation epilogues and the TF32 operand split (csrc/mlp_epilogue.cu), and the TF32 weight planes the optimizer keeps
(csrc/optim.cu).

Conventions, chosen so that a subtle error fails loudly instead of hiding inside a tolerance:
  * every output is a view into a larger NaN-filled buffer (>= 64 guard elements and >= one guard row on each side);
    the guards must still be NaN after the call (ragged-tail masks);
  * split-K workspaces, slab scratch and epilogue partials are NaN-filled before each call, so a slot that a reduction
    reads but no CTA wrote shows up as NaN; ticket counters must be back at zero after every call;
  * every shape runs one case with small-integer inputs (no activation or ReLU): TF32 holds such values exactly and fp32
    adds them exactly in any order while every partial sum stays below 2^24, so the result must equal the (exact)
    float64 reference bit for bit -- a dropped row, slab, split or column cannot be absorbed by a tolerance;
  * random cases check accuracy against float64 with the bounds stated next to each check;
  * every call is repeated once and must give bit-identical outputs (fixed reduction order).
The tests without the `gpu` mark check the argument validation of the entry points; nothing is launched there.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24                  # fp32 unit round-off
TANH_ABS = 2.5e-7               # |tanh_ex2(x) - tanh(x)| bound stated in csrc/common.cuh (2.31e-7 measured, H100)
GUARD = 64
M_SKINNY = [1, 5, 8, 37, 2112, 2113, 40000]


# ------------------------------------------------------------------------------------------------------------- helpers
class Guarded:
    """A contiguous output `t` of the given shape inside a NaN-filled buffer: at least GUARD elements and one row on
    each side.  offset (elements) shifts the view off its 16-byte alignment."""

    def __init__(self, *shape, offset=0):
        self.n = math.prod(shape)
        pad = -(-max(GUARD, shape[-1] if len(shape) > 1 else 0) // 4) * 4
        self.lo = pad + offset
        self.buf = torch.full((self.lo + self.n + pad,), float("nan"), device="cuda")
        self.t = self.buf[self.lo:self.lo + self.n].view(shape)

    def check(self, what="output"):
        assert torch.isnan(self.buf[:self.lo]).all() and torch.isnan(self.buf[self.lo + self.n:]).all(), \
            "%s: a write landed outside the output" % what
        return self.t


def nan_scratch(n):
    return torch.full((max(int(n), 4),), float("nan"), device="cuda")


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def ints(lo, hi, *shape):
    return torch.randint(lo, hi + 1, shape, device="cuda").float()


def act64(z, act):
    if act == 1:
        return torch.tanh(z)
    if act == 2:
        return torch.relu(z)
    return z


def dact64(y, act):
    """act'(.) through the activation's output y (the kernels' convention)"""
    if act == 1:
        return 1.0 - y * y
    if act == 2:
        return (y > 0).double()
    return torch.ones_like(y)


def assert_exact(got, ref, what):
    assert got.dtype == torch.float32
    bad = got.double() != ref
    assert not bad.any(), "%s: %d of %d entries differ from the exact integer result (first at %s: %r vs %r)" % (
        what, int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()), got[tuple(bad.nonzero()[0].tolist())].item(),
        ref[tuple(bad.nonzero()[0].tolist())].item())


def assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=err.device)
    assert torch.isfinite(got).all(), "%s: non-finite output" % what
    bad = err > bound
    assert not bad.any(), "%s: %d entries beyond the bound (worst %.3g x its bound, max abs err %.3g)" % (
        what, int(bad.sum()), (err[bad] / bound.expand_as(err)[bad]).max().item(), err.max().item())


def dot_bound(absprod, n_terms):
    """fp32 dot product of n_terms products (bias included), any summation order: 4 n u sum|terms|, plus the MUFU tanh"""
    return 4 * n_terms * U * absprod + 2.5e-7


def stream():
    from torchrl_b200 import ops
    return ops._stream()


def call(name, *args):
    from torchrl_b200 import _lib
    _lib.call(name, *args)


def lib():
    from torchrl_b200 import _lib
    return _lib.load()


def twice(run):
    """run() -> list of output tensors; a second run must reproduce every bit"""
    first = [t.clone() for t in run()]
    second = run()
    for i, (a, b) in enumerate(zip(first, second)):
        assert same_bits(a, b), "output %d differs between two identical calls" % i
    return first


# ====================================================================================== A. pair GEMM, forward and dgrad
PAIR_SHAPES = [(1, 32), (7, 64), (127, 96), (128, 256), (129, 512), (1000, 32), (2047, 96), (2048, 512),
               (16384 + 37, 256), (1, 512), (129, 32), (16384 + 37, 64)]
PAIR_EPI = [(False, 0), (True, 0), (True, 1), (True, 2)]       # (bias present, act); no bias: no epilogue


def pair_all_forms(a, b_nt, bias, act):
    """C from all four routes (nt / nn layout x raw / pre-split B): they must agree bit for bit -- the pre-split planes
    are the same cvt.rna split the kernel does in shared memory, and the nn route feeds wgmma the same K-major tiles."""
    from torchrl_b200 import ops
    from torchrl_b200.networks import fused
    M = a.shape[0]
    b_nn = b_nt.t().contiguous()
    outs = []
    for b, nmajor in ((b_nt, False), (b_nn, True)):
        for pre in (False, True):
            out = Guarded(M, 256)
            ops.gemm3_pair(a, b, out=out.t, planes=fused.split_tf32(b) if pre else None, b_nmajor=nmajor, bias=bias,
                           act=act)
            outs.append(out.check("C (nmajor=%d presplit=%d)" % (nmajor, pre)))
    for i, o in enumerate(outs[1:], 1):
        assert same_bits(o, outs[0]), "route %d differs from the raw nt route" % i
    return outs[0]


@pytest.mark.gpu
@pytest.mark.parametrize("i,M,K", [(i,) + s for i, s in enumerate(PAIR_SHAPES)])
def test_pair_gemm_matches_fp64(i, M, K):
    torch.manual_seed(100 + i)
    # integer-exact: |sum| <= 512 * 64 < 2^24
    has_bias, act = PAIR_EPI[i % 4]
    act = 2 if act == 1 else act
    a, b = ints(-8, 8, M, K), ints(-8, 8, 256, K)
    bias = ints(-8, 8, 256) if has_bias else None
    c = twice(lambda: [pair_all_forms(a, b, bias, act)])[0]
    z = a.double() @ b.double().t() + (bias.double() if has_bias else 0)
    assert_exact(c, act64(z, act), "integer C M=%d K=%d" % (M, K))

    # random: within 8x the fp32 cuBLAS GEMM's own error (relative to max|z|) + 5e-7, and within the growth bound
    # 5e-6 * max(1, K/256) of the tensor core's truncating accumulation; tanh and relu are 1-Lipschitz, so the bound on
    # z carries over to act(z) (plus the MUFU tanh's own error)
    has_bias, act = PAIR_EPI[(i + 1) % 4]
    a, b = torch.randn(M, K, device="cuda"), torch.randn(256, K, device="cuda") / 8
    bias = torch.randn(256, device="cuda") if has_bias else None
    c = pair_all_forms(a, b, bias, act)
    z = a.double() @ b.double().t() + (bias.double() if has_bias else 0)
    z32 = (a @ b.t() + (bias if has_bias else 0)).double()
    scale = z.abs().max().item()
    err32 = (z32 - z).abs().max().item() / scale
    rel = min(8 * err32 + 5e-7, 5e-6 * max(1.0, K / 256))
    assert_within(c, act64(z, act), rel * scale + (TANH_ABS if act == 1 else 0.0), "random C M=%d K=%d" % (M, K))


def tanh_probe_values():
    """about 2^20 points over [-20, 20], a dense patch around 0, and +-0 / +-denormals / +-huge finite values"""
    x = torch.cat([torch.linspace(-20, 20, (1 << 20) - 4096, device="cuda"),
                   torch.linspace(-1e-3, 1e-3, 4096 - 32, device="cuda"),
                   torch.tensor([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -1.4e-45, 1e-30, -1e-30, 1e38, -1e38, 88.0, -88.0,
                                 44.5, -44.5, 9.0, -9.0] * 2, device="cuda")])
    assert x.numel() == 1 << 20
    return x


def check_tanh(y, x, what):
    ref = torch.tanh(x.double())
    err = (y.double() - ref).abs()
    print("%s: max |tanh_ex2(x) - tanh(x)| = %.3g" % (what, err.max().item()))
    assert torch.isfinite(y).all(), what
    assert err.max().item() < TANH_ABS, "%s: %.3g" % (what, err.max().item())
    assert same_bits(y[x.abs() > 44], torch.sign(x[x.abs() > 44])), "%s: no saturation" % what


@pytest.mark.gpu
def test_pair_epilogue_tanh_probe():
    """C = tanh_ex2(x) of exactly x: each output column selects one column of A (B[n, k] = [k == n % 32], zero bias),
    so acc + cor reproduces x exactly (x = hi + lo) before the activation.  +-inf and NaN enter through the bias: in A
    they would not survive the operand split (lo = inf - inf)."""
    from torchrl_b200 import ops
    x = tanh_probe_values()
    a = x.view(-1, 32)
    b = (torch.arange(32, device="cuda")[None, :] == (torch.arange(256, device="cuda")[:, None] % 32)).float()
    out = Guarded(a.shape[0], 256)
    ops.gemm3_pair(a, b, out=out.t, bias=torch.zeros(256, device="cuda"), act=1)
    c = out.check()
    check_tanh(c, a[:, torch.arange(256, device="cuda") % 32], "pair epilogue")
    bias = torch.zeros(256, device="cuda")
    bias[:3] = torch.tensor([float("inf"), -float("inf"), float("nan")])
    out = Guarded(1, 256)
    ops.gemm3_pair(torch.zeros(1, 32, device="cuda"), b, out=out.t, bias=bias, act=1)
    c = out.check()[0]
    assert c[0].item() == 1.0 and c[1].item() == -1.0 and math.isnan(c[2].item())
    a = torch.zeros(1, 32, device="cuda")
    a[0, 5] = float("nan")
    out = Guarded(1, 256)
    ops.gemm3_pair(a, b, out=out.t, bias=torch.zeros(256, device="cuda"), act=1)
    assert torch.isnan(out.check()).all()                  # NaN * 0 is NaN: a NaN input poisons its whole row


# ======================================================================================== B. weight-gradient pair GEMM
def _tn_k(splits):
    step = 32 * splits
    return -(-2048 // step) * step


TN_CASES = [(M, s, _tn_k(s)) for s in (1, 2, 3, 7, 8, 9, 64, 65) for M in (256, 512)] + [(256, 64, 16384),
                                                                                        (512, 64, 16384)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,splits,K", TN_CASES)
def test_pair_tn_matches_fp64(M, splits, K):
    """C (M x 256) = A (K x M)^T B (K x 256) with a deterministic split-K reduction (splits not a multiple of 8 take the
    ragged 8-group loop of pair_splitk_reduce_kernel); the second call reuses the first call's workspace."""
    from torchrl_b200 import ops
    torch.manual_seed(M + splits + K)

    def run(a, b):
        ws = nan_scratch(splits * M * 256)
        outs = []
        for _ in range(2):
            out = Guarded(M, 256)
            ops.gemm3_pair_tn(a, b, out=out.t, splits=splits, workspace=ws)
            outs.append(out.check())
        assert same_bits(outs[0], outs[1]), "second call on a reused workspace differs"
        return outs[0]

    a, b = ints(-8, 8, K, M), ints(-8, 8, K, 256)          # |sum| <= 16384 * 64 < 2^24
    assert_exact(run(a, b), a.double().t() @ b.double(), "integer tn M=%d splits=%d" % (M, splits))
    a, b = torch.randn(K, M, device="cuda"), torch.randn(K, 256, device="cuda") / 8
    c = run(a, b)
    ref = a.double().t() @ b.double()
    scale = ref.abs().max().item()
    err = (c.double() - ref).abs().max().item() / scale
    err32 = ((a.t() @ b).double() - ref).abs().max().item() / scale
    kpc = K // splits
    print("tn M=%d K=%d splits=%d: rel err %.2e (fp32 cuBLAS %.2e)" % (M, K, splits, err, err32))
    # the truncating tensor-core accumulation grows ~linearly with the K steps one CTA accumulates; callers keep
    # K / splits <= 256, where the result must also be within 8x cuBLAS fp32's own error
    assert err < 5e-6 * max(1.0, kpc / 256), err
    if kpc <= 256:
        assert err < 8 * err32 + 5e-7, (err, err32)


# ============================================================================================= C. skinny kernels
def k_fwd(X, W, b, act):
    M, K = X.shape
    H = W.shape[0]
    out = Guarded(M, H)
    call("trl_skinny_k_fwd", X.data_ptr(), W.data_ptr(), b.data_ptr(), out.t.data_ptr(), M, K, H, act, stream())
    return out.check("Y")


K_FWD_CASES = [(K, 256) for K in range(1, 25)] + [(K, H) for H in (4, 12, 64, 100, 400, 1024) for K in (1, 11, 17, 24)]


@pytest.mark.gpu
@pytest.mark.parametrize("K,H", K_FWD_CASES)
def test_skinny_k_fwd_matches_fp64(K, H):
    """Y = act(X W^T + b), K <= 24 (one instantiation per K), H % 4 == 0 up to 1024.  At K = 24, H = 1024 and 128 rows
    per CTA the kernel takes ~111 KB of shared memory (the raised-limit launch)."""
    torch.manual_seed(K * 1031 + H)
    for j, M in enumerate(M_SKINNY):
        act = (K + H + j) % 3
        X, W, b = ints(-3, 3, M, K), ints(-3, 3, H, K), ints(-3, 3, H)
        y = twice(lambda: [k_fwd(X, W, b, 2 if act == 1 else act)])[0]
        assert_exact(y, act64(X.double() @ W.double().t() + b.double(), 2 if act == 1 else act),
                     "integer K=%d H=%d M=%d" % (K, H, M))
        X, W, b = torch.randn(M, K, device="cuda"), torch.randn(H, K, device="cuda"), torch.randn(H, device="cuda")
        y = k_fwd(X, W, b, act)
        ref = act64(X.double() @ W.double().t() + b.double(), act)
        absprod = X.double().abs() @ W.double().abs().t() + b.double().abs()
        assert_within(y, ref, dot_bound(absprod, K + 1), "random K=%d H=%d M=%d act=%d" % (K, H, M, act))


@pytest.mark.gpu
def test_skinny_k_fwd_tanh_probe():
    """K = 1, W = 1, b = 0: Y = tanh_ex2(x) of exactly x; +-inf saturate to +-1 and NaN propagates."""
    x = torch.cat([tanh_probe_values(), torch.tensor([float("inf"), -float("inf"), float("nan"), 0.0], device="cuda")])
    y = k_fwd(x.view(-1, 1), torch.ones(4, 1, device="cuda"), torch.zeros(4, device="cuda"), 1)
    for h in range(4):
        check_tanh(y[:-4, h], x[:-4], "skinny_k_fwd column %d" % h)
    assert (y[-4] == 1).all() and (y[-3] == -1).all() and torch.isnan(y[-2]).all() and (y[-1] == 0).all()


def skinny_tn(A, B, colsum, out_t):
    M, H = A.shape
    K = B.shape[1]
    out = Guarded(*((K, H) if out_t else (H, K)))
    cs = Guarded(K) if colsum else None
    ws = nan_scratch(lib().trl_skinny_tn_scratch_floats(M, H, K))
    call("trl_skinny_tn", A.data_ptr(), B.data_ptr(), out.t.data_ptr(), cs.t.data_ptr() if colsum else None, M, H, K,
         int(out_t), ws.data_ptr(), stream())
    return [out.check("Out")] + ([cs.check("colsum")] if colsum else [])


def act_wgrad(G, Y, X, act):
    M, H = G.shape
    K = X.shape[1]
    dw, db = Guarded(H, K), Guarded(H)
    ws = nan_scratch(lib().trl_skinny_tn_scratch_floats(M, H, K))
    call("trl_skinny_act_wgrad", G.data_ptr(), Y.data_ptr(), X.data_ptr(), dw.t.data_ptr(), db.t.data_ptr(), M, H, K,
         act, ws.data_ptr(), stream())
    return [dw.check("dW"), db.check("db")]


TN_SKINNY_CASES = [(K, 256) for K in range(1, 25)] + [(K, H) for H in (32, 96, 128) for K in (1, 17, 24)]


def _three_ms(idx):
    """the two slab-shape edges in every case, one more M in rotation (all of M_SKINNY over the cases)"""
    rest = [1, 8, 37, 2112, 40000]
    return [5, 2113, rest[idx % len(rest)]]


@pytest.mark.gpu
@pytest.mark.parametrize("idx,K,H", [(i,) + c for i, c in enumerate(TN_SKINNY_CASES)])
def test_skinny_tn_and_act_wgrad_match_fp64(idx, K, H):
    """Out = A^T B [+ colsum(B)] and the fused first-layer backward dW = (G act'(Y))^T X, db = colsum(G act'(Y)):
    per-CTA slabs then a fixed-order slab sum.  Reduction bound over M: 1e-5 * sum |terms|."""
    torch.manual_seed(idx)
    for j, M in enumerate(_three_ms(idx)):
        out_t, colsum, act = (idx + j) % 2, (idx + j) % 3 != 0, (idx + 2 * j) % 3
        # integer-exact (|sum| <= 40000 * 9 < 2^24)
        A, B = ints(-3, 3, M, H), ints(-3, 3, M, K)
        got = twice(lambda: skinny_tn(A, B, colsum, out_t))
        ref = A.double().t() @ B.double()
        assert_exact(got[0], ref.t() if out_t else ref, "integer tn K=%d H=%d M=%d" % (K, H, M))
        if colsum:
            assert_exact(got[1], B.double().sum(0), "integer colsum K=%d H=%d M=%d" % (K, H, M))
        G, Y, X = ints(-3, 3, M, H), ints(-3, 3, M, H), ints(-3, 3, M, K)
        a_int = 2 if act == 1 else act
        dw, db = twice(lambda: act_wgrad(G, Y, X, a_int))
        gz = G.double() * dact64(Y.double(), a_int)
        assert_exact(dw, gz.t() @ X.double(), "integer act_wgrad dW K=%d H=%d M=%d" % (K, H, M))
        assert_exact(db, gz.sum(0), "integer act_wgrad db K=%d H=%d M=%d" % (K, H, M))
        # random
        A, B = torch.randn(M, H, device="cuda"), torch.randn(M, K, device="cuda")
        got = skinny_tn(A, B, colsum, out_t)
        ref, bnd = A.double().t() @ B.double(), 1e-5 * (A.double().abs().t() @ B.double().abs())
        assert_within(got[0], ref.t() if out_t else ref, bnd.t() if out_t else bnd, "random tn K=%d H=%d M=%d" % (K, H, M))
        if colsum:
            assert_within(got[1], B.double().sum(0), 1e-5 * B.double().abs().sum(0), "random colsum")
        G, X = torch.randn(M, H, device="cuda"), torch.randn(M, K, device="cuda")
        Y = torch.tanh(torch.randn(M, H, device="cuda")) if act == 1 else torch.randn(M, H, device="cuda")
        dw, db = act_wgrad(G, Y, X, act)
        gz = G.double() * dact64(Y.double(), act)
        assert_within(dw, gz.t() @ X.double(), 1e-5 * (gz.abs().t() @ X.double().abs()) + 1e-30,
                      "random act_wgrad dW K=%d H=%d M=%d act=%d" % (K, H, M, act))
        assert_within(db, gz.sum(0), 1e-5 * gz.abs().sum(0) + 1e-30, "random act_wgrad db")


def n_fwd(X, W, b):
    M, H = X.shape
    N = W.shape[0]
    out = Guarded(M, N)
    call("trl_skinny_n_fwd", X.data_ptr(), W.data_ptr(), b.data_ptr(), out.t.data_ptr(), M, H, N, stream())
    return out.check("Y")


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("N", list(range(1, 9)))
def test_skinny_n_fwd_matches_fp64(N, H):
    """Y = X W^T + b for the output layer: N in 1..8 (instantiations NB = 1, 2, 4, 8), H = 128 (HC = 1) or 256."""
    torch.manual_seed(N * 7 + H)
    for M in M_SKINNY:
        X, W, b = ints(-3, 3, M, H), ints(-3, 3, N, H), ints(-3, 3, N)
        y = twice(lambda: [n_fwd(X, W, b)])[0]
        assert_exact(y, X.double() @ W.double().t() + b.double(), "integer N=%d H=%d M=%d" % (N, H, M))
        X, W, b = torch.randn(M, H, device="cuda"), torch.randn(N, H, device="cuda"), torch.randn(N, device="cuda")
        absprod = X.double().abs() @ W.double().abs().t() + b.double().abs()
        assert_within(n_fwd(X, W, b), X.double() @ W.double().t() + b.double(), dot_bound(absprod, H + 1),
                      "random N=%d H=%d M=%d" % (N, H, M))


def n_dgrad(G, W):
    M, N = G.shape
    H = W.shape[1]
    out = Guarded(M, H)
    call("trl_skinny_n_dgrad", G.data_ptr(), W.data_ptr(), out.t.data_ptr(), M, H, N, stream())
    return out.check("dX")


def n_dgrad_act(G, W, Y, act):
    M, N = G.shape
    H = W.shape[1]
    gz, db = Guarded(M, H), Guarded(H)
    ws = nan_scratch(lib().trl_skinny_dgrad_act_scratch_floats(M, H))
    call("trl_skinny_n_dgrad_act", G.data_ptr(), W.data_ptr(), Y.data_ptr(), gz.t.data_ptr(), db.t.data_ptr(), M, H, N,
         act, ws.data_ptr(), stream())
    return [gz.check("gz"), db.check("db")]


N_DGRAD_CASES = [(N, H) for H in (4, 12, 128, 256, 400, 512, 1024) for N in range(1, 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx,N,H", [(i,) + c for i, c in enumerate(N_DGRAD_CASES)])
def test_skinny_n_dgrad_and_dgrad_act_match_fp64(idx, N, H):
    """dX = G W (N <= 8, H % 4 == 0 up to 1024) and its fusion with the hidden activation backward,
    gz = (G W) * act'(Y), db = colsum(gz) (per-CTA column partials, then the slab sum)."""
    torch.manual_seed(idx + 5000)
    for j, M in enumerate(_three_ms(idx)):
        act = (idx + j) % 3
        a_int = 2 if act == 1 else act
        G, W, Y = ints(-3, 3, M, N), ints(-3, 3, N, H), ints(-3, 3, M, H)
        dx = twice(lambda: [n_dgrad(G, W)])[0]
        ref = G.double() @ W.double()
        assert_exact(dx, ref, "integer dgrad N=%d H=%d M=%d" % (N, H, M))
        gz, db = twice(lambda: n_dgrad_act(G, W, Y, a_int))
        gz_ref = ref * dact64(Y.double(), a_int)
        assert_exact(gz, gz_ref, "integer dgrad_act gz N=%d H=%d M=%d" % (N, H, M))
        assert_exact(db, gz_ref.sum(0), "integer dgrad_act db N=%d H=%d M=%d" % (N, H, M))
        G, W = torch.randn(M, N, device="cuda"), torch.randn(N, H, device="cuda")
        Y = torch.tanh(torch.randn(M, H, device="cuda")) if act == 1 else torch.randn(M, H, device="cuda")
        ref, absprod = G.double() @ W.double(), G.double().abs() @ W.double().abs()
        assert_within(n_dgrad(G, W), ref, 4 * N * U * absprod + 1e-30, "random dgrad N=%d H=%d M=%d" % (N, H, M))
        gz, db = n_dgrad_act(G, W, Y, act)
        d = dact64(Y.double(), act)
        # the product with act'(y) adds at most two roundings to the dot product's error
        assert_within(gz, ref * d, 4 * (N + 2) * U * absprod * d.abs() + 1e-30,
                      "random dgrad_act gz N=%d H=%d M=%d act=%d" % (N, H, M, act))
        assert_within(db, (ref * d).sum(0), 1e-5 * (absprod * d.abs()).sum(0) + 1e-30,
                      "random dgrad_act db N=%d H=%d M=%d act=%d" % (N, H, M, act))


def _partial_job(kind, M, H, K, act=0, colsum=True, out_t=0):
    """Launch the first stage of one job (NaN-filled scratch); returns (job tuple for fused.flush_reduces, outputs,
    the same result through the immediate entry point)"""
    if kind == 0:
        A, B = torch.randn(M, H, device="cuda"), torch.randn(M, K, device="cuda")
        ws = nan_scratch(lib().trl_skinny_tn_scratch_floats(M, H, K))
        call("trl_skinny_tn_partial", A.data_ptr(), B.data_ptr(), M, H, K, int(colsum), ws.data_ptr(), stream())
        out, cs = Guarded(*((K, H) if out_t else (H, K))), Guarded(K) if colsum else None
        return ((0, ws, out.t, cs.t if colsum else None, M, H, K, out_t), [out, cs] if colsum else [out],
                skinny_tn(A, B, colsum, out_t))
    G = torch.randn(M, H, device="cuda")
    Y = torch.tanh(torch.randn(M, H, device="cuda"))
    if kind == 1:
        X = torch.randn(M, K, device="cuda")
        ws = nan_scratch(lib().trl_skinny_tn_scratch_floats(M, H, K))
        call("trl_skinny_act_wgrad_partial", G.data_ptr(), Y.data_ptr(), X.data_ptr(), M, H, K, act, ws.data_ptr(),
             stream())
        dw, db = Guarded(H, K), Guarded(H)
        return (1, ws, dw.t, db.t, M, H, K, 0), [dw, db], act_wgrad(G, Y, X, act)
    G = torch.randn(M, K, device="cuda")                   # K plays N, the output width
    W = torch.randn(K, H, device="cuda")
    ws = nan_scratch(lib().trl_skinny_dgrad_act_scratch_floats(M, H))
    gz, db = Guarded(M, H), Guarded(H)
    call("trl_skinny_n_dgrad_act_partial", G.data_ptr(), W.data_ptr(), Y.data_ptr(), gz.t.data_ptr(), M, H, K, act,
         ws.data_ptr(), stream())
    return (2, ws, None, db.t, M, H, 0, 0), [gz, db], n_dgrad_act(G, W, Y, act)


JOB_SPECS = [(0, 2113, 256, 17, 0, True, 1), (1, 40000, 128, 5, 1, True, 0), (2, 37, 400, 6, 2, True, 0),
             (0, 8, 32, 24, 0, False, 0), (2, 2112, 256, 1, 1, True, 0), (1, 5, 96, 24, 2, True, 0),
             (0, 40000, 64, 3, 0, True, 0), (2, 2113, 1024, 8, 0, True, 0), (1, 1, 256, 11, 0, True, 0),
             (0, 37, 256, 2, 0, False, 1), (2, 40000, 12, 3, 1, True, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("njobs", [8, 11])
def test_skinny_reduce_jobs_equal_immediate_entry_points(njobs):
    """First stages alone, then the slab sums of every pending job through fused.flush_reduces (one launch per group of
    8 jobs): each result is bit-equal to the entry point that reduces immediately."""
    from torchrl_b200.networks import fused
    torch.manual_seed(njobs)
    jobs = []
    with fused.deferred_reduces():
        for spec in JOB_SPECS[:njobs]:
            job, outs, immediate = _partial_job(*spec)
            fused._DEFER.append(job)
            jobs.append((spec, outs, immediate))
        fused.flush_reduces()
    for spec, outs, immediate in jobs:
        assert len(outs) == len(immediate)
        for o, ref in zip(outs, immediate):
            assert same_bits(o.check("job %r" % (spec,)), ref), "job %r differs from its immediate entry point" % (spec,)
    vp = ctypes.c_void_p
    nine = 9
    z = (ctypes.c_int * nine)()
    assert lib().trl_skinny_reduce_jobs(nine, z, (vp * nine)(), (vp * nine)(), (vp * nine)(), (ctypes.c_int64 * nine)(),
                                        z, z, z, None) == -1


# ========================================================================================================= D. epilogues
@pytest.mark.gpu
@pytest.mark.parametrize("H", [1, 3, 4, 132, 260, 1024])
@pytest.mark.parametrize("offset", [0, 1])
def test_bias_act_fwd_matches_fp64(H, offset):
    """z <- act(z + b) in place: float4 path (H % 4 == 0, aligned) and scalar path (H % 4 != 0, or a view 4 bytes
    off its 16-byte alignment)."""
    torch.manual_seed(H + offset)
    for M in (1, 127, 129):
        for act in range(3):
            integer = act != 1
            z0 = ints(-3, 3, M, H) if integer else torch.randn(M, H, device="cuda")
            b = ints(-3, 3, H) if integer else torch.randn(H, device="cuda")

            def run():
                z = Guarded(M, H, offset=offset)
                z.t.copy_(z0)
                call("trl_bias_act_fwd", z.t.data_ptr(), b.data_ptr(), M, H, act, stream())
                return [z.check("z")]
            y = twice(run)[0]
            ref = act64(z0.double() + b.double(), act)
            if integer:
                assert_exact(y, ref, "bias_act_fwd H=%d M=%d act=%d" % (H, M, act))
            else:          # one rounded add, then libdevice tanhf (a couple of ulp)
                assert_within(y, ref, dot_bound(z0.double().abs() + b.double().abs(), 2),
                              "bias_act_fwd H=%d M=%d act=%d" % (H, M, act))


@pytest.mark.gpu
@pytest.mark.parametrize("H", [4, 132, 256, 260, 400])
@pytest.mark.parametrize("M", [1, 128, 129, 16384 + 37])
def test_bias_act_bwd_matches_fp64(M, H):
    """gz = g * act'(y) and db = colsum(gz) with one ticket per 128-column block (blocks partly past H); gz may alias g.
    The scratch is exactly trl_bias_act_bwd_scratch_floats long and NaN-filled; tickets are back at zero after every
    call."""
    torch.manual_seed(M + H)
    tickets = torch.zeros(-(-H // 128), dtype=torch.int32, device="cuda")
    n_scratch = int(lib().trl_bias_act_bwd_scratch_floats(M, H))
    for act in range(3):
        for alias in (False, True):
            integer = act != 1
            g0 = ints(-3, 3, M, H) if integer else torch.randn(M, H, device="cuda")
            y = ints(-3, 3, M, H) if act == 2 else (torch.tanh(torch.randn(M, H, device="cuda")) if act == 1
                                                    else torch.randn(M, H, device="cuda"))

            def run():
                g = Guarded(M, H)
                g.t.copy_(g0)
                gz = g if alias else Guarded(M, H)
                db = Guarded(H)
                scratch = Guarded(n_scratch)        # exactly the advertised size, NaN-filled, guarded
                call("trl_bias_act_bwd", g.t.data_ptr(), y.data_ptr(), gz.t.data_ptr(), db.t.data_ptr(), M, H, act,
                     scratch.t.data_ptr(), tickets.data_ptr(), stream())
                assert (tickets == 0).all(), "tickets not reset"
                scratch.check("scratch")
                return [gz.check("gz"), db.check("db")]
            gz, db = twice(run)
            gz_ref = g0.double() * dact64(y.double(), act)
            what = "bias_act_bwd M=%d H=%d act=%d alias=%d" % (M, H, act, alias)
            if integer:
                assert_exact(gz, gz_ref, what + " gz")
                assert_exact(db, gz_ref.sum(0), what + " db")
            else:          # 1 - y*y and the product: three roundings
                assert_within(gz, gz_ref, 4 * 3 * U * g0.double().abs() * (1 + y.double() ** 2), what + " gz")
                assert_within(db, gz_ref.sum(0), 1e-5 * gz_ref.abs().sum(0) + 1e-30, what + " db")


# ====================================================================================================== E. TF32 planes
def rna_tf32_bits(x):
    """NumPy bit-level cvt.rna.tf32.f32 of finite fp32 values: round the magnitude to 10 mantissa bits, ties away from
    zero (add half of the dropped range to the sign-magnitude bits, then clear them)"""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x1000) & ~np.uint64(0x1FFF)) & 0xFFFFFFFF).astype(np.uint32)


def split_inputs(n, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    bits = x.view(np.uint32).copy()
    # exact ties (dropped bits == 0x1000) on both even and odd kept mantissas: rna rounds them all away from zero,
    # round-to-nearest-even only the odd ones
    tie = rng.random(n) < 0.25
    bits[tie] = (bits[tie] & ~np.uint32(0x1FFF)) | np.uint32(0x1000)
    x = bits.view(np.float32)
    x[: min(n, 2)] = np.array([0.0, -0.0], dtype=np.float32)[: min(n, 2)]
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 1023, (1 << 20) + 3])
@pytest.mark.parametrize("offset", [0, 1])
def test_split_tf32_is_rna_bit_exact(n, offset):
    """hi = cvt.rna.tf32(x) bit for bit, lo = x - hi exactly; aligned (float4 kernel + tail) and 4-byte-offset views
    (scalar kernel)."""
    x_np = split_inputs(n, n + offset)
    ref_hi = rna_tf32_bits(x_np)
    bits = x_np.view(np.uint32)
    if n > 16:      # ties with an even kept mantissa: rna rounds them up, round-to-nearest-even would not
        assert (((bits & 0x1FFF) == 0x1000) & ((bits & 0x2000) == 0)).any()
    x = Guarded(n, offset=offset)
    x.t.copy_(torch.from_numpy(x_np))

    def run():
        hi, lo = Guarded(n, offset=offset), Guarded(n, offset=offset)
        call("trl_split_tf32", x.t.data_ptr(), n, hi.t.data_ptr(), lo.t.data_ptr(), stream())
        return [hi.check("hi"), lo.check("lo")]
    hi_t, lo_t = twice(run)
    hi_np = hi_t.cpu().numpy().view(np.uint32)
    bad = hi_np != ref_hi
    assert not bad.any(), "hi differs from rna at %d places (e.g. x=%r: %08x vs %08x)" % (
        bad.sum(), x_np[bad][0], hi_np[bad][0], ref_hi[bad][0])
    assert torch.equal(lo_t.double(), x.t.double() - torch.from_numpy(ref_hi.view(np.float32)).cuda().double())


def _two_segment_adam():
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.flat import FlatAdam
    nets = [networks.Net(input_shape=17, output_shape=6, hidden_shapes=[256, 256], append_hidden_shapes=[],
                         base_type=networks.MLPBase, activation_func=nn.Tanh).cuda(),
            networks.Net(input_shape=17, output_shape=1, hidden_shapes=[64, 256], append_hidden_shapes=[],
                         base_type=networks.MLPBase, activation_func=nn.ReLU).cuda()]
    return nets, FlatAdam(nets, lrs=[1e-3, 3e-4], eps=1e-5, max_norms=[0.5, None])


def assert_planes_current(flat, what):
    from torchrl_b200.networks import fused
    hi, lo = fused.split_tf32(flat.data)
    assert same_bits(flat.hi, hi) and same_bits(flat.lo, lo), "%s: TF32 planes differ from split_tf32(data)" % what


@pytest.mark.gpu
def test_optimizer_planes_equal_split_of_the_weights():
    """Inside presplit() the GEMM reads the weights' TF32 planes straight from FlatParams.hi / .lo, so after every fused
    Adam step (any active-segment mask) and Polyak update they must equal split_tf32(data) over the whole buffer,
    padding included."""
    import copy
    from torchrl_b200 import ops
    from torchrl_b200.flat import FlatParams
    from torchrl_b200.networks import fused
    torch.manual_seed(7)
    nets, opt = _two_segment_adam()
    target = FlatParams([copy.deepcopy(n) for n in nets])       # same layout as opt
    with fused.presplit():
        assert_planes_current(opt, "presplit entry")
        for mask in (opt.all_mask, 0b01, 0b10, opt.all_mask):
            before = opt.data.clone()
            for p in opt.params:
                p.grad.normal_()
            opt.step(active_mask=mask)
            for s in range(2):
                moved = not torch.equal(opt.seg_slice(s), before[opt.seg_begin[s]:opt.seg_begin[s + 1]])
                assert moved == bool((mask >> s) & 1)
            assert_planes_current(opt, "after Adam step mask=%d" % mask)
        assert_planes_current(target, "presplit entry (target)")
        for _ in range(3):
            ops.polyak_update(target.data, opt.data, 0.005, planes=(target.hi, target.lo))
            assert_planes_current(target, "after Polyak update")


@pytest.mark.gpu
def test_presplit_mlp_equals_in_kernel_split():
    """MLP(256, 256) forward and backward at M = 4096: the GEMMs reading the optimizer's pre-split planes give exactly
    the results of the GEMMs that split the weights in shared memory."""
    from torchrl_b200.networks import fused
    torch.manual_seed(8)
    nets, opt = _two_segment_adam()
    net = nets[0]
    x = torch.randn(4096, 17, device="cuda", requires_grad=True)
    w = torch.randn(4096, 6, device="cuda")
    params = list(net.parameters())

    def run():
        y = net(x)
        return [y.detach()] + list(torch.autograd.grad(y, [x] + params, w))
    outside = run()
    with fused.presplit():
        assert fused._planes_of(params[2]) is not None
        inside = run()
    for i, (a, b) in enumerate(zip(outside, inside)):
        assert same_bits(a, b), "tensor %d differs between pre-split planes and the in-kernel split" % i


# ====================================================================================== F. module-level routes
@pytest.mark.gpu
@pytest.mark.parametrize("act_name", ["Tanh", "ReLU"])
@pytest.mark.parametrize("hidden,inp,out,x_grad", [([64, 64], 3, 1, False), ([128, 128], 11, 4, True),
                                                   ([400, 300], 24, 8, False), ([128, 128], 24, 1, False),
                                                   ([64, 64], 11, 8, True), ([400, 300], 3, 4, True)])
def test_narrow_and_wide_mlps_match_plain_torch(hidden, inp, out, x_grad, act_name):
    """Default "tc3" routing at M >= 2048 for hidden widths the benchmark never uses (skinny first layers of width 64,
    128 and 400; the H = 128 output layer) against cuBLAS fp32 with the skinny kernels off."""
    import copy
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.networks import fused
    torch.manual_seed(inp * out + hidden[0])
    M = 4096
    net = networks.Net(input_shape=inp, output_shape=out, hidden_shapes=hidden, append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=getattr(nn, act_name)).cuda()
    ref = copy.deepcopy(net)
    x = torch.randn(M, inp, device="cuda", requires_grad=x_grad)
    x0 = x.detach().clone().requires_grad_(x_grad)
    w = torch.randn(M, out, device="cuda")
    if act_name == "ReLU":
        # samples with a hidden pre-activation within round-off of the ReLU kink take no part in the backward pass
        # (the two routes may round them to different sides); see test_skinny_layers_match_plain_torch
        with torch.no_grad():
            fcs = [m for m in ref.modules() if isinstance(m, nn.Linear)]
            h, risky = x.detach().double(), torch.zeros(M, dtype=torch.bool, device="cuda")
            for fc in fcs[:-1]:
                z = h @ fc.weight.double().t() + fc.bias.double()
                risky |= (z.abs() < max(2e-5, 1e-5 * z.abs().max().item())).any(dim=1)
                h = torch.relu(z)
        assert risky.float().mean().item() < 0.25
        w[risky] = 0.0
    assert fused.get_matmul_mode() == "tc3" and fused._SKINNY
    y1 = net(x)
    (y1 * w).sum().backward()
    fused.set_skinny(False)
    fused.set_matmul_mode("fp32")
    try:
        y0 = ref(x0)
        (y0 * w).sum().backward()
    finally:
        fused.set_matmul_mode("tc3")
        fused.set_skinny(True)
    torch.testing.assert_close(y1, y0, rtol=2e-5, atol=2e-6)
    if x_grad:
        torch.testing.assert_close(x.grad, x0.grad, rtol=1e-4, atol=1e-5 * x0.grad.abs().max().item())
    for (n1, p1), (n0, p0) in zip(net.named_parameters(), ref.named_parameters()):
        torch.testing.assert_close(p1.grad, p0.grad, rtol=1e-4, atol=2e-5 * (p0.grad.abs().max().item() + 1e-12),
                                   msg=n1)


# ============================================================================= G. argument validation (no GPU needed)
def _host_ptr(buf):
    return ctypes.addressof(buf)


def _rejects(native_lib, rc, needle):
    assert rc == -1
    msg = native_lib.trl_last_error().decode()
    assert needle in msg, msg


def test_gemm3_pair_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    p16 = p + (-p % 16)
    _rejects(native_lib, native_lib.trl_gemm3_pair(p16, p16, None, p16, 128, 48, 0, None, 0, None), "multiple of 32")
    _rejects(native_lib, native_lib.trl_gemm3_pair(p16 + 4, p16, None, p16, 128, 64, 0, None, 0, None), "aligned")
    _rejects(native_lib, native_lib.trl_gemm3_pair(p16, p16, p16 + 4, p16, 128, 64, 1, None, 0, None), "aligned")
    _rejects(native_lib, native_lib.trl_gemm3_pair(p16, p16, None, p16, 128, 64, 0, None, 3, None), "activation")


def test_gemm3_pair_tn_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    p16 = p + (-p % 16)
    _rejects(native_lib, native_lib.trl_gemm3_pair_tn(p16, p16, p16, 384, 2048, 1, None, None), "multiple of 256")
    _rejects(native_lib, native_lib.trl_gemm3_pair_tn(p16, p16, p16, 256, 2048 + 32, 2, p16, None), "32*splits")


def test_skinny_entry_points_reject_bad_shapes(native_lib):
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    p16 = p + (-p % 16)
    _rejects(native_lib, native_lib.trl_skinny_k_fwd(p16, p16, p16, p16, 100, 25, 256, 0, None), "K<=24")
    _rejects(native_lib, native_lib.trl_skinny_k_fwd(p16, p16, p16, p16, 100, 17, 1028, 0, None), "H<=1024")
    _rejects(native_lib, native_lib.trl_skinny_n_fwd(p16, p16, p16, p16, 100, 192, 4, None), "H in {128, 256}")
    vp = ctypes.c_void_p
    z = (ctypes.c_int * 9)()
    _rejects(native_lib, native_lib.trl_skinny_reduce_jobs(9, z, (vp * 9)(), (vp * 9)(), (vp * 9)(),
                                                           (ctypes.c_int64 * 9)(), z, z, z, None), "njobs 9")
