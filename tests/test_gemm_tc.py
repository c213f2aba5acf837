"""wgmma 3xTF32 GEMM (csrc/gemm_tf32x3.cu) vs float64: fp32-faithful (error of the order of the cuBLAS fp32
SIMT GEMM's own error, ~1e-6 relative to max|C|), for the forward/dgrad shape and the split-K wgrad shape."""
import numpy as np
import pytest


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,splits", [(128, 32, 1), (128, 256, 1), (16384, 256, 1), (300, 64, 1), (256, 16384, 64),
                                        (256, 1024, 4), (4096, 512, 2)])
def test_gemm_tf32x3_matches_fp64(M, K, splits):
    import torch
    from torchrl_b200 import ops
    torch.manual_seed(M + K)
    a = torch.randn(M, K, device="cuda")
    b = torch.randn(256, K, device="cuda") / 8
    ref = a.double() @ b.double().t()
    out = ops.gemm_tf32x3_nt(a, b, splits=splits)
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    err = (out.double() - ref).abs().max().item() / scale
    err32 = ((a @ b.t()).double() - ref).abs().max().item() / scale
    print("M=%d K=%d splits=%d  rel err 3xTF32(wgmma) %.2e  fp32 cuBLAS %.2e" % (M, K, splits, err, err32))
    # fp32-faithful: within a small multiple of the fp32 SIMT GEMM's own error (plain TF32 sits at ~3e-4)
    assert err < 8 * err32 + 5e-7, (err, err32)


@pytest.mark.gpu
def test_gemm_tf32x3_error_grows_with_per_cta_reduction_length():
    """The tensor core's fp32 accumulation truncates, so the error grows ~linearly with the number of K steps
    accumulated by one CTA (2e-6 at 256, ~7e-6 at 1024, relative to max|C|): callers keep K/splits <= 256.
    Still ~40x better than plain TF32 at the same length."""
    import torch
    from torchrl_b200 import ops
    torch.manual_seed(0)
    a = torch.randn(256, 1024, device="cuda")
    b = torch.randn(256, 1024, device="cuda") / 8
    ref = a.double() @ b.double().t()
    scale = ref.abs().max().item()
    e_long = (ops.gemm_tf32x3_nt(a, b, splits=1).double() - ref).abs().max().item() / scale
    e_split = (ops.gemm_tf32x3_nt(a, b, splits=4).double() - ref).abs().max().item() / scale
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        e_tf32 = ((a @ b.t()).double() - ref).abs().max().item() / scale
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    print("K=1024 in one CTA %.2e, split in 4 x 256 %.2e, plain TF32 %.2e" % (e_long, e_split, e_tf32))
    assert e_long < 2e-5 and e_split < 5e-6 and e_long < e_tf32 / 10


@pytest.mark.gpu
def test_transpose_kernel():
    import torch
    from torchrl_b200 import ops
    x = torch.randn(1000, 257, device="cuda")
    assert torch.equal(ops.transpose_f32(x), x.t().contiguous())


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,splits", [(128, 32, 1), (256, 256, 1), (256, 16384, 64), (256, 4096, 16), (384, 2048, 8)])
def test_gemm_tf32x3_tn_matches_fp64(M, K, splits):
    """Weight-gradient shape: C = A^T B with the reduction index as the row index of both operands."""
    import torch
    from torchrl_b200 import ops
    torch.manual_seed(M + K + 1)
    a = torch.randn(K, M, device="cuda")
    b = torch.randn(K, 256, device="cuda") / 8
    ref = a.double().t() @ b.double()
    out = ops.gemm_tf32x3_tn(a, b, splits=splits)
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    err = (out.double() - ref).abs().max().item() / scale
    err32 = ((a.t() @ b).double() - ref).abs().max().item() / scale
    print("tn M=%d K=%d splits=%d  rel err 3xTF32(wgmma) %.2e  fp32 cuBLAS %.2e" % (M, K, splits, err, err32))
    # fp32-faithful: within a small multiple of the fp32 SIMT GEMM's own error (plain TF32 sits at ~3e-4)
    assert err < 8 * err32 + 5e-7, (err, err32)
