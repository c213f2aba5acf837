"""Fused bias+activation epilogue (csrc/mlp_epilogue.cu) vs the plain PyTorch layer sequence of MLPBase
(/root/reference/torchrl/networks/base.py:24-44).  Same fp32 formula per element; tolerance covers the
tanhf-vs-torch.tanh implementation difference (1e-6) and the bias-gradient summation order (1e-5 rel)."""
import numpy as np
import pytest


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["tanh", "relu"])
@pytest.mark.parametrize("M,inp,hidden", [(16384, 17, (256, 256)), (300, 23, (64, 400, 300)), (5, 17, (8,))])
def test_fused_mlp_matches_plain_torch(act, M, inp, hidden):
    import copy
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.networks import fused
    torch.manual_seed(0)
    A = nn.Tanh if act == "tanh" else nn.ReLU
    net = networks.Net(input_shape=inp, output_shape=6, hidden_shapes=list(hidden), append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=A).cuda()
    ref = copy.deepcopy(net)
    x = torch.randn(M, inp, device="cuda")
    w = torch.randn(M, 6, device="cuda")
    fused.set_fused_epilogue(True)
    fused.set_matmul_mode("fp32")          # isolate the epilogue kernels: same cuBLAS GEMMs on both sides
    try:
        y1 = net(x)
        (y1 * w).sum().backward()
        fused.set_fused_epilogue(False)
        y0 = ref(x)
        (y0 * w).sum().backward()
    finally:
        fused.set_fused_epilogue(True)
        fused.set_matmul_mode("tc3")
    torch.testing.assert_close(y1, y0, rtol=1e-5, atol=1e-6)
    for (n1, p1), (n0, p0) in zip(net.named_parameters(), ref.named_parameters()):
        scale = p0.grad.abs().max().item() + 1e-12
        torch.testing.assert_close(p1.grad, p0.grad, rtol=1e-4, atol=1e-5 * scale, msg=n1)


@pytest.mark.gpu
def test_fused_path_handles_leading_dims_and_no_grad():
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    net = networks.MLPBase(input_shape=17, hidden_shapes=[32, 32], activation_func=nn.Tanh).cuda()
    x = torch.randn(1, 40, 17, device="cuda")
    with torch.no_grad():
        y = net(x)
    assert y.shape == (1, 40, 32)
    torch.testing.assert_close(y, net.seq_fcs(x), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_tf32x3_matmul_is_fp32_faithful():
    """Error-compensated 3xTF32 GEMM vs float64: its error must be of the order of the fp32 SIMT GEMM's own
    error (and ~1000x smaller than plain TF32)."""
    import torch
    from torchrl_b200.networks import fused
    torch.manual_seed(0)
    a = torch.randn(4096, 256, device="cuda")
    b = torch.randn(256, 256, device="cuda") / 16
    ref = (a.double() @ b.double())
    a_hi, a_lo = fused.split_tf32(a)
    b_hi, b_lo = fused.split_tf32(b)
    torch.testing.assert_close(a_hi + a_lo, a, rtol=0, atol=0)             # exact split
    assert (a_hi.view(torch.int32) & 0x1FFF).abs().max().item() == 0          # hi is TF32-representable
    out3 = fused.mm3(a_hi, a_lo, b_hi, b_lo).double()
    out32 = (a @ b).double()
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        out_tf32 = (a @ b).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    scale = ref.abs().max().item()
    e3, e32, e1 = ((o - ref).abs().max().item() / scale for o in (out3, out32, out_tf32))
    print("max rel err: 3xTF32 %.2e  fp32 %.2e  TF32 %.2e" % (e3, e32, e1))
    assert e3 < 4 * e32 + 1e-7 and e3 < e1 / 50


@pytest.mark.gpu
def test_tf32x3_mlp_matches_fp32_mlp():
    import copy
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.networks import fused
    torch.manual_seed(1)
    net = networks.Net(input_shape=17, output_shape=6, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    ref = copy.deepcopy(net)
    x = torch.randn(16384, 17, device="cuda")
    w = torch.randn(16384, 6, device="cuda")
    fused.set_matmul_mode("tf32x3")
    try:
        y1 = net(x)
        (y1 * w).sum().backward()
    finally:
        fused.set_matmul_mode("fp32")
    try:
        y0 = ref(x)
        (y0 * w).sum().backward()
    finally:
        fused.set_matmul_mode("tc3")
    torch.testing.assert_close(y1, y0, rtol=2e-5, atol=2e-6)
    for (n1, p1), (n0, p0) in zip(net.named_parameters(), ref.named_parameters()):
        scale = p0.grad.abs().max().item() + 1e-12
        torch.testing.assert_close(p1.grad, p0.grad, rtol=1e-4, atol=2e-5 * scale, msg=n1)


@pytest.mark.gpu
def test_tc3_mlp_matches_fp32_mlp():
    """MLP(256,256) forward/backward with the hand-written wgmma 3xTF32 GEMM on the 256-wide layer."""
    import copy
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.networks import fused
    torch.manual_seed(2)
    net = networks.Net(input_shape=17, output_shape=6, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    ref = copy.deepcopy(net)
    x = torch.randn(16384, 17, device="cuda")
    w = torch.randn(16384, 6, device="cuda")
    fused.set_matmul_mode("tc3")
    try:
        y1 = net(x)
        (y1 * w).sum().backward()
    finally:
        fused.set_matmul_mode("fp32")
    try:
        y0 = ref(x)
        (y0 * w).sum().backward()
    finally:
        fused.set_matmul_mode("tc3")
    torch.testing.assert_close(y1, y0, rtol=2e-5, atol=2e-6)
    for (n1, p1), (n0, p0) in zip(net.named_parameters(), ref.named_parameters()):
        scale = p0.grad.abs().max().item() + 1e-12
        torch.testing.assert_close(p1.grad, p0.grad, rtol=1e-4, atol=2e-5 * scale, msg=n1)


@pytest.mark.gpu
@pytest.mark.parametrize("act_name", ["Tanh", "ReLU"])
@pytest.mark.parametrize("inp,out,M,x_grad", [(17, 6, 16384, True), (17, 6, 16384, False), (17, 1, 16384, False),
                                               (23, 1, 4096, True), (23, 8, 4100, False), (17, 8, 1500, False),
                                               (5, 3, 9000, False)])
def test_skinny_layers_match_plain_torch(inp, out, M, x_grad, act_name):
    """First layer (K = obs_dim) and output layer (N = act_dim / 1) through csrc/skinny.cu vs cuBLAS, including
    the two backward fusions: first-layer dW/db straight from (g, y) when the input needs no gradient, and the
    output-layer dgrad fused with the hidden activation backward (M >= 8192: the _MLPTail node)."""
    import copy
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.networks import fused
    torch.manual_seed(inp * out)
    net = networks.Net(input_shape=inp, output_shape=out, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=getattr(nn, act_name)).cuda()
    ref = copy.deepcopy(net)
    x = torch.randn(M, inp, device="cuda", requires_grad=x_grad)
    x0 = x.detach().clone().requires_grad_(x_grad)
    w = torch.randn(M, out, device="cuda")
    if act_name == "ReLU":
        # relu'(y) = [y > 0] is discontinuous: a hidden unit whose pre-activation lies within round-off of zero can
        # land on either side (the 3xTF32 tensor-core layer and the fp32 SIMT layer round differently), which changes
        # that sample's whole back-propagated row.  Such samples are identified in fp64 (any hidden pre-activation
        # with |z| < 1e-5 max|z|, several times the 2e-6 max|z| round-off of the 3xTF32 layer) and take no part in the backward pass (zero upstream
        # gradient): for every remaining sample both routes see the same mask, so the SAME entry-wise round-off
        # tolerances as for Tanh apply -- a wrong mask or scale in the fused kernels cannot hide.
        with torch.no_grad():
            fcs = [m for m in ref.modules() if isinstance(m, nn.Linear)]
            h, risky = x.detach().double(), torch.zeros(M, dtype=torch.bool, device="cuda")
            for fc in fcs[:-1]:
                z = h @ fc.weight.double().t() + fc.bias.double()
                risky |= (z.abs() < max(2e-5, 1e-5 * z.abs().max().item())).any(dim=1)
                h = torch.relu(z)
        assert risky.float().mean().item() < 0.25, "too many samples near a ReLU kink for a meaningful comparison"
        w[risky] = 0.0
    assert fused._SKINNY                      # default route
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

    def close(a, b, scale, name):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=2e-5 * scale, msg=name)
    if x_grad:
        close(x.grad, x0.grad, 0.5 * x0.grad.abs().max().item(), "x")
    for (n1, p1), (n0, p0) in zip(net.named_parameters(), ref.named_parameters()):
        close(p1.grad, p0.grad, p0.grad.abs().max().item() + 1e-12, n1)


@pytest.mark.gpu
def test_skinny_backward_is_deterministic():
    """Fixed combination order in every reduction: two runs give bit-identical gradients."""
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    torch.manual_seed(3)
    net = networks.Net(input_shape=17, output_shape=6, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    x = torch.randn(16384, 17, device="cuda")
    w = torch.randn(16384, 6, device="cuda")
    grads = []
    for _ in range(2):
        net.zero_grad(set_to_none=True)
        (net(x) * w).sum().backward()
        grads.append([p.grad.clone() for p in net.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("out", [1, 6])
def test_deferred_slab_sums_equal_the_immediate_ones(out):
    """Inside fused.deferred_reduces() (with direct_grad: gradients written straight into the flat buffer) the skinny
    weight / bias gradients launch only their first stage; flush_reduces() sums all slabs in ONE launch
    (trl_skinny_reduce_jobs).  Same kernels, same fold order: the gradients are bit-identical to the immediate route."""
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200.flat import FlatAdam
    from torchrl_b200.networks import fused
    torch.manual_seed(out)
    M = 16384
    net = networks.Net(input_shape=17, output_shape=out, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    opt = FlatAdam([net], lrs=[1e-3], eps=1e-5, max_norms=[0.5])
    x = torch.randn(M, 17, device="cuda")
    w = torch.randn(M, out, device="cuda")
    with fused.presplit(), fused.direct_grad():
        y = net(x)
        torch.autograd.backward([y], [w])
    immediate = opt.grad.clone()
    assert float(immediate.abs().max()) > 0
    opt.zero_grad()
    with fused.presplit(), fused.direct_grad(), fused.deferred_reduces():
        y = net(x)
        torch.autograd.backward([y], [w])
        n_jobs = len(fused._DEFER)
        fused.flush_reduces()
    assert n_jobs == 3                          # first-layer dW/db, output-layer dW/db, last hidden layer's db
    assert torch.equal(opt.grad, immediate)
    # leaving the scope with pending jobs is an error, not a silent loss of gradients
    opt.zero_grad()
    with pytest.raises(RuntimeError):
        with fused.presplit(), fused.direct_grad(), fused.deferred_reduces():
            torch.autograd.backward([net(x)], [w])
