"""The dgrad GEMM with the first layer's backward as its epilogue (trl_gemm3_pair_dgrad_act_wgrad): for an MLP whose input
needs no gradient, dH1 = gz2 W2 is reduced to the first layer's weight / bias gradient slab partials inside the dgrad
launch.  They must be bit-identical to the two-launch route they replace (the dgrad on the transposed pre-split planes,
then trl_skinny_act_wgrad), at every slab size the skinny kernels use: 63-row slabs at M = 16384, a ragged last slab,
64-row slabs at the largest accepted M, and tiles of several 16- or 8-row slabs.

Scratch buffers are NaN-filled (a slab no CTA wrote shows up), calls are repeated, replayed from a CUDA graph and run on
two streams at once.  The argument checks need no GPU.
"""
import ctypes

import pytest
import torch

ACTS = {1: torch.tanh, 2: torch.relu}


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def problem(M, K, act, seed):
    from torchrl_b200.networks import fused
    g = torch.Generator(device="cuda").manual_seed(seed)
    gz = torch.randn(M, 256, device="cuda", generator=g)
    w = torch.randn(256, 256, device="cuda", generator=g) / 16
    hi, lo = fused.split_tf32(w)
    planes_t = (hi.t().contiguous(), lo.t().contiguous())
    h1 = ACTS[act](torch.randn(M, 256, device="cuda", generator=g))
    x = torch.randn(M, K, device="cuda", generator=g)
    return gz, w, planes_t, h1, x


def scratch(M, K):
    from torchrl_b200 import _lib
    return torch.full((int(_lib.load().trl_skinny_tn_scratch_floats(M, 256, K)),), float("nan"), device="cuda")


def unfused(gz, w, planes_t, h1, x, act):
    """The parent route: dH1 stored by the dgrad, then the skinny first-layer backward (partials and dW1 / db1)."""
    from torchrl_b200 import _lib, ops
    M, K = x.shape
    dh1 = ops.gemm3_pair(gz, w, planes=planes_t)
    part = scratch(M, K)
    _lib.call("trl_skinny_act_wgrad_partial", dh1.data_ptr(), h1.data_ptr(), x.data_ptr(), M, 256, K, act,
              part.data_ptr(), ops._stream())
    dw = torch.empty(256, K, device="cuda")
    db = torch.empty(256, device="cuda")
    _lib.call("trl_skinny_act_wgrad", dh1.data_ptr(), h1.data_ptr(), x.data_ptr(), dw.data_ptr(), db.data_ptr(), M, 256,
              K, act, scratch(M, K).data_ptr(), ops._stream())
    return part, dw, db


@pytest.mark.gpu
@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("K", [17, 23])
@pytest.mark.parametrize("M", [16384, 16421, 16896, 4096, 2048])
def test_fused_partials_equal_the_two_launch_route(M, K, act):
    from torchrl_b200 import ops
    from torchrl_b200.networks import fused
    gz, w, planes_t, h1, x = problem(M, K, act, seed=M + 31 * K + act)
    ref_part, ref_dw, ref_db = unfused(gz, w, planes_t, h1, x, act)
    part = ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x, act, scratch(M, K))
    torch.cuda.synchronize()
    assert same_bits(part, ref_part), "slab partials differ in %d entries" % int((part != ref_part).sum())
    # the immediate reduce (one job) and the deferred flush give the parent's dW1 / db1
    dw, db = torch.full_like(ref_dw, float("nan")), torch.full_like(ref_db, float("nan"))
    fused._reduce_jobs([(1, part, dw, db, M, 256, K, 0)])
    assert same_bits(dw, ref_dw) and same_bits(db, ref_db)
    dw2, db2 = torch.full_like(ref_dw, float("nan")), torch.full_like(ref_db, float("nan"))
    with fused.deferred_reduces():
        fused._DEFER.append((1, part, dw2, db2, M, 256, K, 0))
        fused.flush_reduces()
    assert same_bits(dw2, ref_dw) and same_bits(db2, ref_db)
    # and those are the first layer's gradients
    gz1 = ((gz.double() @ w.double()) * (1 - h1.double() ** 2 if act == 1 else (h1 > 0).double()))
    exact_dw = gz1.t() @ x.double()
    assert ((dw.double() - exact_dw).abs().max() / exact_dw.abs().max()).item() < 1e-4
    assert ((db.double() - gz1.sum(0)).abs().max() / gz1.sum(0).abs().max()).item() < 1e-4


@pytest.mark.gpu
def test_fused_partials_repeat_replay_and_run_on_two_streams():
    from torchrl_b200 import ops
    M, K, act = 16384, 17, 1
    gz, w, planes_t, h1, x = problem(M, K, act, seed=5)
    ref_part = unfused(gz, w, planes_t, h1, x, act)[0]
    outs = [ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x, act, scratch(M, K)) for _ in range(2)]
    # CUDA graph replay
    ws = scratch(M, K)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x, act, ws)       # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x, act, ws)
    ws.fill_(float("nan"))
    graph.replay()
    graph.replay()
    outs.append(ws)
    # two streams at once, each with its own scratch
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    w1, w2 = scratch(M, K), scratch(M, K)
    for s, buf in ((s1, w1), (s2, w2)):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x, act, buf)
    for s in (s1, s2):
        torch.cuda.current_stream().wait_stream(s)
    outs += [w1, w2]
    torch.cuda.synchronize()
    for i, o in enumerate(outs):
        assert same_bits(o, ref_part), "run %d differs in %d entries" % (i, int((o != ref_part).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("fork", [False, True])
def test_net_gradient_through_the_fused_dgrad(fork, monkeypatch):
    """A 17 -> 256 -> 256 -> 6 Net inside presplit + transposed_planes + direct_grad + deferred_reduces (the PPO
    minibatch body) takes the fused route and leaves the flat gradient the unfused entry points leave."""
    import contextlib

    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200 import ops
    from torchrl_b200.flat import FlatAdam
    from torchrl_b200.networks import fused
    torch.manual_seed(11)
    M = 16384
    net = networks.Net(input_shape=17, output_shape=6, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    opt = FlatAdam([net], lrs=[1e-3], eps=1e-5, max_norms=[0.5])
    x = torch.randn(M, 17, device="cuda")
    w = torch.randn(M, 6, device="cuda")
    calls = []
    real = ops.gemm3_pair_dgrad_act_wgrad
    monkeypatch.setattr(ops, "gemm3_pair_dgrad_act_wgrad", lambda *a: calls.append(1) or real(*a))

    def step(transposed):
        opt.zero_grad()
        tp = fused.transposed_planes(opt) if transposed else contextlib.nullcontext()
        with fused.presplit(), fused.direct_grad(), fused.deferred_reduces(), tp:
            y = net(x)
            with (fused.backward_fork() if fork else contextlib.nullcontext()):
                torch.autograd.backward([y], [w])
            n_jobs = len(fused._DEFER)
            fused.flush_reduces()
        torch.cuda.synchronize()
        return opt.grad.clone(), n_jobs, y.detach().clone()

    ref, ref_jobs, ref_y = step(False)
    assert not calls, "the fused dgrad ran outside transposed_planes()"
    got, jobs, y = step(True)
    assert len(calls) == 1, "the fused dgrad did not run"
    assert jobs == ref_jobs == 3
    assert same_bits(y, ref_y)
    assert float(ref.abs().max()) > 0
    assert same_bits(got, ref), "flat gradients differ in %d entries" % int((got != ref).sum())


def _rejects(native_lib, rc, needle):
    assert rc == -1
    msg = native_lib.trl_last_error().decode()
    assert needle in msg, msg


def test_fused_dgrad_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    p16 = p + (-p % 16)
    fn = native_lib.trl_gemm3_pair_dgrad_act_wgrad
    ok = (p16, p16, p16, p16, p16)
    _rejects(native_lib, fn(*ok, 16897, 17, 1, p16, None), "M=16897")
    _rejects(native_lib, fn(*ok, 0, 17, 1, p16, None), "M=0")
    for K in (0, 25, 64):
        _rejects(native_lib, fn(*ok, 16384, K, 1, p16, None), "1<=K<=24")
    _rejects(native_lib, fn(*ok, 16384, 17, 3, p16, None), "unknown activation")
    _rejects(native_lib, fn(*ok, 16384, 17, 1, None, None), "null pointer")
    _rejects(native_lib, fn(p16, p16, p16, None, p16, 16384, 17, 1, p16, None), "null pointer")
    for i in range(4):
        args = list(ok)
        args[i] = p16 + 4
        _rejects(native_lib, fn(*args, 16384, 17, 1, p16, None), "16-byte aligned")
    _rejects(native_lib, fn(*ok, 16384, 17, 1, p16 + 8, None), "16-byte aligned")
