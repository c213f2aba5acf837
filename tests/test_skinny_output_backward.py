"""The output layer's whole backward in one pass over y2 (trl_skinny_n_dgrad_act_wgrad): besides gz2 = (g W3) * act'(y2)
and the hidden layer's bias-gradient slabs, the launch writes the output layer's weight / bias gradient slab partials
(dW3 = g^T y2, db3 = colsum(g)).  Everything must be bit-identical to the two-launch route it replaces
(trl_skinny_n_dgrad_act_partial, then trl_skinny_tn_partial), and so must the final dW3 / db3 / db2 through the
immediate form and the deferred flush, at every slab size the skinny kernels use: 63-row slabs at M = 16384, a ragged
last slab, 64-row slabs at M = 16896, and 16- and 8-row slabs.

Scratch buffers and outputs are NaN-filled (a slab no CTA wrote shows up), calls are repeated, replayed from a CUDA graph
and run on two streams at once.  The argument checks need no GPU.
"""
import ctypes

import pytest
import torch

ACTS = {1: torch.tanh, 2: torch.relu}
H = 256


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def problem(M, N, act, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    grad = torch.randn(M, N, device="cuda", generator=g)
    w3 = torch.randn(N, H, device="cuda", generator=g) / 16
    y2 = ACTS[act](torch.randn(M, H, device="cuda", generator=g))
    return grad, w3, y2


def scratches(M, N):
    from torchrl_b200 import _lib
    lib = _lib.load()
    return nan(int(lib.trl_skinny_dgrad_act_scratch_floats(M, H))), nan(int(lib.trl_skinny_tn_scratch_floats(M, H, N)))


def two_launch(grad, w3, y2, act):
    """The parent route: the output-layer dgrad + activation backward, then skinny_tn over the same y2 and g (partials
    and the immediate dW3 / db3 / db2)."""
    from torchrl_b200 import _lib, ops
    M, N = grad.shape
    gz, (ws2, ws3) = nan(M, H), scratches(M, N)
    _lib.call("trl_skinny_n_dgrad_act_partial", grad.data_ptr(), w3.data_ptr(), y2.data_ptr(), gz.data_ptr(), M, H, N,
              act, ws2.data_ptr(), ops._stream())
    _lib.call("trl_skinny_tn_partial", y2.data_ptr(), grad.data_ptr(), M, H, N, 1, ws3.data_ptr(), ops._stream())
    db2, dw3, db3 = nan(H), nan(N, H), nan(N)
    s2, s3 = scratches(M, N)
    _lib.call("trl_skinny_n_dgrad_act", grad.data_ptr(), w3.data_ptr(), y2.data_ptr(), nan(M, H).data_ptr(),
              db2.data_ptr(), M, H, N, act, s2.data_ptr(), ops._stream())
    _lib.call("trl_skinny_tn", y2.data_ptr(), grad.data_ptr(), dw3.data_ptr(), db3.data_ptr(), M, H, N, 1,
              s3.data_ptr(), ops._stream())
    return (gz, ws2, ws3), (db2, dw3, db3)


def fused_partial(grad, w3, y2, act):
    from torchrl_b200 import ops
    M, N = grad.shape
    gz, (ws2, ws3) = nan(M, H), scratches(M, N)
    ops.skinny_n_dgrad_act_wgrad_partial(grad, w3, y2, act, gz, ws2, ws3)
    return gz, ws2, ws3


def assert_same(got, ref, names):
    for name, a, b in zip(names, got, ref):
        assert same_bits(a, b), "%s differs in %d entries" % (name, int((a.view(torch.int32) != b.view(torch.int32)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("N", [1, 6, 8])
@pytest.mark.parametrize("M", [16384, 16421, 16896, 4096, 2048])
def test_fused_pass_equals_the_two_launch_route(M, N, act):
    from torchrl_b200 import ops
    from torchrl_b200.networks import fused
    grad, w3, y2 = problem(M, N, act, seed=M + 31 * N + act)
    ref_part, ref_out = two_launch(grad, w3, y2, act)
    part = fused_partial(grad, w3, y2, act)
    torch.cuda.synchronize()
    assert_same(part, ref_part, ("gz", "db2 slabs", "dW3 / db3 slabs"))
    # the immediate form (one reduce launch for both) and the deferred flush give the parent's db2 / dW3 / db3
    out = nan(H), nan(N, H), nan(N)
    gz = nan(M, H)
    ops.skinny_n_dgrad_act_wgrad(grad, w3, y2, act, gz, *out, *scratches(M, N))
    assert_same((gz,) + out, (ref_part[0],) + ref_out, ("gz", "db2", "dW3", "db3"))
    out2 = nan(H), nan(N, H), nan(N)
    with fused.deferred_reduces():
        fused._DEFER.append((2, part[1], None, out2[0], M, H, 0, 0))
        fused._DEFER.append((0, part[2], out2[1], out2[2], M, H, N, 1))
        fused.flush_reduces()
    assert_same(out2, ref_out, ("db2", "dW3", "db3"))
    # and those are the output layer's gradients.  Each entry is an fp32 sum whose longest chain is about 80 additions
    # (<= 32 rows per row lane, the lane combine, <= 9 slabs per reduce group, 32 group sums), so its error is below
    # 80 * 2^-24 * (sum of the absolute terms) < 1e-5 * that sum; the sums cancel, so the bound is not relative to them.
    exact_dw = grad.double().t() @ y2.double()
    assert ((out[1].double() - exact_dw).abs() <= 1e-5 * (grad.double().abs().t() @ y2.double().abs())).all()
    exact_db = grad.double().sum(0)
    assert ((out[2].double() - exact_db).abs() <= 1e-5 * grad.double().abs().sum(0)).all()


@pytest.mark.gpu
def test_fused_pass_repeats_replays_and_runs_on_two_streams():
    from torchrl_b200 import ops
    M, N, act = 16384, 6, 1
    grad, w3, y2 = problem(M, N, act, seed=5)
    ref = two_launch(grad, w3, y2, act)[0]
    outs = [fused_partial(grad, w3, y2, act) for _ in range(2)]
    # CUDA graph replay
    bufs = (nan(M, H),) + scratches(M, N)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.skinny_n_dgrad_act_wgrad_partial(grad, w3, y2, act, *bufs)           # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.skinny_n_dgrad_act_wgrad_partial(grad, w3, y2, act, *bufs)
    for b in bufs:
        b.fill_(float("nan"))
    graph.replay()
    graph.replay()
    outs.append(bufs)
    # two streams at once, each with its own buffers
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    b1, b2 = (nan(M, H),) + scratches(M, N), (nan(M, H),) + scratches(M, N)
    for s, b in ((s1, b1), (s2, b2)):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.skinny_n_dgrad_act_wgrad_partial(grad, w3, y2, act, *b)
    for s in (s1, s2):
        torch.cuda.current_stream().wait_stream(s)
    outs += [b1, b2]
    torch.cuda.synchronize()
    for i, o in enumerate(outs):
        assert_same(o, ref, ("run %d gz" % i, "run %d db2 slabs" % i, "run %d dW3 / db3 slabs" % i))


@pytest.mark.gpu
@pytest.mark.parametrize("scope", ["minibatch", "minibatch_fork", "plain"])
def test_net_gradient_through_the_fused_pass(scope, monkeypatch):
    """A 17 -> 256 -> 256 -> 6 Net takes the fused pass, inside the PPO minibatch scopes (deferred slab sums, with and
    without the companion stream) and outside them (immediate form, gradients through autograd), and leaves the
    gradients that the two-launch route leaves."""
    import contextlib

    import torch.nn as nn
    import torchrl_b200.networks as networks
    from torchrl_b200 import _lib, ops
    from torchrl_b200.flat import FlatAdam
    from torchrl_b200.networks import fused
    torch.manual_seed(11)
    M, N = 16384, 6
    net = networks.Net(input_shape=17, output_shape=N, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    opt = FlatAdam([net], lrs=[1e-3], eps=1e-5, max_norms=[0.5])
    x = torch.randn(M, 17, device="cuda")
    w = torch.randn(M, N, device="cuda")
    calls = []

    def unfused_partial(g, w3, y, act, gz, ws2, ws3):
        _lib.call("trl_skinny_n_dgrad_act_partial", g.data_ptr(), w3.data_ptr(), y.data_ptr(), gz.data_ptr(), M, H, N,
                  act, ws2.data_ptr(), ops._stream())
        _lib.call("trl_skinny_tn_partial", y.data_ptr(), g.data_ptr(), M, H, N, 1, ws3.data_ptr(), ops._stream())

    def unfused(g, w3, y, act, gz, db, dw, dbias, ws2, ws3):
        _lib.call("trl_skinny_n_dgrad_act", g.data_ptr(), w3.data_ptr(), y.data_ptr(), gz.data_ptr(), db.data_ptr(), M,
                  H, N, act, ws2.data_ptr(), ops._stream())
        _lib.call("trl_skinny_tn", y.data_ptr(), g.data_ptr(), dw.data_ptr(), dbias.data_ptr(), M, H, N, 1,
                  ws3.data_ptr(), ops._stream())

    real = ops.skinny_n_dgrad_act_wgrad_partial, ops.skinny_n_dgrad_act_wgrad
    count = lambda f: lambda *a: calls.append(1) or f(*a)

    def step(reference):
        monkeypatch.setattr(ops, "skinny_n_dgrad_act_wgrad_partial", unfused_partial if reference else count(real[0]))
        monkeypatch.setattr(ops, "skinny_n_dgrad_act_wgrad", unfused if reference else count(real[1]))
        if scope == "plain":
            y = net(x)
            grads = torch.autograd.grad([y], list(net.parameters()), [w])
            torch.cuda.synchronize()
            return torch.cat([t.reshape(-1) for t in grads]), y.detach().clone()
        opt.zero_grad()
        fork = fused.backward_fork() if scope == "minibatch_fork" else contextlib.nullcontext()
        with fused.presplit(), fused.direct_grad(), fused.deferred_reduces(), fused.transposed_planes(opt):
            y = net(x)
            with fork:
                torch.autograd.backward([y], [w])
            assert len(fused._DEFER) == 3
            fused.flush_reduces()
        torch.cuda.synchronize()
        return opt.grad.clone(), y.detach().clone()

    ref, ref_y = step(True)
    assert not calls
    got, y = step(False)
    assert len(calls) == 1, "the fused output-layer pass did not run"
    assert same_bits(y, ref_y)
    assert float(ref.abs().max()) > 0
    assert same_bits(got, ref), "gradients differ in %d entries" % int((got != ref).sum())


def _rejects(native_lib, rc, needle):
    assert rc == -1
    msg = native_lib.trl_last_error().decode()
    assert needle in msg, msg


def test_fused_pass_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    p16 = p + (-p % 16)
    part = native_lib.trl_skinny_n_dgrad_act_wgrad_partial
    full = native_lib.trl_skinny_n_dgrad_act_wgrad
    ok = (p16, p16, p16, p16)
    for N in (0, 9):
        _rejects(native_lib, part(*ok, 16384, 256, N, 1, p16, p16, None), "1<=N<=8")
    for h in (128, 512):
        _rejects(native_lib, part(*ok, 16384, h, 6, 1, p16, p16, None), "H==256")
    _rejects(native_lib, part(*ok, 0, 256, 6, 1, p16, p16, None), "M=0")
    _rejects(native_lib, part(*ok, 16384, 256, 6, 3, p16, p16, None), "unknown activation")
    for i in range(4):
        args = list(ok)
        args[i] = None
        _rejects(native_lib, part(*args, 16384, 256, 6, 1, p16, p16, None), "null pointer")
    _rejects(native_lib, part(*ok, 16384, 256, 6, 1, None, p16, None), "null pointer")
    _rejects(native_lib, part(*ok, 16384, 256, 6, 1, p16, None, None), "null pointer")
    for i in (1, 2, 3):
        args = list(ok)
        args[i] = p16 + 4
        _rejects(native_lib, part(*args, 16384, 256, 6, 1, p16, p16, None), "16-byte aligned")
    _rejects(native_lib, part(*ok, 16384, 256, 6, 1, p16, p16 + 8, None), "16-byte aligned")
    for i in range(3):
        outs = [p16] * 3
        outs[i] = None
        _rejects(native_lib, full(*ok, *outs, 16384, 256, 6, 1, p16, p16, None), "null pointer")
    _rejects(native_lib, full(*ok, p16, p16, p16, 16384, 256, 9, 1, p16, p16, None), "1<=N<=8")
