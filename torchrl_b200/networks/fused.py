"""Linear (+ activation) layers of MLPBase (/root/reference/torchrl/networks/base.py:24-44) on this library's kernels.

Routing of one Linear layer (default matmul mode "tc3"):
  * 256 output units, reduction length a multiple of 32, >= _TC3_MIN_ROWS rows: the hand-written wgmma 3xTF32
    GEMM (csrc/gemm_pair.cu; fp32-faithful) -- forward with bias + activation in the register epilogue,
    dgrad reading the weights N-major (no transpose), wgrad with both operands M/N-major and deterministic split-K.
    Inside a `presplit()` scope the weights come as pre-split TF32 planes kept current by the fused Adam / Polyak
    kernels (flat.FlatParams.hi / .lo); elsewhere the kernel splits them in shared memory.
  * first layer (K = obs_dim <= 24) and output layer (<= 8 units): csrc/skinny.cu (fp32 kernels that stream one
    (M x H) matrix each, weights in registers).  Their weight / bias gradients are "per-CTA slabs, then a slab sum";
    inside `deferred_reduces()` (the fused minibatch body) only the first stages run and ONE launch sums all slabs.
  * anything else: cuBLAS fp32 SIMT + the fused bias/activation epilogues of csrc/mlp_epilogue.cu.
Numerically every route is fp32 arithmetic (3xTF32: 2e-6 relative at K = 256); the bias gradient is a fixed-order
two-level sum.
"""
import weakref

import torch
import torch.nn as nn

from .. import ops
from ..ops import split_tf32

ACT_CODES = {nn.Tanh: 1, nn.ReLU: 2}
_ENABLED = True
# "tc3"   : 256-wide layers with >= _TC3_MIN_ROWS rows on the hand-written wgmma 3xTF32 kernel
#           (csrc/gemm_pair.cu, fp32-faithful), skinny first / output layers on csrc/skinny.cu,
#           everything else cuBLAS fp32 SIMT                                                   [default]
# "fp32"  : cuBLAS fp32 SIMT sgemm everywhere
# "tf32x3": error-compensated TF32 through three cuBLAS GEMMs (kept for comparison; no faster than fp32)
_MATMUL_MODE = "tc3"
_TC3_MIN_ROWS = 2048             # below this the SIMT sgemm's latency wins
_TF32X3_MIN_DIM = 64             # layers narrower than this stay on the plain path


def set_matmul_mode(mode):
    """"tc3" (default): 256-wide layers on the wgmma 3xTF32 kernel, the rest cuBLAS fp32 SIMT; "fp32": cuBLAS
    fp32 SIMT everywhere; "tf32x3": x@w as x_hi@w_hi + x_lo@w_hi + x_hi@w_lo through three cuBLAS TF32 GEMMs
    (operands split by csrc/mlp_epilogue.cu:split_tf32_kernel; kept for comparison)."""
    global _MATMUL_MODE
    assert mode in ("fp32", "tf32x3", "tc3")
    _MATMUL_MODE = mode


# ---- pre-split weight planes ------------------------------------------------------------------------------------
_FLATS = weakref.WeakSet()       # live flat.FlatParams objects
_PLANES = {}                     # weight address -> (hi, lo) views into the owning FlatParams' planes
_PRESPLIT_DEPTH = 0
_TRANSPOSED = None               # the open transposed_planes scope
_T_STREAMS = {}


def _drop_planes(ptrs):
    for q in ptrs:
        _PLANES.pop(q, None)


def register_flat(flat):
    """Called by flat.FlatParams: remember its TF32 planes per 2-D parameter (dropped when the object dies)."""
    views = flat.plane_views()
    _PLANES.update(views)
    _FLATS.add(flat)
    weakref.finalize(flat, _drop_planes, list(views.keys()))


class presplit:
    """Scope in which the 256-wide layers read their weights from the pre-split planes.  On entry every live flat
    parameter buffer refreshes its planes from the current weights (one small launch each); inside the scope the
    weights may only change through the fused Adam / Polyak kernels or FlatParams.copy_from, which keep the planes
    current.  Used by the collectors' epochs and the agents' update loops; direct layer calls outside a scope split
    the weights in shared memory instead (always correct, 32 KB more conversion per stage)."""

    def __enter__(self):
        global _PRESPLIT_DEPTH
        if _PRESPLIT_DEPTH == 0 and _MATMUL_MODE == "tc3":
            for f in list(_FLATS):
                f.refresh_split()
        _PRESPLIT_DEPTH += 1
        return self

    def __exit__(self, *a):
        global _PRESPLIT_DEPTH
        _PRESPLIT_DEPTH -= 1


def presplit_scope(fn):
    """Decorator: run the method inside a `presplit()` scope."""
    import functools

    @functools.wraps(fn)
    def wrapped(*a, **k):
        with presplit():
            return fn(*a, **k)
    return wrapped


def _planes_of(weight):
    return _PLANES.get(weight.data_ptr()) if _PRESPLIT_DEPTH > 0 else None


class transposed_planes:
    """Scope inside `presplit()` in which the dgrad GEMMs of the square 256 x 256 weights of the given flat parameter
    buffers read transposed pre-split planes, i.e. K-major like the forward, instead of transposing the N-major weight
    tile in shared memory on every K block (same products, same bits).  On entry the buffers rewrite their transposed
    planes from their current hi / lo planes on a companion stream (under graph capture: a parallel branch); the first
    dgrad on each stream waits for them, and the exit joins the companion stream.  These weights must not change inside
    the scope before the last dgrad (the PPO / A2C minibatch body steps the optimizer after its backward passes)."""

    def __init__(self, *flats):
        self.flats = flats

    def __enter__(self):
        global _TRANSPOSED
        self.prev, self.event, self.joined, self.table = _TRANSPOSED, None, set(), {}
        if _PRESPLIT_DEPTH > 0 and _MATMUL_MODE == "tc3":
            self.main = torch.cuda.current_stream()
            key = self.main.cuda_stream
            if key not in _T_STREAMS:
                _T_STREAMS[key] = torch.cuda.Stream(device=self.main.device)
            self.side = _T_STREAMS[key]
            self.side.wait_stream(self.main)
            with torch.cuda.stream(self.side):
                for f in self.flats:
                    f.refresh_transposed()
                    self.table.update(f.transposed_views())
            self.event = torch.cuda.Event()
            self.event.record(self.side)
        _TRANSPOSED = self
        return self

    def __exit__(self, *a):
        global _TRANSPOSED
        _TRANSPOSED = self.prev
        if self.event is not None:
            self.main.wait_stream(self.side)

    def planes(self, weight):
        """(hi^T, lo^T) of `weight`, ready on the current stream, or None."""
        pl = self.table.get(weight.data_ptr()) if _PRESPLIT_DEPTH > 0 else None
        if pl is not None:
            st = torch.cuda.current_stream()
            if st.cuda_stream not in self.joined:
                st.wait_event(self.event)
                self.joined.add(st.cuda_stream)
        return pl


def mm_fwd(x, weight, bias=None, act=0):
    """act(x (M,K) @ weight (256,K)^T + bias) on the tensor cores."""
    return ops.gemm3_pair(x, weight, planes=_planes_of(weight), bias=bias, act=act)


def mm_dgrad(gz, weight):
    """gz (M,256) @ weight (256,256): inside `transposed_planes()` from the weight's transposed pre-split planes
    (K-major, the forward's route), elsewhere the pair kernel reads the weights N-major (no transpose)."""
    planes_t = _TRANSPOSED.planes(weight) if _TRANSPOSED is not None else None
    if planes_t is not None:
        return ops.gemm3_pair(gz, weight, planes=planes_t)
    return ops.gemm3_pair(gz, weight, planes=_planes_of(weight), b_nmajor=True)


def get_matmul_mode():
    return _MATMUL_MODE


def _tc3_ok(rows, n_out, k):
    """Shapes served by the hand-written wgmma 3xTF32 kernel (csrc/gemm_tf32x3.cu): 256 output columns,
    reduction length a multiple of 32, enough rows to fill the chip (one 128-row tile per CTA)."""
    return _MATMUL_MODE == "tc3" and rows >= _TC3_MIN_ROWS and n_out == 256 and k >= 32 and k % 32 == 0


def _stream_key():
    """Scratch buffers (split-K slabs, reduction partials, tickets) are per CUDA stream: the critic and the actor
    branch of a minibatch run concurrently on two streams (algo/on_policy/a2c.py) and must not share them."""
    return torch.cuda.current_stream().cuda_stream


_SCRATCH = {}
_SCRATCH_KINDS = {      # kind -> (fp32 elements, zeroed int32 tickets) for the sizes (M, H, K) of the launch
    "tn": lambda M, H, K: (ops.skinny_tn_scratch_floats(M, H, K), 0),      # skinny_tn / _act_wgrad slabs
    "dgrad_act": lambda M, H, K: (ops.skinny_dgrad_act_scratch_floats(M, H), 0),
    "bias_act": lambda M, H, K: (max(ops.bias_act_bwd_scratch_floats(M, H), 4), (H + 127) // 128),
    "cluster": lambda M, H, K: (8 * H * 256, H // 8),                      # gemm3_pair_tn_cluster, H output rows
}


def _scratch(kind, device, M=0, H=0, K=0, job=None):
    """The scratch of one kind of launch, allocated on first use and reused: a float32 tensor, or (float32, tickets)
    where the launch counts arrivals.  The float32 part is torch.empty (every launch writes its slabs before reading
    them); tickets start zeroed and the kernels leave them zero.  One buffer per stream (_stream_key), or with
    job = the kind of a deferred job: the buffer of the next _DEFER slot, whose slabs must survive until the flush."""
    key = (kind, M, H, K, str(device), _stream_key() if job is None else ("defer", len(_DEFER), job))
    ws = _SCRATCH.get(key)
    if ws is None:
        floats, tickets = _SCRATCH_KINDS[kind](M, H, K)
        ws = torch.empty(floats, dtype=torch.float32, device=device)
        if tickets:
            ws = ws, torch.zeros(tickets, dtype=torch.int32, device=device)
        _SCRATCH[key] = ws
    return ws


def wgrad(gz, x, out=None):
    """dW = gz^T @ x  for gz (M,H), x (M,K): split-K batched GEMM + partial sum.

    The direct `mm(gz.t(), x)` lands on a slow cuBLAS `nt` kernel for this shape class (tiny output, K =
    minibatch).  Splitting the reduction over S slabs exposes S x more
    CTAs; the S partial products are summed in a fixed order (deterministic)."""
    M, H = gz.shape
    K = x.shape[1]
    if _tc3_ok(M, K, M) and H % 128 == 0 and M % (32 * 64) == 0:
        # wgmma 3xTF32, operands consumed M/N-major from their row-major storage, deterministic split-K
        if H % 256 == 0:
            # split-K summed inside the launch (8 group partials + arrival tickets instead of 64 slabs)
            return ops.gemm3_pair_tn_cluster(gz, x, *_scratch("cluster", gz.device, H=H), out=out, splits=64)
        return ops.gemm_tf32x3_tn(gz, x, out=out, splits=64)
    if (_MATMUL_MODE != "fp32" and K <= 24 and H % 32 == 0 and H <= 256 and _skinny_ok(gz)
            and (out is None or out.is_contiguous())):
        return skinny_tn(gz, x, out=out)                 # (H,K) = gz^T x, first-layer weight gradient
    if H < 4 or M < 4096:
        return torch.mm(gz.t(), x, out=out) if out is not None else torch.mm(gz.t(), x)
    S = 16 if min(H, K) >= 128 else 64
    while S > 1 and M % S:
        S //= 2
    if S == 1:
        return torch.mm(gz.t(), x, out=out) if out is not None else torch.mm(gz.t(), x)
    m = M // S
    part = torch.bmm(gz.view(S, m, H).transpose(1, 2), x.view(S, m, K))
    return torch.sum(part, 0, out=out) if out is not None else part.sum(0)


def mm3(a_hi, a_lo, b_hi, b_lo):
    """a@b from pre-split operands: three TF32 tensor-core GEMMs accumulated in fp32."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        out = torch.mm(a_lo, b_hi)
        out.addmm_(a_hi, b_lo)
        out.addmm_(a_hi, b_hi)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return out


_DIRECT_GRAD = False
_FORK = None
_FORK_STREAMS = {}


class backward_fork:
    """Scope around ONE `torch.autograd.backward` call of an MLP with a fused tail: the weight-gradient work that nothing
    downstream in that backward pass depends on (the 256 x 256 wgrad GEMM) is issued on a companion stream while the
    dgrad GEMM and the first-layer backward continue on the calling stream; the scope's exit joins the two (under
    graph capture: a parallel branch).  Tensors the companion stream reads are kept alive until the join.  Outside
    such a scope the backward is strictly sequential."""

    def __enter__(self):
        global _FORK
        self.main = torch.cuda.current_stream()
        key = self.main.cuda_stream
        if key not in _FORK_STREAMS:
            _FORK_STREAMS[key] = torch.cuda.Stream(device=self.main.device)
        self.side = _FORK_STREAMS[key]
        self.keep, self.used, self.prev = [], False, _FORK
        _FORK = self
        return self

    def __exit__(self, *a):
        global _FORK
        _FORK = self.prev
        if self.used:
            self.main.wait_stream(self.side)
        self.keep.clear()


def _fork_here():
    f = _FORK
    if f is not None and torch.cuda.current_stream().cuda_stream == f.main.cuda_stream:
        return f
    return None


class direct_grad:
    """Context manager: inside it the fused layers write weight / bias gradients STRAIGHT into the parameters'
    pre-allocated `.grad` storage (views of the agent's flat gradient buffer, zeroed by the fused Adam step) and
    return None to autograd, which removes one AccumulateGrad add-kernel per parameter tensor.  Valid only
    when every parameter receives exactly one gradient contribution per backward and `.grad` is zero on
    entry -- true for the PPO minibatch update, which is the only user."""

    def __enter__(self):
        global _DIRECT_GRAD
        self.prev = _DIRECT_GRAD
        _DIRECT_GRAD = True

    def __exit__(self, *a):
        global _DIRECT_GRAD
        _DIRECT_GRAD = self.prev


def _grad_out(param):
    """The parameter's own `.grad` storage when direct mode is on (else None)."""
    return param.grad if (_DIRECT_GRAD and param.grad is not None) else None


def set_fused_epilogue(flag):
    """Globally enable/disable the fused epilogue path (default on for CUDA inputs)."""
    global _ENABLED
    _ENABLED = bool(flag)


def fused_enabled():
    return _ENABLED


_SKINNY_MIN_ROWS = 1024
_SKINNY = True         # csrc/skinny.cu serves the first (K = obs_dim) and output (N <= 8) layers


def set_skinny(flag):
    """Route the first (K = obs_dim <= 24) and output (N <= 8) Linear layers through csrc/skinny.cu (default on).
    scripts/skinny_probe.py times them against cuBLAS.  `set_skinny(False)` restores cuBLAS for these layers."""
    global _SKINNY
    _SKINNY = bool(flag)


def _skinny_ok(x):
    return _SKINNY and _ENABLED and x.is_cuda and x.shape[0] >= _SKINNY_MIN_ROWS


# ---- deferred second stages ---------------------------------------------------------------------------------------------
# Every skinny weight / bias gradient is "per-CTA slabs, then a small kernel that sums the slabs".  Inside a
# `deferred_reduces()` scope (the fused minibatch body, where gradients go straight into the flat buffer and nobody reads
# them before the optimizer) only the first stages are launched; `flush_reduces()` sums the slabs of ALL pending jobs in
# ONE launch (trl_skinny_reduce_jobs): six few-microsecond launches per PPO minibatch become one.
_DEFER = None           # list of pending jobs while a scope is open (backward runs on autograd threads: module state)


class deferred_reduces:
    def __enter__(self):
        global _DEFER
        self._prev = _DEFER
        _DEFER = []
        return self

    def __exit__(self, *exc):
        global _DEFER
        jobs, _DEFER = _DEFER, self._prev
        if jobs and exc[0] is None:
            raise RuntimeError("deferred_reduces: %d pending jobs; call flush_reduces() inside the scope" % len(jobs))
        return False


def flush_reduces():
    """Second stages of every job recorded since the scope opened, on the current stream (which must already be ordered
    after the streams the first stages ran on)."""
    global _DEFER
    jobs = _DEFER
    if not jobs:
        return
    for i in range(0, len(jobs), 8):
        _reduce_jobs(jobs[i:i + 8])
    _DEFER = []


_reduce_jobs = ops.skinny_reduce_jobs          # one launch for up to 8 jobs of the _DEFER tuple format


def _can_defer(*outs):
    """Deferral is only sound when every output is a slice of the flat gradient buffer (direct_grad): autograd would
    otherwise accumulate a tensor that is not complete yet."""
    return _DEFER is not None and all(o is not None for o in outs)


def skinny_tn(a, b, out=None, colsum=None, out_transposed=False):
    """out = a^T @ b for a (M,H), b (M,K<=32) [+ colsum = b.sum(0)]: csrc/skinny.cu, two deterministic stages."""
    M, H = a.shape
    K = b.shape[1]
    if out is None:
        out = torch.empty((K, H) if out_transposed else (H, K), dtype=torch.float32, device=a.device)
    return ops.skinny_tn(a, b, out, colsum, out_transposed, _scratch("tn", a.device, M, H, K))


class _LinearAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, act):
        tc = (_MATMUL_MODE == "tf32x3" and min(x.shape[0], x.shape[1], weight.shape[0]) >= _TF32X3_MIN_DIM)
        if _first_skinny_ok(x, weight, bias):
            # skinny first layer: GEMM + bias + activation in one memory-bound launch
            z = ops.skinny_k_fwd(x, weight, bias, act)
            ctx.save_for_backward(x, weight, z)
            ctx.act, ctx.tc, ctx.params = act, False, (weight, bias)
            return z
        if _tc3_ok(x.shape[0], weight.shape[0], x.shape[1]) and weight.is_contiguous():
            # wgmma: act(x (M,K) . W (256,K)^T + b), bias + activation fused into the epilogue
            z = mm_fwd(x, weight, bias=bias, act=act)
            ctx.save_for_backward(x, weight, z)
            ctx.act, ctx.tc, ctx.params = act, False, (weight, bias)
            return z
        elif tc:
            x_hi, x_lo = split_tf32(x)
            w_hi, w_lo = split_tf32(weight)
            z = mm3(x_hi, x_lo, w_hi.t(), w_lo.t())
            ctx.save_for_backward(x_hi, x_lo, w_hi, w_lo, z)
        else:
            z = torch.mm(x, weight.t())
            ctx.save_for_backward(x, weight, z)
        ops.bias_act_fwd(z, bias, act)
        ctx.act = act
        ctx.tc = tc
        ctx.params = (weight, bias)        # the Parameter objects themselves (for direct-grad mode)
        return z

    @staticmethod
    def backward(ctx, g):
        if ctx.tc:
            return _LinearAct._backward_tc(ctx, g)
        x, weight, y = ctx.saved_tensors
        return _linear_act_bwd(g, x, weight, y, ctx.act, ctx.params, ctx.needs_input_grad) + (None,)


def _first_skinny_ok(x, weight, bias):
    """The skinny first-layer forward (csrc/skinny.cu k_fwd) serves x (M, K <= 24) . weight^T."""
    return (_MATMUL_MODE != "fp32" and _skinny_ok(x) and x.shape[1] <= 24 and weight.shape[0] % 4 == 0
            and weight.shape[0] <= 1024 and weight.is_contiguous() and bias.is_contiguous())


def _act_wgrad_ok(x, y, dw_out):
    """The first layer's weight / bias gradient (its input needs no gradient) runs as ONE skinny pass over g and y."""
    H = y.shape[1]
    return (_MATMUL_MODE != "fp32" and _skinny_ok(y) and x.shape[1] <= 24 and H % 32 == 0 and H <= 256
            and x.is_contiguous() and (dw_out is None or dw_out.is_contiguous()))


def _linear_act_bwd(g, x, weight, y, act, params, needs_input_grad):
    """(dx, dW, db) of y = act(x W^T + b) for the upstream gradient g (None where not needed / written directly)."""
    g = g if g.is_contiguous() else g.contiguous()
    M, H = y.shape
    w_param, b_param = params
    db_out, dw_out = _grad_out(b_param), _grad_out(w_param)
    db = db_out if db_out is not None else torch.empty(H, dtype=torch.float32, device=y.device)
    K = x.shape[1]
    if not needs_input_grad[0] and _act_wgrad_ok(x, y, dw_out):
        # first layer (its input needs no gradient): dW and db straight from g and y in ONE pass over the
        # (M, H) matrices; the activation gradient gz is never written to memory
        dw = dw_out if dw_out is not None else torch.empty(H, K, dtype=torch.float32, device=y.device)
        if _can_defer(dw_out, db_out):
            ws = _scratch("tn", y.device, M, H, K, job=1)
            ops.skinny_act_wgrad_partial(g, y, x, act, ws)
            _DEFER.append((1, ws, dw, db, M, H, K, 0))
            return None, None, None
        ops.skinny_act_wgrad(g, y, x, dw, db, act, _scratch("tn", y.device, M, H, K))
        return None, None if dw_out is not None else dw, None if db_out is not None else db
    gz = torch.empty_like(y)
    ops.bias_act_bwd(g, y, gz, db, act, *_scratch("bias_act", y.device, M, H))
    dx = None
    if needs_input_grad[0]:
        if _tc3_ok(M, weight.shape[1], H) and weight.is_contiguous():
            dx = mm_dgrad(gz, weight)
        else:
            dx = torch.mm(gz, weight)
    dw = wgrad(gz, x, out=dw_out) if needs_input_grad[1] else None
    return (dx, None if dw_out is not None else dw,
            None if db_out is not None else (db if needs_input_grad[2] else None))


def _backward_tc(ctx, g):
    x_hi, x_lo, w_hi, w_lo, y = ctx.saved_tensors
    g = g if g.is_contiguous() else g.contiguous()
    M, H = y.shape
    gz = torch.empty_like(y)
    db = torch.empty(H, dtype=torch.float32, device=y.device)
    ops.bias_act_bwd(g, y, gz, db, ctx.act, *_scratch("bias_act", y.device, M, H))
    g_hi, g_lo = split_tf32(gz)
    dx = mm3(g_hi, g_lo, w_hi, w_lo) if ctx.needs_input_grad[0] else None
    dw = mm3(g_hi.t(), g_lo.t(), x_hi, x_lo) if ctx.needs_input_grad[1] else None
    return dx, dw, (db if ctx.needs_input_grad[2] else None), None


_LinearAct._backward_tc = staticmethod(_backward_tc)


class _LinearPlain(torch.autograd.Function):
    """Linear without activation (the output layer of Net): cuBLAS forward, split-K wgrad backward."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.params = (weight, bias)
        N, H = weight.shape
        ctx.skinny = (_MATMUL_MODE != "fp32" and _skinny_ok(x) and N <= 8 and H in (128, 256)
                      and weight.is_contiguous())
        if ctx.skinny:
            return ops.skinny_n_fwd(x, weight, bias)
        return torch.addmm(bias, x, weight.t())

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        g = g if g.is_contiguous() else g.contiguous()
        w_param, b_param = ctx.params
        db_out, dw_out = _grad_out(b_param), _grad_out(w_param)
        if ctx.skinny:
            N = weight.shape[0]
            dx = ops.skinny_n_dgrad(g, weight) if ctx.needs_input_grad[0] else None
            db = db_out if db_out is not None else torch.empty(N, dtype=torch.float32, device=x.device)
            dw = skinny_tn(x, g, out=dw_out, colsum=db, out_transposed=True)     # dW (N,H) = g^T x, db = sum g
            return dx, None if dw_out is not None else dw, None if db_out is not None else db
        dx = torch.mm(g, weight) if ctx.needs_input_grad[0] else None
        dw = wgrad(g, x, out=dw_out) if ctx.needs_input_grad[1] else None
        db = None
        if ctx.needs_input_grad[2]:
            db = torch.sum(g, 0, out=db_out) if db_out is not None else g.sum(0)
        return dx, None if dw_out is not None else dw, None if db_out is not None else db


class _MLPTail(torch.autograd.Function):
    """Last hidden layer + output layer of an MLP head as ONE autograd node, optionally with a skinny first layer:
        h1 = act1(x W1^T + b1)  (csrc/skinny.cu k_fwd; only when w1 is given, x then needs no gradient)
        y2 = act(h1 W2^T + b2)  (wgmma 3xTF32, bias + activation in the epilogue)
        out = y2 W3^T + b3      (csrc/skinny.cu n_fwd)
    The hidden layer is 256 wide: that is the width which admits the wgmma GEMM (tail_ok), and the width the output
    layer's fused backward serves.  So the backward runs the output layer's whole backward and the activation backward
    of the hidden layer as one pass over y2 (trl_skinny_n_dgrad_act_wgrad: gz2 and db2, the (M, 256) dgrad matrix
    never stored un-activated, and the output layer's dW3 / db3 slab partials, bit for bit those of skinny_tn; the
    companion stream carries the wgrad alone), and, with the first layer, the dgrad dH1 = gz2 W2 with the first
    layer's weight / bias gradient: inside `transposed_planes()` trl_gemm3_pair_dgrad_act_wgrad reduces dH1 to
    dW1 / db1 slab partials in its epilogue, so dH1 is never stored (elsewhere: mm_dgrad, then the skinny first-layer
    backward, the same bits)."""

    @staticmethod
    def forward(ctx, x, w1, b1, act1, w2, b2, w3, b3, act):
        assert w2.shape[0] == 256 == w3.shape[1], "_MLPTail needs a 256-wide hidden layer"
        h1 = ops.skinny_k_fwd(x, w1, b1, act1) if w1 is not None else x
        y2 = mm_fwd(h1, w2, bias=b2, act=act)
        out = ops.skinny_n_fwd(y2, w3, b3)
        ctx.save_for_backward(x, w1, h1, w2, y2, w3)
        ctx.act, ctx.act1 = act, act1
        ctx.params = (w1, b1, w2, b2, w3, b3)
        return out

    @staticmethod
    def backward(ctx, g):
        x0, w1, x, w2, y2, w3 = ctx.saved_tensors
        g = g if g.is_contiguous() else g.contiguous()
        M, H = y2.shape
        N = w3.shape[0]
        dev = y2.device
        w1p, b1p, w2p, b2p, w3p, b3p = ctx.params
        dw2_out, db2_out, dw3_out, db3_out = _grad_out(w2p), _grad_out(b2p), _grad_out(w3p), _grad_out(b3p)
        db2 = db2_out if db2_out is not None else torch.empty(H, dtype=torch.float32, device=dev)
        db3 = db3_out if db3_out is not None else torch.empty(N, dtype=torch.float32, device=dev)
        gz = torch.empty_like(y2)
        dw3 = dw3_out if dw3_out is not None else torch.empty(N, H, dtype=torch.float32, device=dev)
        # gz2, db2 and dW3 (N,H) = g^T y2, db3 = sum g in one pass over y2
        if _can_defer(db2_out, dw3_out, db3_out) and len(_DEFER) < 63:     # two more jobs, at most 64 pending
            ws = _scratch("dgrad_act", dev, M, H, job=2)
            _DEFER.append((2, ws, None, db2, M, H, 0, 0))
            ws3 = _scratch("tn", dev, M, H, N, job=0)
            _DEFER.append((0, ws3, dw3, db3, M, H, N, 1))
            ops.skinny_n_dgrad_act_wgrad_partial(g, w3, y2, ctx.act, gz, ws, ws3)
        else:
            ops.skinny_n_dgrad_act_wgrad(g, w3, y2, ctx.act, gz, db2, dw3, db3, _scratch("dgrad_act", dev, M, H),
                                         _scratch("tn", dev, M, H, N))
        first = w1 is not None
        want_dx = ctx.needs_input_grad[0] and not first
        fk = _fork_here() if dw2_out is not None and dw3_out is not None else None
        if fk is not None:
            # the weight gradient that feeds nothing but the optimizer: companion stream (see backward_fork)
            fk.side.wait_stream(fk.main)
            with torch.cuda.stream(fk.side):
                dw2 = wgrad(gz, x, out=dw2_out)
            fk.keep += [gz, x]
            fk.used = True
        first_grads = _first_layer_bwd(ctx, gz, x0, w1, x, w2) if first else None
        dx = mm_dgrad(gz, w2) if want_dx else None
        if fk is None:
            dw2 = wgrad(gz, x, out=dw2_out)
        tail = (None if dw2_out is not None else dw2, None if db2_out is not None else db2,
                None if dw3_out is not None else dw3, None if db3_out is not None else db3, None)
        if first:
            return (None,) + first_grads + (None,) + tail
        return (dx, None, None, None) + tail


def _first_layer_bwd(ctx, gz, x0, w1, h1, w2):
    """(dW1, db1) from gz2: dH1 = gz2 W2 feeds nothing else (x0 needs no gradient).  Inside `transposed_planes()`
    the dgrad's epilogue forms the first layer's slab partials (dH1 never stored); elsewhere mm_dgrad, then the
    skinny first-layer backward.  The slab sums are the same kernels either way: deferred inside deferred_reduces()."""
    M, H = h1.shape
    K = x0.shape[1]
    w1p, b1p = ctx.params[0], ctx.params[1]
    dw_out, db_out = _grad_out(w1p), _grad_out(b1p)
    planes_t = (_TRANSPOSED.planes(w2) if _TRANSPOSED is not None and H == 256
                and tuple(w2.shape) == (256, 256) else None)
    if planes_t is None or M > _DGRAD_FIRST_MAX_ROWS or not _act_wgrad_ok(x0, h1, dw_out):
        return _linear_act_bwd(mm_dgrad(gz, w2), x0, w1, h1, ctx.act1, (w1p, b1p), (False, True, True))[1:]
    dw = dw_out if dw_out is not None else torch.empty(H, K, dtype=torch.float32, device=h1.device)
    db = db_out if db_out is not None else torch.empty(H, dtype=torch.float32, device=h1.device)
    if _can_defer(dw_out, db_out):
        ws = _scratch("tn", h1.device, M, H, K, job=1)
        ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x0, ctx.act1, ws)
        _DEFER.append((1, ws, dw, db, M, H, K, 0))
        return None, None
    ws = _scratch("tn", h1.device, M, H, K)
    ops.gemm3_pair_dgrad_act_wgrad(gz, planes_t, h1, x0, ctx.act1, ws)
    _reduce_jobs([(1, ws, dw, db, M, H, K, 0)])
    return None if dw_out is not None else dw, None if db_out is not None else db


_DGRAD_FIRST_MAX_ROWS = 16896    # trl_gemm3_pair_dgrad_act_wgrad: slabs of at most 64 rows (sk_rows_per_cta)


def tail_ok(h, fc, act_module, head):
    """True when `head(act(fc(h)))` can run as one _MLPTail node: 256-wide hidden layer on the wgmma kernel, an
    output layer of at most 8 units, enough rows, gradients being recorded."""
    if not (_ENABLED and _SKINNY and h.is_cuda and h.dtype == torch.float32):
        return False
    rows = h.numel() // h.shape[-1]
    return (type(act_module) in ACT_CODES and rows >= max(_TC3_MIN_ROWS, _SKINNY_MIN_ROWS)
            and _tc3_ok(rows, fc.out_features, fc.in_features) and head.in_features == fc.out_features
            and head.out_features <= 8 and fc.bias is not None and head.bias is not None
            and fc.weight.is_contiguous() and head.weight.is_contiguous())


def first_ok(x, fc, act_module):
    """True when act(fc(x)) can open an _MLPTail node as its skinny first layer: x needs no gradient and the layer
    takes the skinny forward of _LinearAct."""
    if not (can_fuse(x, fc, act_module) and not x.requires_grad and x.dim() >= 1):
        return False
    return _first_skinny_ok(x.reshape(-1, x.shape[-1]), fc.weight, fc.bias)


def mlp_tail(h, fc, act_code, head, first=None):
    """head(act(fc(h))) as one _MLPTail node; first = (fc1, act1_code): h is the input of that skinny first layer."""
    lead = h.shape[:-1]
    h2 = h.reshape(-1, h.shape[-1])
    if not h2.is_contiguous():
        h2 = h2.contiguous()
    w1, b1, act1 = (first[0].weight, first[0].bias, first[1]) if first is not None else (None, None, 0)
    out = _MLPTail.apply(h2, w1, b1, act1, fc.weight, fc.bias, head.weight, head.bias, act_code)
    return out.reshape(tuple(lead) + (out.shape[-1],))


def linear_plain(x, fc):
    lead = x.shape[:-1]
    x2 = x.reshape(-1, x.shape[-1])
    if not x2.is_contiguous():
        x2 = x2.contiguous()
    out = _LinearPlain.apply(x2, fc.weight, fc.bias)
    return out.reshape(tuple(lead) + (out.shape[-1],))


def linear_act(x, fc, act_code):
    """act(fc(x)) through the fused path; x may have any number of leading dims."""
    lead = x.shape[:-1]
    x2 = x.reshape(-1, x.shape[-1])
    if not x2.is_contiguous():
        x2 = x2.contiguous()
    out = _LinearAct.apply(x2, fc.weight, fc.bias, act_code)
    return out.reshape(tuple(lead) + (out.shape[-1],))


def can_fuse(x, fc, act_module):
    return (_ENABLED and x.is_cuda and x.dtype == torch.float32 and type(act_module) in ACT_CODES
            and fc.out_features % 4 == 0 and fc.bias is not None)
