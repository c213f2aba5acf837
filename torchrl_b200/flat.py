"""Flat parameter / gradient buffers and the fused multi-segment Adam (K11, csrc/optim.cu).

A *segment* is the parameter set of one optimizer of the reference (e.g. PPO: pf and vf,
/root/reference/torchrl/algo/on_policy/a2c.py:29-39).  All segments live in one contiguous fp32
buffer; ``nn.Parameter.data`` and ``.grad`` become views into it, so
  * global-norm clipping + Adam + zero_grad is two launches for the whole agent,
  * the multi-GPU path all-reduces ONE tensor (K12).
"""
import ctypes

import torch

from . import ops

F32, F64, I32 = torch.float32, torch.float64, torch.int32


def _params_of(seg):
    if isinstance(seg, torch.nn.Module):
        return [p for p in seg.parameters()]
    return list(seg)


class FlatParams:
    """Re-home the parameters of several segments into one flat buffer (data only)."""

    def __init__(self, segments, device=None):
        self.segments = [_params_of(s) for s in segments]
        plist = [p for seg in self.segments for p in seg]
        assert plist, "no parameters"
        self.device = torch.device(device) if device is not None else plist[0].device
        # every parameter starts on a 16-byte boundary (4 floats) so kernels can use float4 on weight /
        # bias views; the padding elements are zero, receive zero gradient and stay zero under Adam
        self.offsets = []
        self.seg_begin = [0]
        off = 0
        for seg in self.segments:
            for p in seg:
                off = (off + 3) // 4 * 4
                self.offsets.append(off)
                off += p.numel()
            off = (off + 3) // 4 * 4
            self.seg_begin.append(off)
        self.total = self.seg_begin[-1]
        self.data = torch.zeros(self.total, dtype=F32, device=self.device)
        for p, o in zip(plist, self.offsets):
            n = p.numel()
            self.data[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.data[o:o + n].view(p.shape)
        self.params = plist
        # TF32 planes of every parameter (hi = tf32(w), lo = w - hi) for the pre-split B operand of the CTA-pair
        # GEMM (csrc/gemm_pair.cu): written by the fused Adam / Polyak kernels, refreshed from `data` on entry
        # to a `networks.fused.presplit()` scope, looked up by the weight's address inside such a scope only.
        self.hi = torch.zeros(self.total, dtype=F32, device=self.device)
        self.lo = torch.zeros(self.total, dtype=F32, device=self.device)
        # the same planes transposed, for the square 256 x 256 weights only: the dgrad GEMM reads them K-major, like the
        # forward (written by refresh_transposed on entry to a `networks.fused.transposed_planes(flat)` scope)
        self._square = [(p, o) for p, o in zip(self.params, self.offsets) if tuple(p.shape) == (256, 256)]
        self.hi_t = torch.zeros(len(self._square), 256, 256, dtype=F32, device=self.device)
        self.lo_t = torch.zeros(len(self._square), 256, 256, dtype=F32, device=self.device)
        if self.device.type == "cuda":
            from .networks import fused
            fused.register_flat(self)

    def plane_views(self):
        """{weight address: (hi, lo)} for the 2-D parameters."""
        out = {}
        for p, o in zip(self.params, self.offsets):
            if p.dim() == 2:
                n = p.numel()
                out[p.data_ptr()] = (self.hi[o:o + n].view(p.shape), self.lo[o:o + n].view(p.shape))
        return out

    def transposed_views(self):
        """{weight address: (hi^T, lo^T)} for the square 256 x 256 weights."""
        return {p.data_ptr(): (self.hi_t[i], self.lo_t[i]) for i, (p, _) in enumerate(self._square)}

    def refresh_transposed(self):
        """hi_t / lo_t <- the transposes of the current hi / lo planes of the square weights."""
        for i, (_, o) in enumerate(self._square):
            ops.transpose_f32(self.hi[o:o + 65536].view(256, 256), out=self.hi_t[i])
            ops.transpose_f32(self.lo[o:o + 65536].view(256, 256), out=self.lo_t[i])

    def refresh_split(self):
        """Recompute both planes from `data` (one launch)."""
        ops.split_tf32(self.data, self.hi, self.lo)

    def copy_from(self, src_flat_data):
        """data <- src (a flat tensor of the same layout); the planes follow."""
        self.data.copy_(src_flat_data)
        self.refresh_split()

    def seg_slice(self, i, j=None):
        j = i + 1 if j is None else j
        return self.data[self.seg_begin[i]:self.seg_begin[j]]


class FlatAdam(FlatParams):
    """Adam over flat segments with per-segment lr / eps / max-norm, matching torch.optim.Adam +
    torch.nn.utils.clip_grad_norm_ applied per segment (the reference's per-network optimizers)."""

    def __init__(self, segments, lrs, eps=1e-8, max_norms=None, betas=(0.9, 0.999), device=None, dist=None):
        super().__init__(segments, device)
        n = len(self.segments)
        assert n <= 8
        self.nseg = n
        # data parallel over PeerComm (distributed.py): the flat gradient lives in a peer-mapped region so that the
        # fused all-reduce kernel reads it in place; `reduced` receives the sum over ranks
        region = dist.grad_buffer(self.total) if dist is not None and getattr(dist, "active", False) else None
        self._grad_region = region
        if region is not None:
            self.grad = region
            self.grad.zero_()
            self.reduced = torch.zeros(self.total, dtype=F32, device=self.device)
            self._comm_scratch = torch.zeros(ops.comm_scratch_doubles(n), dtype=F64, device=self.device)
        else:
            self.grad = torch.zeros(self.total, dtype=F32, device=self.device)
        self.exp_avg = torch.zeros(self.total, dtype=F32, device=self.device)
        self.exp_avg_sq = torch.zeros(self.total, dtype=F32, device=self.device)
        for p, o in zip(self.params, self.offsets):
            p.grad = self.grad[o:o + p.numel()].view(p.shape)
        lrs = [float(x) for x in (lrs if isinstance(lrs, (list, tuple)) else [lrs] * n)]
        eps = [float(x) for x in (eps if isinstance(eps, (list, tuple)) else [eps] * n)]
        if max_norms is None:
            max_norms = [0.0] * n
        max_norms = [0.0 if m is None else float(m) for m in (max_norms if isinstance(max_norms, (list, tuple))
                                                              else [max_norms] * n)]
        self.lr_host = torch.tensor(lrs, dtype=F32).pin_memory() if torch.cuda.is_available() else torch.tensor(lrs)
        self.lr = self.lr_host.to(self.device)
        self.initial_lrs = list(lrs)
        self.betas = (float(betas[0]), float(betas[1]))
        self.step_counts = torch.zeros(n, dtype=I32, device=self.device)
        self.sumsq3 = torch.zeros(3 * n, dtype=F64, device=self.device)
        self._scratch = torch.zeros(ops.grad_sumsq_blocks(n), dtype=F64, device=self.device)
        self._ticket = torch.zeros(1, dtype=I32, device=self.device)
        self._seg_c = (ctypes.c_int64 * (n + 1))(*self.seg_begin)
        self._max_norm_c = (ctypes.c_float * n)(*max_norms)
        self._eps_c = (ctypes.c_float * n)(*eps)
        self.all_mask = (1 << n) - 1

    def set_lr(self, seg, lr):
        """Host-side LR schedule (update_linear_schedule, /root/reference/torchrl/algo/utils.py:28-32):
        the value goes to a device scalar so captured graphs pick it up without re-capture."""
        self.lr_host[seg] = float(lr)
        self.lr.copy_(self.lr_host, non_blocking=True)

    def zero_grad(self):
        self.grad.zero_()

    def step(self, active_mask=None, grad_scale=1.0, zero_grad=True, reduced=False):
        """clip (per segment, global norm) + Adam + zero the gradient: two launches.  reduced=True: the gradient
        exchange kernel (distributed.reduce_grads) has already left the summed gradient in `self.reduced` together
        with its norms / step counts and zeroed `self.grad`: only the Adam launch remains.
        (A one-launch variant with a grid barrier between the norm and the update was measured at 9.3 us against 7.5 us
        for these two launches on the PPO agent's 141 k parameters, and dropped.)"""
        mask = self.all_mask if active_mask is None else int(active_mask)
        src = self.grad
        if reduced:
            src, zero_grad = self.reduced, False
        else:
            ops.grad_sumsq(self.grad, self._seg_c, self.nseg, mask, self.sumsq3, self.step_counts, self.betas,
                           self._scratch, self._ticket)
        ops.adam_step(self.data, src, self.exp_avg, self.exp_avg_sq, self._seg_c, self.nseg, mask, self.sumsq3, self.lr,
                      self._max_norm_c, self._eps_c, self.betas, grad_scale, zero_grad, self.hi, self.lo)

    def grad_norms(self):
        """Pre-clip total norm per segment of the last step (what clip_grad_norm_ returns)."""
        return torch.sqrt(self.sumsq3[:self.nseg])
