"""TRPO on the device (API of /root/reference/torchrl/algo/on_policy/trpo.py:13-282).

One natural-gradient policy step per epoch on the WHOLE rollout (trpo.py:153-230, 263-272), then `v_opt_times`
sweeps of value-function minibatches (trpo.py:232-261, 274-279) through the A2C minibatch loop with only the value
segment of the fused optimizer stepping.

How the policy step maps onto this library:
  * surrogate gradient: at ratio = 1 the gradient of -mean(ratio * adv) - c_ent * mean(ent) is the policy gradient,
    i.e. the actor loss kernel in policy-gradient mode + one backward through the fused MLP layers into the flat
    gradient buffer (the flat layout replaces parameters_to_vector);
  * Fisher-vector products WITHOUT double backward: the Hessian of KL(pi_theta || pi_theta0) at theta0 is J^T D J
    with J the Jacobian of the policy's outputs (what trpo.py:64-84 obtains by differentiating the KL twice).  For a
    Gaussian policy the outputs are (mean, std) and D = diag(1/std^2, 2/std^2); for a categorical one they are the
    logits and D = diag(p) - p p^T (trl_categorical_fisher_vp, DESIGN §6 deviation 20).  J v is a tangent forward
    pass through the net (`layer_plan`: Linear or Conv2d layers of the trunk, then append_fcs) on activations cached
    once per policy step: per layer x dW^T + t W^T (cuBLAS) or conv(x, dW) + conv(t, W) (cuDNN), then the bias and
    activation-derivative step in one launch (trl_tangent_bias_act).  J^T u is an ordinary backward pass (retained
    graph).  One product = 1 tangent forward + 1 backward instead of a double backward through autograd graphs the
    custom layers do not provide;
  * conjugate gradient with fp64 dot products like trpo.py:88-111, entirely on the device (the early exit on
    rdotr < residual_tol becomes a mask: no host sync per iteration);
  * line search (trpo.py:131-151): candidate parameters are written into the flat buffer and scored (categorical:
    one trl_categorical_surrogate launch after the forward); one host comparison per backtrack (the control flow IS
    the algorithm).
The distribution-specific pieces (surrogate gradient, KL weighting of J v, log-probs, score) live on the policy heads
(policy_heads.py); this class does not branch on the policy type.  On the pixel path the whole rollout's uint8 frames
are scaled once per policy step (OnRLAlgo._prep_obs).
Reference quirk kept (SURVEY.md appendix A style): with a vec env the reference feeds (T, N, .) tensors, so
`torch.sum(kl, 1)` in mean_kl_divergence sums over the ENV axis and the mean runs over (T, act_dim) -- (T, A) for the
categorical KL over probs: its KL -- and therefore its Fisher matrix -- is N / act_dim (N / A) times the per-sample
KL.  `reference_quirks=True` (default) reproduces that scaling for (T, N) batches so that step sizes match the
reference; False uses the per-sample KL.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...networks import fused
from ...networks.base import CNNBase, MLPBase
from .. import utils as atu
from .a2c import A2C

_LAYERS = (nn.Linear, nn.Conv2d)


def layer_plan(net):
    """[(Linear | Conv2d, activation module or None)] of a networks.Net in forward order: the trunk's layers
    (MLPBase.fcs or CNNBase.convs), then append_fcs.  None if the net holds anything else (a LayerNorm, an
    activation other than Tanh / ReLU, a layer without bias)."""
    if getattr(net, "add_ln", False) or not isinstance(getattr(net, "base", None), (MLPBase, CNNBase)):
        return None
    mods = list(net.base.convs if isinstance(net.base, CNNBase) else net.base.fcs) + list(net.append_fcs)
    plan, i = [], 0
    while i < len(mods):
        layer = mods[i]
        if not isinstance(layer, _LAYERS) or layer.bias is None:
            return None
        act = mods[i + 1] if i + 1 < len(mods) and not isinstance(mods[i + 1], _LAYERS) else None
        if act is not None and type(act) not in fused.ACT_CODES:
            return None
        plan.append((layer, act))
        i += 1 if act is None else 2
    return plan if plan and plan[-1][1] is None else None


class TRPO(A2C):
    def __init__(self, max_kl, cg_damping, v_opt_times, cg_iters, residual_tol, reference_quirks=True, **kwargs):
        super().__init__(**kwargs)
        self.max_kl, self.cg_damping, self.cg_iters = max_kl, cg_damping, cg_iters
        self.residual_tol, self.v_opt_times = residual_tol, v_opt_times
        self.vf_sample_key = ["obs", "estimate_returns"]
        self.reference_quirks = bool(reference_quirks)
        self._plan = layer_plan(self.pf)
        if self._plan is None or not self._head.trpo_ok(self.pf):
            raise NotImplementedError(self._head.trpo_unsupported)
        self._obs_dims = 3 if isinstance(self.pf.base, CNNBase) else 1

    # ------------------------------------------------------------------ value-function sweeps (A2C loop, vf only)
    def _passes(self):
        return self.v_opt_times

    def _gather_keys(self):
        return ["obs", "estimate_returns"]

    def _step_mask(self):
        return 0b10

    def _critic_step(self, batch, st, info):
        v = self.vf(batch["obs"])
        g_v, _ = ops.ppo_critic_loss(v.reshape(-1), batch["estimate_returns"].reshape(-1), None, False, 0.0,
                                     st["scratch"], info=info[16:17])
        torch.autograd.backward([v], [0.5 * g_v.reshape(v.shape)])       # 0.5 * mean((V - R)^2), trpo.py:244

    def _actor_step(self, batch, st, info):
        pass

    def _epoch_adv_stats(self):
        pass                                                             # the value sweeps use no advantages

    def _prepare_batch(self, batch, st):
        pass

    def _decode_info(self, row, norms, st):
        return {'Training/vf_loss': 0.5 * float(row[16]), 'grad_norm/vf': float(norms[1])}

    # ------------------------------------------------------------------ policy step
    def _forward_cache(self, obs):
        """The output of every layer with an activation (no grad): what the tangent forward pass needs."""
        ys, x = [], obs
        with torch.no_grad():
            for layer, act in self._plan[:-1]:
                if isinstance(layer, nn.Linear):
                    x = MLPBase._pair(x.reshape(x.shape[0], -1), layer, act)
                else:
                    x = act(layer(x))
                ys.append(x)
        return ys

    def _view(self, vec, p):
        """The slice of a flat pf-segment vector that corresponds to parameter `p`."""
        i = next(k for k, q in enumerate(self.opt.params) if q is p)
        o = self.opt.offsets[i] - self.opt.seg_begin[0]
        return vec[o:o + p.numel()].view(p.shape)

    def _tangent_forward(self, obs, ys, v):
        """J v: directional derivative of the net's output along the parameter direction v (flat, pf-segment
        layout).  Per layer x dW^T + t W^T (conv(x, dW) + conv(t, W)), then (t + db) * act'(y) in one launch."""
        x, t = obs, None
        for li, (layer, act) in enumerate(self._plan):
            W, dW, db = layer.weight, self._view(v, layer.weight), self._view(v, layer.bias)
            if isinstance(layer, nn.Conv2d):
                conv = lambda inp, w: F.conv2d(inp, w, None, layer.stride, layer.padding, layer.dilation,  # noqa: E731
                                               layer.groups)
                tz = conv(x, dW)
                if t is not None:
                    tz.add_(conv(t, W))
            else:
                x = x.reshape(x.shape[0], -1)
                tz = torch.mm(x, dW.t())
                if t is not None:
                    tz.addmm_(t.reshape(t.shape[0], -1), W.t())
            y = ys[li] if act is not None else None
            t = ops.tangent_bias_act(tz, db, y, fused.ACT_CODES[type(act)] if act is not None else 0)
            x = y
        return t

    def _fvp(self, v, obs, ys, outs, kl_scale):
        """(H_KL + damping I) v with H_KL = J^T D J (see module docstring); v and the result in pf-segment layout."""
        with torch.no_grad():
            dout = self._tangent_forward(obs, ys, v)
        seg = self.opt.grad[self.opt.seg_begin[0]:self.opt.seg_begin[1]]
        seg.zero_()
        self._head.trpo_fisher_backward(self.pf, outs, dout, lambda p: self._view(v, p), kl_scale)
        out = seg.clone() + self.cg_damping * v
        seg.zero_()
        return out

    def _kl_scale(self, env_axis):
        """N / act_dim (N / A) for a (T, N) batch under reference_quirks, else 1 (module docstring)."""
        if not self.reference_quirks or env_axis is None:
            return 1.0
        return float(env_axis) / self._plan[-1][0].out_features

    def _policy_batch(self, batch):
        """(obs (B, ...), acts, advs (B,), env-axis size or None) of an explicit whole batch: flat (B, .) or the
        (T, N, .) whole-rollout layout; uint8 frames are scaled once (OnRLAlgo._prep_obs), not merely cast."""
        b = self._device_batch(batch, ('obs', 'acts', 'advs'))
        obs, acts, advs = b['obs'], b['acts'], b['advs']
        lead = tuple(obs.shape[:obs.dim() - self._obs_dims])
        obs = obs.reshape((-1,) + tuple(obs.shape[len(lead):]))
        return obs, acts.reshape(obs.shape[0], -1), advs.reshape(-1), (lead[1] if len(lead) >= 2 else None)

    @fused.presplit_scope
    def fisher_vector_product(self, batch, v):
        """(H_KL + cg_damping I) v on an explicit whole batch at the current policy (trpo.py:65-86, the reference's
        hessian_vector_product); v and the result are flat vectors in the order of pf.parameters()
        (parameters_to_vector), not the padded layout of the flat buffer."""
        obs, acts, advs, env_axis = self._policy_batch(batch)
        outs = self._head.trpo_forward(self.pf, obs)
        params = list(self.pf.parameters())
        seg = torch.zeros(self.opt.seg_begin[1] - self.opt.seg_begin[0], dtype=torch.float32, device=self.device)
        o = 0
        for p in params:
            self._view(seg, p).copy_(v[o:o + p.numel()].view(p.shape))
            o += p.numel()
        out = self._fvp(seg, obs, self._forward_cache(obs), outs, self._kl_scale(env_axis))
        return torch.cat([self._view(out, p).reshape(-1) for p in params])

    @fused.presplit_scope
    def update(self, batch):
        """The natural-gradient policy step on an explicit whole batch (trpo.py:153-230): obs (..., obs shape),
        acts (..., a) -- action indices for a categorical policy --, advs (..., 1) as arrays or device tensors.
        Returns the reference's info dict."""
        self.training_update_num += 1
        obs, acts, advs, env_axis = self._policy_batch(batch)
        B = obs.shape[0]
        kl_scale = self._kl_scale(env_axis)
        info32 = torch.zeros(32, dtype=torch.float32, device=self.device)
        st = ops.vec_stats(advs, out=info32[20:24])
        advn = ((advs - st[0]) / (st[1] + 1e-4)).contiguous()                       # trpo.py:171 (1e-4, not 1e-5)
        # trpo.py:177-180: ratio = p / (p.detach() + 1e-8) with p = exp(log_prob): its value AND its gradient carry
        # the factor w = p / (p + 1e-8) (1 for any action the policy could have taken, 0 for log-probs below ~ -18)
        logp_old = self._head.trpo_log_prob(self.pf, obs, acts)
        p_old = torch.exp(logp_old)
        advw = (advn * (p_old / (p_old + 1e-8))).contiguous()
        seg0 = slice(self.opt.seg_begin[0], self.opt.seg_begin[1])
        # ---- surrogate gradient (ratio = 1): policy-gradient mode of the actor kernel + one backward --------------
        self.opt.grad[seg0].zero_()
        outs = self._head.trpo_forward(self.pf, obs)
        self._head.trpo_actor(outs, acts, advw, self.entropy_coeff, info32[0:16])
        g = self.opt.grad[seg0].clone()
        self.opt.grad[seg0].zero_()
        ops.vec_stats(logp_old, out=info32[24:28])
        ent_mean = info32[11:12].clone()
        surrogate = -(advw.mean()) - self.entropy_coeff * ent_mean
        if bool((g != 0).any()):
            ys = self._forward_cache(obs)
            fvp = lambda v: self._fvp(v, obs, ys, outs, kl_scale)                  # noqa: E731
            step_dir = self._conjugate_gradient(fvp, -g)
            shs = 0.5 * torch.dot(step_dir, fvp(step_dir))
            lm = torch.sqrt(shs / self.max_kl)
            fullstep = step_dir / lm
            gdotstepdir = -torch.dot(g, step_dir)
            theta0 = self.opt.data[seg0].clone()
            del ys
            score = self._scorer(obs, acts, advn, logp_old)
            theta = self._linesearch(theta0, fullstep, gdotstepdir / lm, score)
            if bool(torch.isnan(theta).any()):
                self.opt.data[seg0].copy_(theta0)                                 # "NaN detected. Skipping update..."
            else:
                self.opt.data[seg0].copy_(theta)
            self.opt.refresh_split()
        del outs
        row = info32.cpu().numpy()
        info = atu.four_stats('advs', row[20:24])
        info['Training/policy_loss'] = float(surrogate.item())
        info.update(atu.four_stats('logprob', row[24:28]))
        return info

    def _conjugate_gradient(self, fvp, b):
        """trpo.py:88-111 with the early exit turned into a mask (once rdotr < residual_tol nothing changes)."""
        p, r = b.clone(), b.clone()
        x = torch.zeros_like(b)
        rdotr = torch.dot(r.double(), r.double())
        alive = torch.ones((), dtype=torch.float64, device=b.device)
        for _ in range(self.cg_iters):
            z = fvp(p)
            v = (rdotr / torch.dot(p.double(), z.double())) * alive
            x = x + v.float() * p
            r = r - v.float() * z
            newrdotr = torch.dot(r.double(), r.double())
            mu = newrdotr / rdotr
            p = torch.where(alive > 0, r + mu.float() * p, p)
            rdotr = torch.where(alive > 0, newrdotr, rdotr)
            alive = alive * (rdotr >= self.residual_tol).to(torch.float64)
        return x

    def _scorer(self, obs, acts, advn, logp_old):
        """theta -> the surrogate at theta (trpo.py:113-129), a device scalar: theta is written into the flat buffer
        and the policy head scores the candidate."""
        seg0 = slice(self.opt.seg_begin[0], self.opt.seg_begin[1])
        scratch = self._head.trpo_scratch(obs.shape[0], self.device)

        def score(theta):
            self.opt.data[seg0].copy_(theta)
            self.opt.refresh_split()
            return self._head.trpo_score(self.pf, obs, acts, logp_old, advn, scratch)
        return score

    def _linesearch(self, x, fullstep, expected_improve_rate, score):
        """trpo.py:131-151: backtracking on the surrogate; returns the accepted parameter vector (or x)."""
        fval = score(x)
        for stepfrac in .5 ** np.arange(10):
            stepfrac = float(stepfrac)
            xnew = x + stepfrac * fullstep
            newfval = score(xnew)
            actual_improve = fval - newfval
            ratio = actual_improve / (expected_improve_rate * stepfrac)
            if bool((ratio > 0.1) & (actual_improve > 0)):
                return xnew
        return x

    def update_vf(self, batch):
        """One value-function minibatch on an explicit batch (trpo.py:232-261): the value sweeps' step."""
        return A2C.update(self, batch)

    def update_per_epoch(self, flush_infos=True):
        """trpo.py:263-279: returns, LR decay, one whole-rollout policy step, v_opt_times value sweeps."""
        self.process_epoch_samples()
        atu.update_linear_schedule(self.pf_optimizer, self.current_epoch, self.num_epochs, self.plr)
        atu.update_linear_schedule(self.vf_optimizer, self.current_epoch, self.num_epochs, self.vlr)
        rb = self.replay_buffer
        info = self.update({"obs": rb._obs, "acts": rb._acts, "advs": rb._advs})     # uint8 frames scaled once
        self._last_policy_info = info
        if self.logger is not None:
            self.logger.add_update_info(info)
        with fused.presplit():
            self._minibatch_epoch(flush_infos)                   # the value sweeps
