"""TRPO on the device (API of /root/reference/torchrl/algo/on_policy/trpo.py:13-282).

One natural-gradient policy step per epoch on the WHOLE rollout (trpo.py:153-230, 263-272), then `v_opt_times`
sweeps of value-function minibatches (trpo.py:232-261, 274-279) through the A2C minibatch loop with only the value
segment of the fused optimizer stepping.

How the policy step maps onto this library:
  * surrogate gradient: at ratio = 1 the gradient of -mean(ratio * adv) - c_ent * mean(ent) is the policy gradient,
    i.e. the actor loss kernel in policy-gradient mode + one backward through the fused MLP layers into the flat
    gradient buffer (the flat layout replaces parameters_to_vector);
  * Fisher-vector products WITHOUT double backward: for a Gaussian policy the Hessian of KL(pi_theta || pi_theta0) at
    theta0 is J^T D J with J = d(mean, std)/d theta and D = diag(1/std^2, 2/std^2) (what trpo.py:64-84 obtains by
    differentiating the KL twice).  J v is a tangent forward pass through the MLP on activations cached once per
    epoch (two GEMMs per layer); J^T u is an ordinary backward pass (retained graph) through the fused layers.  One
    product = 1 tangent forward + 1 backward instead of a double backward through autograd graphs the custom layers
    do not provide;
  * conjugate gradient with fp64 dot products like trpo.py:88-111, entirely on the device (the early exit on
    rdotr < residual_tol becomes a mask: no host sync per iteration);
  * line search (trpo.py:131-151): candidate parameters are written into the flat buffer and scored with the
    log-prob kernel; one host comparison per backtrack (the control flow IS the algorithm).
Reference quirk kept (SURVEY.md appendix A style): with a vec env the reference feeds (T, N, .) tensors, so
`torch.sum(kl, 1)` in mean_kl_divergence sums over the ENV axis and the mean runs over (T, act_dim): its KL -- and
therefore its Fisher matrix -- is N / act_dim times the per-sample KL.  `reference_quirks=True` (default) reproduces
that scaling for rollouts with N > 1 so that step sizes match the reference; False uses the per-sample KL.
"""
import numpy as np
import torch

from ... import ops
from ...networks import fused
from .. import utils as atu
from .a2c import A2C


class TRPO(A2C):
    def __init__(self, max_kl, cg_damping, v_opt_times, cg_iters, residual_tol, reference_quirks=True, **kwargs):
        super().__init__(**kwargs)
        self.max_kl, self.cg_damping, self.cg_iters = max_kl, cg_damping, cg_iters
        self.residual_tol, self.v_opt_times = residual_tol, v_opt_times
        self.vf_sample_key = ["obs", "estimate_returns"]
        self.reference_quirks = bool(reference_quirks)
        if not hasattr(self.pf, "logstd"):
            raise NotImplementedError("TRPO here needs a Gaussian policy with a free log-std vector "
                                      "(GuassianContPolicyBasicBias, what examples/trpo_continuous_vec.py builds)")

    # ------------------------------------------------------------------ value-function sweeps (A2C loop, vf only)
    def _passes(self):
        return self.v_opt_times

    def _gather_keys(self):
        return ["obs", "estimate_returns"]

    def _step_mask(self):
        return 0b10

    def _critic_step(self, batch, info):
        v = self.vf(batch["obs"])
        g_v, _ = ops.ppo_critic_loss(v.reshape(-1), batch["estimate_returns"].reshape(-1), None, False, 0.0,
                                     self._mb_state["scratch"], info=info[16:17])
        torch.autograd.backward([v], [0.5 * g_v.reshape(v.shape)])       # 0.5 * mean((V - R)^2), trpo.py:244

    def _actor_step(self, batch, info):
        pass

    def _epoch_adv_stats(self):
        pass                                                             # the value sweeps use no advantages

    def _decode_info(self, row, norms, gs):
        return {'Training/vf_loss': 0.5 * float(row[16]), 'grad_norm/vf': float(norms[1])}

    # ------------------------------------------------------------------ policy step
    def _layers(self):
        """Linear layers of the policy's mean network in forward order + the hidden activation code."""
        pairs = self.pf.base._pairs
        assert pairs is not None and len(self.pf.append_fcs) == 1, "TRPO needs an MLPBase trunk + one linear head"
        kinds = {type(a) for _, a in pairs}
        assert len(kinds) == 1 and next(iter(kinds)) in fused.ACT_CODES, "one activation type (Tanh / ReLU)"
        return [fc for fc, _ in pairs] + [self.pf.append_fcs[0]], fused.ACT_CODES[next(iter(kinds))]

    def _forward_cache(self, obs):
        """Activations of every hidden layer (no grad): what the tangent forward pass needs."""
        ys, x = [], obs
        with torch.no_grad():
            for fc, act in self.pf.base._pairs:
                x = self.pf.base._pair(x, fc, act)
                ys.append(x)
        return ys

    def _view(self, vec, p):
        """The slice of a flat pf-segment vector that corresponds to parameter `p`."""
        i = next(k for k, q in enumerate(self.opt.params) if q is p)
        o = self.opt.offsets[i] - self.opt.seg_begin[0]
        return vec[o:o + p.numel()].view(p.shape)

    def _tangent_forward(self, obs, ys, v):
        """J v: directional derivative of (mean, std) along the parameter direction v (flat, pf-segment layout)."""
        fcs, code = self._layers()
        x, t = obs, None
        for li, fc in enumerate(fcs):
            dW, db = self._view(v, fc.weight), self._view(v, fc.bias)
            tz = x @ dW.t() + db
            if t is not None:
                tz = tz + t @ fc.weight.t()
            if li < len(fcs) - 1:
                y = ys[li]
                t = tz * (1.0 - y * y) if code == 1 else tz * (y > 0).to(tz.dtype)
                x = y
            else:
                t = tz
        ls = self.pf.logstd
        inside = ((ls > -20.0) & (ls < 2.0)).to(ls.dtype)                # derivative of the clamp
        dstd = torch.exp(torch.clamp(ls, -20.0, 2.0)) * inside * self._view(v, ls)
        return t, dstd

    def _fvp(self, v, obs, ys, mean, std_vec, kl_scale):
        """(H_KL + damping I) v with H_KL = J^T D J (see module docstring); v and the result in pf-segment layout."""
        with torch.no_grad():
            dmean, dstd = self._tangent_forward(obs, ys, v)
            B = mean.shape[0]
            u_mean = (dmean / (std_vec * std_vec)) * (kl_scale / B)
            u_std = (2.0 * dstd / (std_vec * std_vec)) * kl_scale
        seg = self.opt.grad[self.opt.seg_begin[0]:self.opt.seg_begin[1]]
        seg.zero_()
        std_param = torch.exp(torch.clamp(self.pf.logstd, -20.0, 2.0))
        torch.autograd.backward([mean, std_param], [u_mean, u_std], retain_graph=True)
        out = seg.clone() + self.cg_damping * v
        seg.zero_()
        return out

    def _log_probs(self, obs, acts, out=None):
        with torch.no_grad():
            mean, log_std = self._policy_outputs(self.pf, obs)
            return ops.gaussian_log_prob(mean, log_std, acts, self.tanh_action, out=out)

    @fused.presplit_scope
    def update(self, batch):
        """The natural-gradient policy step on an explicit whole batch (trpo.py:153-230): obs (..., o), acts (..., a),
        advs (..., 1) as arrays or device tensors.  Returns the reference's info dict."""
        self.training_update_num += 1
        obs_in = batch['obs']
        lead = tuple(obs_in.shape[:-1])
        env_axis = lead[1] if len(lead) >= 2 else 1
        obs, acts, advs = self._minibatch(batch, ('obs', 'acts', 'advs'))
        obs = obs.reshape(-1, obs.shape[-1])
        B = obs.shape[0]
        acts = acts.reshape(B, -1)
        advs = advs.reshape(-1)
        a = acts.shape[1]
        kl_scale = float(env_axis) / a if (self.reference_quirks and len(lead) >= 2) else 1.0
        info32 = torch.zeros(32, dtype=torch.float32, device=self.device)
        st = ops.vec_stats(advs, out=info32[20:24])
        advn = ((advs - st[0]) / (st[1] + 1e-4)).contiguous()                       # trpo.py:171 (1e-4, not 1e-5)
        # trpo.py:177-180: ratio = p / (p.detach() + 1e-8) with p = exp(log_prob): its value AND its gradient carry
        # the factor w = p / (p + 1e-8) (1 for any action the policy could have taken, 0 for log-probs below ~ -18)
        logp_old = self._log_probs(obs, acts)
        p_old = torch.exp(logp_old)
        advw = (advn * (p_old / (p_old + 1e-8))).contiguous()
        seg0 = slice(self.opt.seg_begin[0], self.opt.seg_begin[1])
        # ---- surrogate gradient (ratio = 1): policy-gradient mode of the actor kernel + one backward --------------
        self.opt.grad[seg0].zero_()
        scratch = ops.LossScratch(B, a, self.device)
        mean, log_std = self._policy_outputs(self.pf, obs)
        g_mean, g_ls, _ = ops.ppo_actor_loss(mean, log_std, acts, None, advw, None, 0.0, self.entropy_coeff,
                                             self.tanh_action, scratch, info=info32[0:16])
        torch.autograd.backward([mean, log_std], [g_mean, g_ls], retain_graph=True)
        g = self.opt.grad[seg0].clone()
        self.opt.grad[seg0].zero_()
        ops.vec_stats(logp_old, out=info32[24:28])
        ent_mean = info32[11:12].clone()
        surrogate = -(advw.mean()) - self.entropy_coeff * ent_mean
        if bool((g != 0).any()):
            ys = self._forward_cache(obs)
            std_vec = torch.exp(torch.clamp(self.pf.logstd.detach(), -20.0, 2.0))
            fvp = lambda v: self._fvp(v, obs, ys, mean, std_vec, kl_scale)
            step_dir = self._conjugate_gradient(fvp, -g)
            shs = 0.5 * torch.dot(step_dir, fvp(step_dir))
            lm = torch.sqrt(shs / self.max_kl)
            fullstep = step_dir / lm
            gdotstepdir = -torch.dot(g, step_dir)
            theta0 = self.opt.data[seg0].clone()
            theta = self._linesearch(theta0, fullstep, gdotstepdir / lm, obs, acts, advn, logp_old)
            if bool(torch.isnan(theta).any()):
                self.opt.data[seg0].copy_(theta0)                                 # "NaN detected. Skipping update..."
            else:
                self.opt.data[seg0].copy_(theta)
            self.opt.refresh_split()
        del mean, log_std
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

    def _surrogate_at(self, theta, obs, acts, advn, logp_old):
        seg0 = slice(self.opt.seg_begin[0], self.opt.seg_begin[1])
        self.opt.data[seg0].copy_(theta)
        self.opt.refresh_split()
        logp = self._log_probs(obs, acts)
        return -torch.mean(torch.exp(logp - logp_old) * advn)

    def _linesearch(self, x, fullstep, expected_improve_rate, obs, acts, advn, logp_old):
        """trpo.py:131-151: backtracking on the surrogate; returns the accepted parameter vector (or x)."""
        fval = self._surrogate_at(x, obs, acts, advn, logp_old)
        for stepfrac in .5 ** np.arange(10):
            stepfrac = float(stepfrac)
            xnew = x + stepfrac * fullstep
            newfval = self._surrogate_at(xnew, obs, acts, advn, logp_old)
            actual_improve = fval - newfval
            ratio = actual_improve / (expected_improve_rate * stepfrac)
            if bool((ratio > 0.1) & (actual_improve > 0)):
                return xnew
        return x

    def update_vf(self, batch):
        """One eager value-function minibatch (trpo.py:232-261)."""
        self.training_update_num += 1
        obs, rets = self._minibatch(batch, ('obs', 'estimate_returns'))
        B = obs.shape[0]
        scratch = ops.LossScratch(B, 1, self.device)
        info32 = torch.zeros(32, dtype=torch.float32, device=self.device)
        with fused.presplit():
            v = self.vf(obs)
            g_v, _ = ops.ppo_critic_loss(v.reshape(-1), rets.reshape(-1), None, False, 0.0, scratch, info=info32[16:17])
            torch.autograd.backward([v], [0.5 * g_v.reshape(v.shape)])
            scale = self._optimizer_step(0b10)
        return {'Training/vf_loss': 0.5 * float(info32[16].item()),
                'grad_norm/vf': float(self.opt.grad_norms()[1].item()) * scale}

    def update_per_epoch(self, flush_infos=True):
        """trpo.py:263-279: returns, LR decay, one whole-rollout policy step, v_opt_times value sweeps."""
        self.process_epoch_samples()
        atu.update_linear_schedule(self.pf_optimizer, self.current_epoch, self.num_epochs, self.plr)
        atu.update_linear_schedule(self.vf_optimizer, self.current_epoch, self.num_epochs, self.vlr)
        rb = self.replay_buffer
        info = self.update({"obs": rb._obs, "acts": rb._acts, "advs": rb._advs})
        self._last_policy_info = info
        if self.logger is not None:
            self.logger.add_update_info(info)
        with fused.presplit():
            self._minibatch_epoch(flush_infos)                   # the value sweeps
