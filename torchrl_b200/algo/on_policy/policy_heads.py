"""What the on-policy algorithms (A2C, PPO, V-MPO, TRPO, REINFORCE) need to know about the policy's action distribution,
in one place: how the minibatch step computes the actor loss and its gradient, the old log-probs, TRPO's surrogate
gradient, KL weighting and line-search score, and which distribution-specific scalars are logged.
`policy_head(pf)` picks the helper once, at construction.

  GaussianHead     -- the (tanh-)Gaussian policies of policies/continuous_policy.py (csrc/ppo_loss.cu);
  CategoricalHead  -- CategoricalDisPolicy over logits (csrc/categorical.cu).
"""
import numpy as np
import torch

from ... import ops
from ...networks import fused
from ..utils import four_stats


def gaussian_outputs(pf, obs):
    """(mean, std, log_std) of a Gaussian policy, mean and log_std made contiguous for the kernels."""
    mean, std, log_std = pf(obs)
    mean = mean if mean.is_contiguous() else mean.contiguous()
    log_std = log_std if log_std.is_contiguous() else log_std.contiguous()
    return mean, std, log_std


class GaussianHead:
    # keys the reference's PPO.update_actor logs besides the clipped-surrogate statistics (ppo.py:81-84)
    ppo_extra_keys = ['log_std/mean', 'log_std/std', 'log_std/max', 'log_std/min']

    def __init__(self, pf):
        self.tanh_action = bool(getattr(pf, "tanh_action", False))
        self.shared_logstd = hasattr(pf, "logstd")

    def fused_ok(self, pf):
        """The fused minibatch loop needs a shared log-std PARAMETER (GuassianContPolicyBasicBias)."""
        return hasattr(pf, "logstd")

    def loss_scratch(self, B, a, device):
        return ops.LossScratch(B, a, device)

    def actor(self, pf, obs, acts, old_logp, advs, adv_table, stats_pos, clip, ent_coef, scratch, info, logp_out=None):
        """The actor loss kernel, then autograd through the policy.  With a shared log-std parameter the kernel takes
        the mean and the raw parameter, applies the policy's clamp itself and writes the parameter's gradient straight
        into its slice of the flat gradient buffer (this removes the clamp / exp / clamp-backward / accumulate launches
        on six-element tensors from every minibatch); otherwise autograd runs through the (mean, log_std) of the
        policy's forward.  Returns the std that `std_row` logs: None with a shared log-std parameter."""
        from ...policies.continuous_policy import LOG_SIG_MIN, LOG_SIG_MAX
        if self.shared_logstd:
            mean = pf.mean_net(obs)
            if not mean.is_contiguous():
                mean = mean.contiguous()
            ls, g_ls, ls_clamp, std = pf.logstd.detach(), pf.logstd.grad, (LOG_SIG_MIN, LOG_SIG_MAX), None
        else:
            mean, std, ls = gaussian_outputs(pf, obs)
            if ls.dim() > 1 and ls.shape != mean.shape:
                ls = ls.expand_as(mean).contiguous()
            g_ls, ls_clamp, std = None, None, std.detach().expand_as(mean)
        g_mean, g_ls, _ = ops.ppo_actor_loss(mean, ls, acts.reshape(mean.shape[0], -1), old_logp, advs, adv_table, clip,
                                             ent_coef, self.tanh_action, scratch, g_log_std=g_ls, info=info[0:16],
                                             logp_out=logp_out, stats_pos=stats_pos, ls_clamp=ls_clamp)
        with fused.backward_fork():
            if self.shared_logstd:
                torch.autograd.backward([mean], [g_mean])
            else:
                torch.autograd.backward([mean, ls], [g_mean, g_ls])
        return std

    def std_row(self, pf, std, info):
        """What A2C's std/* (a2c.py:90-94) are derived from at decode: the clamped shared log-std, or the four
        statistics of the autograd route's std."""
        if std is not None:
            ops.vec_stats(std.contiguous().reshape(-1), out=info[28:32])
            return
        from ...policies.continuous_policy import LOG_SIG_MIN, LOG_SIG_MAX
        n = pf.logstd.numel()
        torch.clamp(pf.logstd.detach(), LOG_SIG_MIN, LOG_SIG_MAX, out=info[28:28 + n])

    def a2c_std_info(self, row, B, a):
        if not self.shared_logstd:
            return four_stats('std', row[28:32])
        ls = row[28:28 + a].astype(np.float64)
        sd = np.exp(ls)
        m = sd.mean()
        var = B * ((sd - m) ** 2).sum() / (B * a - 1.0)              # torch.std() of the (B, a) expanded tensor
        return {'std/mean': float(m), 'std/std': float(np.sqrt(var)), 'std/max': float(sd.max()),
                'std/min': float(sd.min())}

    def old_log_prob(self, pf, obs, acts, out):
        mean, _, ls = gaussian_outputs(pf, obs)
        return ops.gaussian_log_prob(mean, ls, acts.reshape(mean.shape[0], -1), self.tanh_action, out=out)

    # ---- TRPO (trpo.py:29-230)
    trpo_unsupported = ("TRPO supports a Gaussian policy with a free log-std vector (GuassianContPolicyBasicBias) or a "
                        "CategoricalDisPolicy, over MLPBase or CNNBase with Tanh or ReLU activations and no LayerNorm")

    def trpo_ok(self, pf):
        return hasattr(pf, "logstd")

    def trpo_forward(self, pf, obs):
        """The outputs whose graph the policy step keeps: (mean, log_std)."""
        mean, _, ls = gaussian_outputs(pf, obs)
        return mean, ls

    def trpo_log_prob(self, pf, obs, acts):
        with torch.no_grad():
            return self.old_log_prob(pf, obs, acts, None)

    def trpo_actor(self, outs, acts, advw, ent_coef, info):
        """The surrogate's gradient at ratio = 1: policy-gradient mode of the actor kernel on advn * w, then one
        backward (graph kept for the Fisher-vector products)."""
        mean, ls = outs
        B = mean.shape[0]
        scratch = ops.LossScratch(B, mean.shape[1], mean.device)
        g_mean, g_ls, _ = ops.ppo_actor_loss(mean, ls, acts.reshape(B, -1), None, advw, None, 0.0, ent_coef,
                                             self.tanh_action, scratch, info=info)
        torch.autograd.backward([mean, ls], [g_mean, g_ls], retain_graph=True)

    def trpo_fisher_backward(self, pf, outs, dmean, v_of, kl_scale):
        """Back-propagates D J v with D = diag(1/std^2, 2/std^2), the Hessian of the Gaussian KL wrt (mean, std)."""
        from ...policies.continuous_policy import LOG_SIG_MIN, LOG_SIG_MAX
        mean = outs[0]
        ls = pf.logstd
        with torch.no_grad():
            std_vec = torch.exp(torch.clamp(ls, LOG_SIG_MIN, LOG_SIG_MAX))
            inside = ((ls > LOG_SIG_MIN) & (ls < LOG_SIG_MAX)).to(ls.dtype)         # derivative of the clamp
            dstd = std_vec * inside * v_of(ls)
            u_mean = (dmean / (std_vec * std_vec)) * (kl_scale / mean.shape[0])
            u_std = (2.0 * dstd / (std_vec * std_vec)) * kl_scale
        std_param = torch.exp(torch.clamp(ls, LOG_SIG_MIN, LOG_SIG_MAX))
        torch.autograd.backward([mean, std_param], [u_mean, u_std], retain_graph=True)

    def trpo_scratch(self, B, device):
        return None

    def trpo_score(self, pf, obs, acts, logp_old, advn, scratch):
        """The line search's surrogate -mean(exp(logp - logp_old) * advn) (trpo.py:113-129), a device scalar."""
        logp = self.trpo_log_prob(pf, obs, acts)
        return -torch.mean(torch.exp(logp - logp_old) * advn)


class CategoricalHead:
    # the reference's PPO.update_actor reads out['log_std'] (ppo.py:52), which CategoricalDisPolicy.update does not
    # return: its discrete PPO raises KeyError.  Here PPO runs and the four log_std/* keys are simply not logged.
    ppo_extra_keys = []

    def __init__(self, pf):
        pass

    def fused_ok(self, pf):
        return True

    def loss_scratch(self, B, a, device):
        return ops.LossScratch(B, 1, device, categorical=True)

    @staticmethod
    def _logits(pf, obs):
        z = pf.logits(obs)
        return z if z.is_contiguous() else z.contiguous()

    def actor(self, pf, obs, acts, old_logp, advs, adv_table, stats_pos, clip, ent_coef, scratch, info, logp_out=None):
        logits = self._logits(pf, obs)
        g, _ = ops.ppo_categorical_actor_loss(logits, acts.reshape(-1), old_logp, advs, adv_table, clip, ent_coef,
                                              scratch, info=info[0:16], logp_out=logp_out, stats_pos=stats_pos)
        with fused.backward_fork():
            torch.autograd.backward([logits], [g])

    def std_row(self, pf, std, info):
        pass

    def a2c_std_info(self, row, B, a):
        return {}                                           # a2c.py:90-94 logs std/* only `if 'std' in out`

    def old_log_prob(self, pf, obs, acts, out):
        return ops.categorical_log_prob(self._logits(pf, obs), acts.reshape(-1).contiguous(), out=out)

    # ---- V-MPO (v_mpo.py:57-133)
    def vmpo_scratch(self, B, device):
        return ops.VMPOScratch(B - B // 2, device)

    def vmpo_actor(self, pf, target_pf, obs, acts, advs, adv_stats, stats_pos, dual, eta_eps, alpha_eps, per_row_kl,
                   scratch, info):
        """The actor step on the k selected rows: both policies' logits on those rows only, one loss kernel that writes
        dL/d[eta, alpha] straight into the duals' slice of the flat gradient, autograd through the policy's logits."""
        logits = self._logits(pf, obs)
        with torch.no_grad():
            tlogits = self._logits(target_pf, obs)
        g = ops.vmpo_categorical_loss(logits, tlogits, acts.reshape(-1), advs.reshape(-1), adv_stats, dual.detach(),
                                      eta_eps, alpha_eps, per_row_kl, scratch, dual.grad, info, stats_pos=stats_pos)
        with fused.backward_fork():
            torch.autograd.backward([logits], [g])

    # ---- TRPO (trpo.py:29-230 with the KL over probs, trpo.py:53-61)
    trpo_unsupported = GaussianHead.trpo_unsupported

    def trpo_ok(self, pf):
        return True

    def trpo_forward(self, pf, obs):
        return (self._logits(pf, obs),)

    def trpo_log_prob(self, pf, obs, acts):
        with torch.no_grad():
            return self.old_log_prob(pf, obs, acts, None)

    def trpo_actor(self, outs, acts, advw, ent_coef, info):
        logits, = outs
        B = logits.shape[0]
        scratch = ops.LossScratch(B, 1, logits.device, categorical=True)
        g, _ = ops.ppo_categorical_actor_loss(logits, acts.reshape(-1).contiguous(), None, advw, None, 0.0, ent_coef,
                                              scratch, info=info)
        torch.autograd.backward([logits], [g], retain_graph=True)

    def trpo_fisher_backward(self, pf, outs, dlogits, v_of, kl_scale):
        """Back-propagates (diag p - p p^T) J v / B * kl_scale, the Hessian of the mean categorical KL wrt the
        logits applied to the logits' tangent: one trl_categorical_fisher_vp launch, then autograd."""
        logits, = outs
        g = ops.categorical_fisher_vp(logits.detach(), dlogits, kl_scale / logits.shape[0])
        torch.autograd.backward([logits], [g], retain_graph=True)

    def trpo_scratch(self, B, device):
        return ops.SurrogateScratch(B, device)

    def trpo_score(self, pf, obs, acts, logp_old, advn, scratch):
        with torch.no_grad():
            return ops.categorical_surrogate(self._logits(pf, obs), acts.reshape(-1).contiguous(), logp_old, advn,
                                             scratch)[0]


def policy_head(pf):
    from ...policies.discrete_policies import CategoricalDisPolicy
    return CategoricalHead(pf) if isinstance(pf, CategoricalDisPolicy) else GaussianHead(pf)
