"""Twin-Q SAC without a V network (API of /root/reference/torchrl/algo/off_policy/twin_sac_q.py:11-250).

Per update (one captured CUDA graph): row gather -> pf(obs) + sampling/log-prob kernel (autograd) ->
Q1,Q2(obs,a) -> temperature loss + its Adam step (1 launch) -> [no grad] pf(next_obs) sample,
target Q's, TD-target kernel -> twin MSE kernel -> Q1,Q2(obs, a~) -> policy-loss kernel -> two
autograd.backward calls seeded with the kernel gradients -> fused clip+Adam over pf|qf1|qf2 ->
Polyak over the flat target buffer -> log row.
The temperature, the sample and the policy's regularisers and statistics live in SoftActorCritic, which SAC and
TwinSAC (sac.py) share.
"""
import numpy as np
import torch
import torch.optim as optim

from ... import ops
from ...policies import distribution as D
from ..utils import four_stats
from .off_rl_algo import OffRLAlgo


class SoftActorCritic(OffRLAlgo):
    """What TwinSAC-Q and SAC / TwinSAC (sac.py) share: the temperature, the policy's sample, the std / mean
    regularisers and the policy statistics.  Info row slots: 0 Reward_Mean | 1 Alpha 2 Alpha_loss | 4.. critic losses |
    10..13 log_std stats | 14..17 mean stats | 18 std_reg 19 mean_reg | 20 policy_loss (kernel part), then the loss
    kernel's log_probs statistics at `_LOG_PROBS`."""
    _LOG_PROBS = None

    def __init__(self, pf, policy_std_reg_weight, policy_mean_reg_weight, reparameterization, automatic_entropy_tuning,
                 target_entropy, **kwargs):
        super().__init__(**kwargs)
        self.pf = pf
        self.automatic_entropy_tuning = automatic_entropy_tuning
        if self.automatic_entropy_tuning:
            self.target_entropy = target_entropy if target_entropy else \
                -float(np.prod(self.env.action_space.shape).item())
            self.log_alpha = torch.zeros(1, device=self.device)
            self._alpha_state = torch.zeros(3, device=self.device)     # exp_avg, exp_avg_sq, step
        self.policy_std_reg_weight = policy_std_reg_weight
        self.policy_mean_reg_weight = policy_mean_reg_weight
        self.reparameterization = bool(reparameterization)
        self.tanh_action = bool(getattr(pf, "tanh_action", True))

    def _sample(self, obs, want_grad):
        mean, std, log_std = self.pf(obs)
        mean_c = mean if mean.is_contiguous() else mean.contiguous()
        ls = log_std if log_std.dim() == 1 else (log_std if log_std.is_contiguous() else log_std.contiguous())
        eps = D.draw_reference_noise(tuple(mean_c.shape), mean_c.device) if D.get_noise_mode() == "reference_cpu" \
            else None
        rng = self.pf._rng_state(mean_c.device)
        if want_grad:
            action, logp, _ = D._SampleFn.apply(mean_c, ls, eps, self.tanh_action, True, rng)
        else:
            out = ops.tanh_gaussian_sample(mean_c, ls, eps=eps, tanh_action=self.tanh_action, want_log_prob=True,
                                           rng=rng)
            action, logp = out["action"], out["log_prob"]
        if eps is None:
            ops.counter_advance(rng.counter)
        return action, logp, mean_c, ls

    def _alpha_step(self, log_probs, sc, info):
        """Temperature loss + its Adam step (one launch); returns log_alpha, or None without entropy tuning."""
        if not self.automatic_entropy_tuning:
            return None
        lp_all = self._all_ranks(log_probs.detach().reshape(-1))      # temperature sees every rank's samples
        alpha_sc = sc
        if lp_all.numel() != sc.B:                  # more samples than the per-rank scratch was sized for
            alpha_sc = getattr(self, "_alpha_sc", None)
            if alpha_sc is None or alpha_sc.B != lp_all.numel():
                alpha_sc = self._alpha_sc = ops.OffPolicyScratch(lp_all.numel(), lp_all.device)
        ops.sac_alpha_step(lp_all, self.target_entropy, self.log_alpha, self._alpha_state, self.plr, alpha_sc,
                           info=info[1:3])
        return self.log_alpha

    def _policy_backward(self, roots, seeds, mean, log_std, info):
        """log_std/* and mean/* statistics, the std / mean regularisers, then one backward into the policy segment
        from the loss kernel's seeded roots plus the regularisers."""
        ops.vec_stats(log_std.detach().reshape(-1) if log_std.is_contiguous() else log_std.detach().contiguous().reshape(-1),
                      out=info[10:14])
        ops.vec_stats(mean.detach().reshape(-1), out=info[14:18])
        if self.policy_std_reg_weight or self.policy_mean_reg_weight:
            std_reg = self.policy_std_reg_weight * (log_std ** 2).mean()
            mean_reg = self.policy_mean_reg_weight * (mean ** 2).mean()
            info[18:19].copy_(std_reg.detach().reshape(1))
            info[19:20].copy_(mean_reg.detach().reshape(1))
            roots.append(std_reg + mean_reg)
            seeds.append(torch.ones((), device=mean.device))
        torch.autograd.backward(roots, seeds, inputs=self.opt.segments[0])

    def _critic_info(self, row):
        raise NotImplementedError

    def _decode_info(self, row, variant):
        info = {'Reward_Mean': float(row[0])}
        if self.automatic_entropy_tuning:
            info["Alpha"] = float(row[1])
            info["Alpha_loss"] = float(row[2])
        info['Training/policy_loss'] = float(row[20] + row[18] + row[19])
        info.update(self._critic_info(row))
        info.update(four_stats('log_std', row[10:14]))
        info.update(four_stats('log_probs', row[self._LOG_PROBS:self._LOG_PROBS + 4]))
        info.update(four_stats('mean', row[14:18]))
        return info


class TwinSACQ(SoftActorCritic):
    _LOG_PROBS = 21              # sac_policy_loss writes [policy_loss, log_probs stats] at 20..24
    TD_COLUMNS = 2

    def __init__(self, pf, qf1, qf2, plr, qlr, optimizer_class=optim.Adam, policy_std_reg_weight=1e-3,
                 policy_mean_reg_weight=1e-3, reparameterization=True, automatic_entropy_tuning=True,
                 target_entropy=None, **kwargs):
        if not reparameterization:
            raise NotImplementedError
        super().__init__(pf, policy_std_reg_weight, policy_mean_reg_weight, reparameterization,
                         automatic_entropy_tuning, target_entropy, **kwargs)
        self.qf1, self.qf2 = qf1, qf2
        self.plr, self.qlr = plr, qlr
        self._init_networks(optimizer_class, [("pf", pf, plr), ("qf1", qf1, qlr), ("qf2", qf2, qlr)], eps=1e-8,
                            max_norms=[self.grad_clip or 0.0] * 3, targets=("qf1", "qf2"))

    def _update_body(self, variant):
        batch, obs, acts, next_obs, rewards, terminals = self._transitions()
        info, sc = self._ub["info"][0], self._ub["scratch"]
        new_actions, log_probs, mean, log_std = self._sample(obs, True)
        q1_pred = self.qf1([obs, acts])
        q2_pred = self.qf2([obs, acts])
        log_alpha = self._alpha_step(log_probs, sc, info)
        with torch.no_grad():
            t_actions, t_logp, _, _ = self._sample(next_obs, False)
            tq1 = self.target_qf1([next_obs, t_actions]).reshape(-1)
            tq2 = self.target_qf2([next_obs, t_actions]).reshape(-1)
            y, _ = ops.td_target(rewards, terminals, tq1, tq2, t_logp.reshape(-1), log_alpha, self.discount, sc,
                                 info=info[0:1], fixed_alpha=1.0)
        g1, g2, _ = self._critic_loss(batch, q1_pred.reshape(-1), q2_pred.reshape(-1), y, info[4:6])
        qn1 = self.qf1([obs, new_actions])
        qn2 = self.qf2([obs, new_actions])
        g_lp, g_qn1, g_qn2, _ = ops.sac_policy_loss(log_probs.reshape(-1), qn1.reshape(-1), qn2.reshape(-1),
                                                    log_alpha, sc, info=info[20:25], fixed_alpha=1.0)
        self._policy_backward([log_probs, qn1, qn2],
                              [g_lp.reshape(log_probs.shape), g_qn1.reshape(qn1.shape), g_qn2.reshape(qn2.shape)],
                              mean, log_std, info)
        self._critic_backward([q1_pred, q2_pred], [g1, g2], 1, 3)
        self._optimizer_step()
        self._update_target_networks()
        self._finish_update()

    def _critic_info(self, row):
        return {'Training/qf1_loss': float(row[4]), 'Training/qf2_loss': float(row[5])}
