"""TD3 (API of /root/reference/torchrl/algo/off_policy/td3.py:10-191).

Keeps the reference's conventions, including the actor/target update firing when
`training_update_num % policy_update_delay` is NON-zero (td3.py:124; SURVEY.md A.8) and the target
action coming from `target_pf.explore` (exploration noise included) before the clipped smoothing
noise is added (td3.py:72-84).  Two captured graph variants: critics only / critics + actor.
"""
import torch
import torch.optim as optim

from ... import ops
from ...policies import distribution as D
from ...policies.continuous_policy import _DeviceRng
from ..utils import four_stats
from .off_rl_algo import OffRLAlgo


class TD3(OffRLAlgo):
    TD_COLUMNS = 2

    def __init__(self, pf, qf1, qf2, plr, qlr, optimizer_class=optim.Adam, policy_update_delay=2,
                 norm_std_policy=0.2, noise_clip=0.5, **kwargs):
        super().__init__(**kwargs)
        self.pf, self.qf1, self.qf2 = pf, qf1, qf2
        self.plr, self.qlr = plr, qlr
        self._init_networks(optimizer_class, [("pf", pf, plr), ("qf1", qf1, qlr), ("qf2", qf2, qlr)], eps=1e-8,
                            max_norms=[self.grad_clip or 0.0] * 3, targets=("pf", "qf1", "qf2"))
        self.policy_update_delay = policy_update_delay
        self.norm_std_policy = norm_std_policy
        self.noise_clip = noise_clip
        self._rng = _DeviceRng()

    def _variant(self):
        return 1 if (self.training_update_num % self.policy_update_delay) else 0

    # info: 0 Reward_Mean | 4 qf1_loss 5 qf2_loss | 6 policy_loss | 10..13 new_actions stats
    def _update_body(self, variant):
        batch, obs, acts, next_obs, rewards, terminals = self._transitions()
        info, sc = self._ub["info"][0], self._ub["scratch"]
        with torch.no_grad():
            t_act = self.target_pf.explore(next_obs)["action"].contiguous()
            if D.get_noise_mode() == "reference_cpu":
                eps = torch.distributions.Normal(torch.zeros(t_act.size()), torch.ones(t_act.size())).sample()
                eps = eps.to(t_act.device)
                t_act = ops.td3_smooth_action(t_act, self.norm_std_policy, self.noise_clip, eps=eps)
            else:
                rng = self._rng.ensure(t_act.device)
                t_act = ops.td3_smooth_action(t_act, self.norm_std_policy, self.noise_clip, rng=rng)
                ops.counter_advance(rng.counter)
            tq1 = self.target_qf1([next_obs, t_act]).reshape(-1)
            tq2 = self.target_qf2([next_obs, t_act]).reshape(-1)
            y, _ = ops.td_target(rewards, terminals, tq1, tq2, None, None, self.discount, sc, info=info[0:1])
        q1_pred = self.qf1([obs, acts])
        q2_pred = self.qf2([obs, acts])
        g1, g2, _ = self._critic_loss(batch, q1_pred.reshape(-1), q2_pred.reshape(-1), y, info[4:6])
        self._critic_backward([q1_pred, q2_pred], [g1, g2], 1, 3)
        self._optimizer_step(0b110)
        if variant == 1:
            new_actions = self._deterministic_policy_step(self.qf1, obs, info)    # qf1 AFTER its step (reference)
            self._optimizer_step(0b001)
            self._update_target_networks()
            ops.vec_stats(new_actions.detach().reshape(-1), out=info[10:14])
        self._finish_update()

    def _decode_info(self, row, variant):
        info = {'Reward_Mean': float(row[0]), 'Training/qf1_loss': float(row[4]), 'Training/qf2_loss': float(row[5])}
        if variant == 1:
            info['Training/policy_loss'] = float(row[6])
            info.update(four_stats('new_actions', row[10:14]))
        return info
