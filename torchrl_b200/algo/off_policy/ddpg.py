"""DDPG (API of /root/reference/torchrl/algo/off_policy/ddpg.py:10-137) on the off-policy kernels.

One update = TD target launch (K10, single critic), critic MSE launch, the deterministic policy gradient
through the (pre-step) critic, ONE fused clip+Adam launch over the flat {pf, qf} buffer and one Polyak
launch.  The reference steps the actor before the critic (ddpg.py:80-92); both losses are evaluated before
either step and touch disjoint parameter sets, so the fused step is the same arithmetic.
"""
import torch
import torch.optim as optim

from ... import ops
from ..utils import four_stats
from .off_rl_algo import OffRLAlgo


class DDPG(OffRLAlgo):
    def __init__(self, pf, qf, plr, qlr, optimizer_class=optim.Adam, **kwargs):
        super().__init__(**kwargs)
        self.pf, self.qf = pf, qf
        self.plr, self.qlr = plr, qlr
        self._init_networks(optimizer_class, [("pf", pf, plr), ("qf", qf, qlr)], eps=1e-8,
                            max_norms=[self.grad_clip or 0.0] * 2, targets=("pf", "qf"))

    # info: 0 Reward_Mean | 4 qf_loss | 6 policy_loss | 10..13 new_actions stats
    def _update_body(self, variant):
        batch, obs, acts, next_obs, rewards, terminals = self._transitions()
        info, sc = self._ub["info"][0], self._ub["scratch"]
        with torch.no_grad():
            t_act = self.target_pf(next_obs).contiguous()
            tq = self.target_qf([next_obs, t_act]).reshape(-1).contiguous()
            y, _ = ops.td_target(rewards, terminals, tq, None, None, None, self.discount, sc, info=info[0:1])
        new_actions = self._deterministic_policy_step(self.qf, obs, info)
        q_pred = self.qf([obs, acts])
        g, _, _ = self._critic_loss(batch, q_pred.reshape(-1), None, y, info[4:6])
        self._critic_backward([q_pred], [g], 1, 2)
        self._optimizer_step(0b11)
        self._update_target_networks()
        ops.vec_stats(new_actions.detach().reshape(-1), out=info[10:14])
        self._finish_update()

    def _decode_info(self, row, variant):
        info = {'Reward_Mean': float(row[0]), 'Training/policy_loss': float(row[6]),
                'Training/qf_loss': float(row[4])}
        info.update(four_stats('new_actions', row[10:14]))
        return info
