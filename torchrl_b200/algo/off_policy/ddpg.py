"""DDPG (API of /root/reference/torchrl/algo/off_policy/ddpg.py:10-137) on the off-policy kernels.

One update = TD target launch (K10, single critic), critic MSE launch, the deterministic policy gradient
through the (pre-step) critic, ONE fused clip+Adam launch over the flat {pf, qf} buffer and one Polyak
launch.  The reference steps the actor before the critic (ddpg.py:80-92); both losses are evaluated before
either step and touch disjoint parameter sets, so the fused step is the same arithmetic.
"""
import copy

import torch
import torch.optim as optim

from ... import ops
from ..utils import four_stats
from .off_rl_algo import OffRLAlgo


class DDPG(OffRLAlgo):
    def __init__(self, pf, qf, plr, qlr, optimizer_class=optim.Adam, **kwargs):
        super().__init__(**kwargs)
        self.pf = pf
        self.target_pf = copy.deepcopy(pf)
        self.qf = qf
        self.target_qf = copy.deepcopy(qf)
        self.to(self.device)
        self.plr, self.qlr = plr, qlr
        self._init_optimizer(optimizer_class, [("pf", pf, plr), ("qf", qf, qlr)], eps=1e-8,
                             max_norms=[self.grad_clip or 0.0] * 2)
        self._init_targets()

    # info: 0 Reward_Mean | 4 qf_loss | 6 policy_loss | 10..13 new_actions stats
    def _update_body(self, variant):
        ub = self._ub
        batch = self._batch()
        info = ub["info"][0]
        sc = ub["scratch"]
        obs, acts, next_obs = batch["obs"], batch["acts"], batch["next_obs"]
        rewards, terminals = batch["rewards"].reshape(-1), batch["terminals"].reshape(-1)
        B = obs.shape[0]
        acts = acts.reshape(B, -1)
        with torch.no_grad():
            t_act = self.target_pf(next_obs).contiguous()
            tq = self.target_qf([next_obs, t_act]).reshape(-1).contiguous()
            y, _ = ops.td_target(rewards, terminals, tq, None, None, None, self.discount, sc, info=info[0:1])
        new_actions = self.pf(obs)
        q_new = self.qf([obs, new_actions])
        info[6:7].copy_((-q_new.detach().mean()).reshape(1))
        seed = torch.full_like(q_new, -1.0 / q_new.numel())
        torch.autograd.backward([q_new], [seed], inputs=self.opt.segments[0])
        q_pred = self.qf([obs, acts])
        g, _, _ = self._critic_loss(batch, q_pred.reshape(-1), None, y, info[4:6])
        torch.autograd.backward([q_pred], [g.reshape(q_pred.shape)], inputs=self.opt.segments[1])
        self._optimizer_step(0b11)
        self._update_target_networks()
        ops.vec_stats(new_actions.detach().reshape(-1), out=info[10:14])
        self._finish_update()

    def _decode_info(self, row, variant):
        info = {'Reward_Mean': float(row[0]), 'Training/policy_loss': float(row[6]),
                'Training/qf_loss': float(row[4])}
        info.update(four_stats('new_actions', row[10:14]))
        return info

    @property
    def networks(self):
        return [self.pf, self.qf, self.target_pf, self.target_qf]

    @property
    def snapshot_networks(self):
        return [["pf", self.pf], ["qf", self.qf]]

    @property
    def target_networks(self):
        return [(self.pf, self.target_pf), (self.qf, self.target_qf)]
