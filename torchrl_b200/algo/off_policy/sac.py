"""Soft actor-critic with a state-value network V and a Polyak-averaged target V
(API of /root/reference/torchrl/algo/off_policy/sac.py:10-231; TwinSAC in twin_sac.py).

Per update (one captured CUDA graph): row gather -> pf(obs) + sampling/log-prob kernel (autograd) ->
Q(obs,a), V(obs), [no grad] V_target(next_obs) -> temperature loss + its Adam step (1 launch) ->
TD-target kernel in its single-critic, no-entropy form y = r + (1-d)*gamma*V_target(s') -> critic MSE
kernel -> Q(obs, a~) -> value/policy loss kernel (value target, value MSE, policy loss, their gradients)
-> three autograd.backward calls seeded with the kernel gradients, each restricted to its own segment ->
fused clip+Adam over pf | critics | vf -> Polyak over the flat target V -> log row.

The reference's `assert v_target == v_pred` (sac.py:130, twin_sac.py:142) raises for every batch of more than
one row; it is not reproduced (DESIGN.md deviation 17): the update is the one the reference runs under `python -O`.
"""
import copy

import numpy as np
import torch
import torch.optim as optim

from ... import ops
from ...flat import FlatAdam, FlatParams
from ..rl_algo import SegmentOptimizer
from .off_rl_algo import OffRLAlgo
from .twin_sac_q import TwinSACQ

_STAT = ("mean", "std", "max", "min")

# info row layout
#  0 Reward_Mean | 1 Alpha 2 Alpha_loss | 4.. critic losses | 10..13 log_std stats | 14..17 mean stats
#  18 std_reg 19 mean_reg | 20 policy_loss (kernel part) 21 vf_loss 22..25 log_probs stats
#  26.. pre-clip gradient norms of pf, the critics and vf (grad_clip only)
_NORMS = 26


class SAC(OffRLAlgo):
    _critic_names = ("qf",)

    def __init__(self, pf, vf, qf, plr, vlr, qlr, optimizer_class=optim.Adam, policy_std_reg_weight=1e-3,
                 policy_mean_reg_weight=1e-3, reparameterization=True, automatic_entropy_tuning=True,
                 target_entropy=None, **kwargs):
        self._init_sac_v(pf, vf, [qf], plr, vlr, qlr, optimizer_class, policy_std_reg_weight, policy_mean_reg_weight,
                         reparameterization, automatic_entropy_tuning, target_entropy, kwargs)

    def _init_sac_v(self, pf, vf, critics, plr, vlr, qlr, optimizer_class, policy_std_reg_weight,
                    policy_mean_reg_weight, reparameterization, automatic_entropy_tuning, target_entropy, kwargs):
        OffRLAlgo.__init__(self, **kwargs)
        self.pf, self.vf = pf, vf
        for name, qf in zip(self._critic_names, critics):
            setattr(self, name, qf)
        self._critics = list(critics)
        self.target_vf = copy.deepcopy(vf)
        self.to(self.device)
        self.plr, self.vlr, self.qlr = plr, vlr, qlr
        if optimizer_class is not optim.Adam:
            raise NotImplementedError("torchrl_b200 fuses clip+Adam in CUDA; only optim.Adam is supported")
        nq = len(critics)
        clip = self.grad_clip if self.grad_clip else 0.0
        # vf last: the Polyak source is one contiguous slice of the flat buffer
        self.opt = FlatAdam([self.pf] + self._critics + [self.vf], lrs=[plr] + [qlr] * nq + [vlr], eps=1e-8,
                            max_norms=[clip] * (nq + 2), device=self.device, dist=self.dist)
        self._vf_seg = nq + 1
        self.pf_optimizer = SegmentOptimizer(self.opt, 0)
        for i, name in enumerate(self._critic_names):
            setattr(self, name + "_optimizer", SegmentOptimizer(self.opt, 1 + i))
        self.vf_optimizer = SegmentOptimizer(self.opt, self._vf_seg)
        self._target_flat = FlatParams([self.target_vf], device=self.device)
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

    _sample = TwinSACQ._sample

    def _target_source(self):
        return self.opt.seg_slice(self._vf_seg)

    def _update_body(self, variant):
        ub = self._ub
        batch = self._batch()
        info = ub["info"][0]
        sc = ub["scratch"]
        obs, acts, next_obs = batch["obs"], batch["acts"], batch["next_obs"]
        rewards, terminals = batch["rewards"].reshape(-1), batch["terminals"].reshape(-1)
        B = obs.shape[0]
        acts = acts.reshape(B, -1)
        new_actions, log_probs, mean, log_std = self._sample(obs, True)        # the update's only sample
        q_preds = [qf([obs, acts]) for qf in self._critics]
        v_pred = self.vf(obs)
        with torch.no_grad():
            target_v = self.target_vf(next_obs).reshape(-1)
        log_alpha = None
        if self.automatic_entropy_tuning:
            lp_all = self._all_ranks(log_probs.detach().reshape(-1))      # temperature sees every rank's samples
            alpha_sc = sc
            if lp_all.numel() != sc.B:                  # more samples than the per-rank scratch was sized for
                alpha_sc = getattr(self, "_alpha_sc", None)
                if alpha_sc is None or alpha_sc.B != lp_all.numel():
                    alpha_sc = self._alpha_sc = ops.OffPolicyScratch(lp_all.numel(), lp_all.device)
            ops.sac_alpha_step(lp_all, self.target_entropy, self.log_alpha, self._alpha_state, self.plr, alpha_sc,
                               info=info[1:3])
            log_alpha = self.log_alpha
        with torch.no_grad():
            y, _ = ops.td_target(rewards, terminals, target_v, None, None, None, self.discount, sc, info=info[0:1])
        q2_pred = q_preds[1].reshape(-1) if len(q_preds) > 1 else None
        g1, g2, _ = ops.twin_mse_loss(q_preds[0].reshape(-1), q2_pred, y, sc, info=info[4:6])
        qns = [qf([obs, new_actions]) for qf in self._critics]
        qn2 = qns[1].reshape(-1) if len(qns) > 1 else None
        g_lp, g_qn1, g_qn2, g_v, _ = ops.sac_v_loss(log_probs.reshape(-1), qns[0].reshape(-1), qn2,
                                                    v_pred.detach().reshape(-1), log_alpha, sc,
                                                    reparameterization=self.reparameterization, info=info[20:26])
        ops.vec_stats(log_std.detach().reshape(-1) if log_std.is_contiguous() else log_std.detach().contiguous().reshape(-1),
                      out=info[10:14])
        ops.vec_stats(mean.detach().reshape(-1), out=info[14:18])
        roots, seeds = [log_probs], [g_lp.reshape(log_probs.shape)]
        if self.reparameterization:                     # the policy gradient also flows through Q(s, a~)
            roots += qns
            seeds += [g.reshape(q.shape) for g, q in zip((g_qn1, g_qn2), qns)]
        if self.policy_std_reg_weight or self.policy_mean_reg_weight:
            std_reg = self.policy_std_reg_weight * (log_std ** 2).mean()
            mean_reg = self.policy_mean_reg_weight * (mean ** 2).mean()
            info[18:19].copy_(std_reg.detach().reshape(1))
            info[19:20].copy_(mean_reg.detach().reshape(1))
            roots.append(std_reg + mean_reg)
            seeds.append(torch.ones((), device=obs.device))
        segs = self.opt.segments
        torch.autograd.backward(roots, seeds, inputs=segs[0])
        torch.autograd.backward(q_preds, [g.reshape(q.shape) for g, q in zip((g1, g2), q_preds)],
                                inputs=[p for s in segs[1:self._vf_seg] for p in s])
        torch.autograd.backward([v_pred], [g_v.reshape(v_pred.shape)], inputs=segs[self._vf_seg])
        self._step()
        if self.grad_clip:
            info[_NORMS:_NORMS + self.opt.nseg].copy_(self.opt.grad_norms())
        self._update_target_networks()
        if self._explicit_batch is None:
            self._finish_update()

    def _decode_info(self, row, variant):
        info = {'Reward_Mean': float(row[0])}
        if self.automatic_entropy_tuning:
            info["Alpha"] = float(row[1])
            info["Alpha_loss"] = float(row[2])
        info['Training/policy_loss'] = float(row[20] + row[18] + row[19])
        info['Training/vf_loss'] = float(row[21])
        for i, name in enumerate(self._critic_names):
            info['Training/%s_loss' % name] = float(row[4 + i])
        if self.grad_clip:
            for i, name in enumerate(("pf",) + self._critic_names + ("vf",)):
                info['Training/%s_grad_norm' % name] = float(row[_NORMS + i])
        for i, s in enumerate(_STAT):
            info['log_std/' + s] = float(row[10 + i])
        for i, s in enumerate(_STAT):
            info['log_probs/' + s] = float(row[22 + i])
        for i, s in enumerate(_STAT):
            info['mean/' + s] = float(row[14 + i])
        return info

    @property
    def networks(self):
        return [self.pf] + self._critics + [self.vf, self.target_vf]

    @property
    def snapshot_networks(self):
        return [["pf", self.pf]] + [[n, q] for n, q in zip(self._critic_names, self._critics)] + [["vf", self.vf]]

    @property
    def target_networks(self):
        return [(self.vf, self.target_vf)]
