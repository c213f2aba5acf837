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
import torch
import torch.optim as optim

from ... import ops
from .twin_sac_q import SoftActorCritic

# info row slots besides SoftActorCritic's: 21 vf_loss 22..25 log_probs stats (sac_v_loss writes 20..25) |
# 26.. pre-clip gradient norms of pf, the critics and vf (grad_clip only)
_NORMS = 26


class SAC(SoftActorCritic):
    _critic_names = ("qf",)
    _LOG_PROBS = 22

    def __init__(self, pf, vf, qf, plr, vlr, qlr, optimizer_class=optim.Adam, policy_std_reg_weight=1e-3,
                 policy_mean_reg_weight=1e-3, reparameterization=True, automatic_entropy_tuning=True,
                 target_entropy=None, **kwargs):
        """`qf`: the critic, or the list of critics that `_critic_names` names (TwinSAC)."""
        super().__init__(pf, policy_std_reg_weight, policy_mean_reg_weight, reparameterization,
                         automatic_entropy_tuning, target_entropy, **kwargs)
        self.vf = vf
        self._critics = qf if isinstance(qf, list) else [qf]
        for name, q in zip(self._critic_names, self._critics):
            setattr(self, name, q)
        self.plr, self.vlr, self.qlr = plr, vlr, qlr
        # vf last: the checkpoint's network order, and the critics' backward reads segments 1 .. vf - 1
        segments = [("pf", pf, plr)] + [(n, q, qlr) for n, q in zip(self._critic_names, self._critics)] + \
            [("vf", vf, vlr)]
        self._vf_seg = self._init_networks(optimizer_class, segments, eps=1e-8,
                                           max_norms=[self.grad_clip or 0.0] * len(segments), targets=("vf",))["vf"]

    def _update_body(self, variant):
        batch, obs, acts, next_obs, rewards, terminals = self._transitions()
        info, sc = self._ub["info"][0], self._ub["scratch"]
        new_actions, log_probs, mean, log_std = self._sample(obs, True)        # the update's only sample
        q_preds = [qf([obs, acts]) for qf in self._critics]
        v_pred = self.vf(obs)
        with torch.no_grad():
            target_v = self.target_vf(next_obs).reshape(-1)
        log_alpha = self._alpha_step(log_probs, sc, info)
        with torch.no_grad():
            y, _ = ops.td_target(rewards, terminals, target_v, None, None, None, self.discount, sc, info=info[0:1])
        q2_pred = q_preds[1].reshape(-1) if len(q_preds) > 1 else None
        g1, g2, _ = self._critic_loss(batch, q_preds[0].reshape(-1), q2_pred, y, info[4:6])
        qns = [qf([obs, new_actions]) for qf in self._critics]
        qn2 = qns[1].reshape(-1) if len(qns) > 1 else None
        g_lp, g_qn1, g_qn2, g_v, _ = ops.sac_v_loss(log_probs.reshape(-1), qns[0].reshape(-1), qn2,
                                                    v_pred.detach().reshape(-1), log_alpha, sc,
                                                    reparameterization=self.reparameterization, info=info[20:26])
        roots, seeds = [log_probs], [g_lp.reshape(log_probs.shape)]
        if self.reparameterization:                     # the policy gradient also flows through Q(s, a~)
            roots += qns
            seeds += [g.reshape(q.shape) for g, q in zip((g_qn1, g_qn2), qns)]
        self._policy_backward(roots, seeds, mean, log_std, info)
        self._critic_backward(q_preds, [g1, g2], 1, self._vf_seg)
        torch.autograd.backward([v_pred], [g_v.reshape(v_pred.shape)], inputs=self.opt.segments[self._vf_seg])
        self._optimizer_step()
        if self.grad_clip:
            info[_NORMS:_NORMS + self.opt.nseg].copy_(self.opt.grad_norms())
        self._update_target_networks()
        self._finish_update()

    def _critic_info(self, row):
        info = {'Training/vf_loss': float(row[21])}
        for i, name in enumerate(self._critic_names):
            info['Training/%s_loss' % name] = float(row[4 + i])
        if self.grad_clip:
            for i, name in enumerate(("pf",) + self._critic_names + ("vf",)):
                info['Training/%s_grad_norm' % name] = float(row[_NORMS + i])
        return info
