"""REINFORCE on the device (API of /root/reference/torchrl/algo/on_policy/reinforce.py:7-81).

The policy-gradient half of A2C: advantages are the discounted returns (`gae` is forced off, and the value function is
a ZeroNet, so the collector stores V = 0 without launching anything and the rollout bootstraps with zeros), the loss is
A2C's policy-gradient mode, L = -mean(logp * (adv - mean) / (std + 1e-5)) - c_ent * mean(ent) (reinforce.py:55-60),
and one Adam (eps 1e-8, the torch default the reference keeps) steps the policy after clipping its gradient norm to 0.5.

The device epoch is A2C's minibatch machinery without the critic branch: the epoch's advantage table in one launch, one
captured graph per minibatch (row gather -> policy forward -> actor loss kernel, which also writes every row's log-prob
-> statistics of those log-probs (1) -> autograd -> clip + Adam -> info row) and one info read-back per epoch.  Both
policy heads are served: the Gaussian policies of the continuous envs and CategoricalDisPolicy (CartPole's MLP, the
SynthAtari CNN).  `update(batch)` is the eager form and returns the reference's info dict.
"""
import numpy as np
import torch
import torch.optim as optim

from ... import ops
from ...networks import fused
from ...networks.nets import ZeroNet
from ..utils import four_stats
from .a2c import A2C


class Reinforce(A2C):
    adam_eps = 1e-8

    def __init__(self, pf, plr, optimizer_class=optim.Adam, entropy_coeff=0.001, **kwargs):
        # a vacant value network keeps the on-policy plumbing shared with A2C (reinforce.py:20-21)
        super().__init__(pf=pf, vf=ZeroNet(), plr=plr, vlr=0.0, optimizer_class=optimizer_class,
                         entropy_coeff=entropy_coeff, **kwargs)
        self.gae = False
        self.sample_key = ["obs", "acts", "advs"]

    def _net_segments(self, plr, vlr):
        return [("pf", self.pf, plr)]

    def _gather_keys(self):
        return ["obs", "acts", "advs"]

    def _mb_setup(self):
        st = super()._mb_setup()
        st["logp"] = torch.zeros(st["B"], dtype=torch.float32, device=self.device)
        return st

    def _critic_step(self, batch, info):
        pass

    def _actor_step(self, batch, info):
        st = self._mb_state
        self._head.minibatch_actor(self.pf, batch["obs"], batch["acts"], None, batch["advs"].reshape(-1),
                                   st["adv_table"], st["upd"], 0.0, self.entropy_coeff, st["scratch"], info,
                                   logp_out=st["logp"])
        ops.vec_stats(st["logp"], out=info[32:36])                     # logprob/* (reinforce.py:70-73)

    @staticmethod
    def _info(adv_stats, n, policy_loss, ent, logp_stats):
        """The reference's info dict.  Its advs/* are NumPy statistics of the batch (reinforce.py:42-45), so advs/std
        is the population std; the kernels' table holds torch's unbiased std of the same moments."""
        mean, std, mx, mn = (float(v) for v in adv_stats)
        info = {'advs/mean': mean, 'advs/std': float(np.float64(std) * np.sqrt((n - 1.0) / n)), 'advs/max': mx,
                'advs/min': mn, 'Training/policy_loss': float(policy_loss), 'ent': float(ent)}
        info.update(four_stats('logprob', logp_stats))
        return info

    def _decode_info(self, row, norms, gs):
        W = self.dist.world_size if (self.dist is not None and self.dist.active) else 1
        return self._info(row[20:24], float(self._mb_state["B"] * W), row[0], row[11], row[32:36])

    @fused.presplit_scope
    def update(self, batch):
        """One REINFORCE update on an explicit batch (reinforce.py:33-75), eagerly, through the same loss kernel and
        the fused optimizer step; returns the reference's info dict (this entry point syncs)."""
        self.training_update_num += 1
        obs, acts, advs = self._minibatch(batch, ('obs', 'acts', 'advs'))
        B = obs.shape[0]
        scratch = self._head.loss_scratch(B, acts.reshape(B, -1), self.device)
        info32 = torch.zeros(24, dtype=torch.float32, device=self.device)
        logp = torch.empty(B, dtype=torch.float32, device=self.device)
        adv_stats = ops.vec_stats(advs.reshape(-1), out=info32[16:20])
        self._head.eager_actor(self.pf, obs, acts, None, advs.reshape(-1), adv_stats, 0.0, self.entropy_coeff,
                               scratch, info32[0:16], logp_out=logp)
        ops.vec_stats(logp, out=info32[20:24])
        self._optimizer_step()
        row = info32.cpu().numpy()
        return self._info(row[16:20], float(advs.numel()), row[0], row[11], row[20:24])

    @property
    def snapshot_networks(self):
        return [("pf", self.pf)]
