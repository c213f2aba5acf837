"""REINFORCE on the device (API of /root/reference/torchrl/algo/on_policy/reinforce.py:7-81).

The policy-gradient half of A2C: advantages are the discounted returns (`gae` is forced off, and the value function is
a ZeroNet, so the collector stores V = 0 without launching anything and the rollout bootstraps with zeros), the loss is
A2C's policy-gradient mode, L = -mean(logp * (adv - mean) / (std + 1e-5)) - c_ent * mean(ent) (reinforce.py:55-60),
and one Adam (eps 1e-8, the torch default the reference keeps) steps the policy after clipping its gradient norm to 0.5.

The device epoch is A2C's minibatch machinery without the critic branch: the epoch's advantage table in one launch, one
captured graph per minibatch (row gather -> policy forward -> actor loss kernel, which also writes every row's log-prob
-> statistics of those log-probs (1) -> autograd -> clip + Adam -> info row) and one info read-back per epoch.  Both
policy heads are served: the Gaussian policies of the continuous envs and CategoricalDisPolicy (CartPole's MLP, the
SynthAtari CNN).  `update(batch)` runs the same minibatch step on an explicit batch and returns the reference's info
dict.
"""
import numpy as np
import torch
import torch.optim as optim

from ... import ops
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

    def _step_state(self, B, U, a):
        st = super()._step_state(B, U, a)
        st["logp"] = torch.zeros(B, dtype=torch.float32, device=self.device)
        return st

    def _critic_step(self, batch, st, info):
        pass

    def _actor_step(self, batch, st, info):
        self._head.actor(self.pf, batch["obs"], batch["acts"], None, batch["advs"].reshape(-1), st["adv_table"],
                         st["upd"], 0.0, self.entropy_coeff, st["scratch"], info, logp_out=st["logp"])
        ops.vec_stats(st["logp"], out=info[32:36])                     # logprob/* (reinforce.py:70-73)

    def _decode_info(self, row, norms, st):
        """The reference's info dict.  Its advs/* are NumPy statistics of the batch (reinforce.py:42-45), so advs/std
        is the population std; the kernels' table holds torch's unbiased std of the same n samples."""
        mean, std, mx, mn = (float(v) for v in row[20:24])
        n = float(st["n"])
        info = {'advs/mean': mean, 'advs/std': float(np.float64(std) * np.sqrt((n - 1.0) / n)), 'advs/max': mx,
                'advs/min': mn, 'Training/policy_loss': float(row[0]), 'ent': float(row[11])}
        info.update(four_stats('logprob', row[32:36]))
        return info

    @property
    def networks(self):
        return [self.pf, self.vf]        # the ZeroNet value function has no optimizer segment but is in checkpoints
