"""Bootstrapped DQN (API of /root/reference/torchrl/algo/off_policy/bootstrapped_dqn.py:7-113).

H heads on one trunk; every head regresses on its own target head, and each stored transition carries a Bernoulli
mask that says which heads learn from it.  The update is DQN's with the loss swapped: one all-heads forward of `qf`,
one of `target_qf`, and the whole masked multi-head TD loss with its gradient in ONE launch
(csrc/bootstrapped.cu).  Collection (per-env heads drawn at episode starts, greedy actions, mask rows) is the pixel
collector's captured step with a BootstrappedDQNDiscretePolicy (collector/pixel.py).

Differences from the reference: `sample_key` names "acts" (the reference's "actions" is not what its own update
reads) and collection goes through the vectorised collector (the reference's take_actions uses the removed in-algo
collection API).
"""
import torch

from ... import ops
from .dqn import DQN


class BootstrappedDQN(DQN):
    def __init__(self, head_num=10, bernoulli_p=0.5, **kwargs):
        super().__init__(**kwargs)
        if hasattr(self.replay_buffer, "update_priorities"):
            raise NotImplementedError("BootstrappedDQN has no prioritised-replay form (the reference has none)")
        self.head_num = head_num
        self.bernoulli_p = bernoulli_p
        self.pf.bernoulli_p = bernoulli_p
        self.sample_key = ["obs", "next_obs", "acts", "rewards", "terminals", "masks"]

    # info: 0 loss 1 q_s_a (mean over samples and heads) 2 Reward_Mean
    def _update_body(self, variant):
        ub = self._ub
        batch = self._batch()
        info = ub["info"][0]
        obs, next_obs = self._prep_obs(batch["obs"]), self._prep_obs(batch["next_obs"])
        acts = batch["acts"].reshape(-1).float().contiguous()
        rewards, terminals = batch["rewards"].reshape(-1), batch["terminals"].reshape(-1)
        masks = batch["masks"].reshape(-1, self.head_num)
        pred = self.qf.all_heads(obs)
        with torch.no_grad():
            next_q = self.target_qf.all_heads(next_obs)
        grad, _ = ops.bootstrapped_dqn_loss(pred, next_q, acts, rewards, terminals, masks, self.discount,
                                            ub["scratch"], info=info[0:3])
        torch.autograd.backward([pred], [grad])
        self._optimizer_step()
        self._update_target_networks()
        self._finish_update()

    def _decode_info(self, row, variant):
        return {'Reward_Mean': float(row[2]), 'Training/qf_loss': float(row[0]), 'q_s_a': float(row[1])}
