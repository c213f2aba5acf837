"""On-policy base: bootstrap the value of the state after the last stored row, turn the epoch's rollout into
advantages / returns on the device (K6), then hand minibatches of whole time-rows to `update`
(API of /root/reference/torchrl/algo/on_policy/on_rl_algo.py:6-48)."""
import torch

from ...networks.nets import ZeroNet
from ..rl_algo import RLAlgo

_KEYS = ("obs", "acts", "advs", "estimate_returns")


class OnRLAlgo(RLAlgo):
    def __init__(self, shuffle=True, tau=None, gae=True, **kwargs):
        super().__init__(**kwargs)
        self.shuffle, self.tau, self.gae = shuffle, tau, gae
        self.sample_key = list(_KEYS)

    def _prep_obs(self, x):
        """uint8 frames of the pixel env -> float32 * obs_scale in one launch (ScaledFloatFrame,
        /root/reference/torchrl/env/atari_wrapper.py:171-180); float observations pass through."""
        if x.dtype != torch.uint8:
            return x
        return self.env.to_float(x.contiguous())

    def _bootstrap_value(self):
        """V(next_obs[T-1]) * (1 - terminals[T-1]) as a contiguous (N,) device vector (on_rl_algo.py:23-27); no
        host copy.  A ZeroNet value function (REINFORCE) bootstraps with zeros and launches nothing."""
        if isinstance(self.vf, ZeroNet):
            return torch.zeros(self.replay_buffer.env_nums, dtype=torch.float32, device=self.device)
        tail = self.replay_buffer.last_sample(['next_obs', 'terminals', 'time_limits'])
        alive = 1.0 - tail['terminals'].reshape(-1).float()
        with torch.no_grad():
            return (self.vf(self._prep_obs(tail['next_obs'])).reshape(-1) * alive).contiguous()

    def process_epoch_samples(self):
        """Fill `_advs` / `_estimate_returns` of the buffer: GAE(lambda = tau) or plain discounted returns
        (on_rl_algo.py:28-33)."""
        last_value = self._bootstrap_value()
        if self.gae:
            self.replay_buffer.generalized_advantage_estimation(last_value, self.discount, self.tau)
        else:
            self.replay_buffer.discount_reward(last_value, self.discount)

    def update_per_epoch(self):
        self.process_epoch_samples()
        record = self.logger.add_update_info
        for batch in self.replay_buffer.one_iteration(self.batch_size, self.sample_key, self.shuffle):
            record(self.update(batch))
