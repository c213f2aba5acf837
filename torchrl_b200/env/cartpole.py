"""Device-resident CartPole-v0 / CartPole-v1 with the vec-env API of SynthVecEnv.

Stands where ``VecEnv(gym.make("CartPole-v1"))`` stands in the reference (/root/reference/torchrl/env/get_env.py:53,
:70-78): gym's closed-form cart-pole dynamics for all N envs in one launch (csrc/cartpole.cu, defined in
oracle/cartpole.py), reward 1 per step, episodes end when |x| > 2.4, |theta| > 12 degrees or at the time limit
(200 steps for v0, 500 for v1).  Observations are the fp32 state (x, x_dot, theta, theta_dot); actions are 0 (push
left) or 1 (push right).  Resets draw every component from U(-0.05, 0.05) with the counter-hash of the synthetic envs,
so the reset and the collector's in-kernel partial reset are the synthetic envs' own.
"""
import numpy as np
import torch

from .. import ops
from ..spaces import Box, Discrete
from .synth import DeviceNormalizer, SynthVecEnv

F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32

MAX_EPISODE_STEPS = {"CartPole-v0": 200, "CartPole-v1": 500}
INIT_SCALE = 0.05
X_THRESHOLD = 2.4
THETA_THRESHOLD = 12 * 2 * np.pi / 360


def is_cartpole(env_id):
    return env_id in MAX_EPISODE_STEPS


class CartPoleVecEnv(SynthVecEnv):
    """N CartPole envs on one GPU.  env_param / first_env / total_envs / dist: as SynthVecEnv."""

    init_scale = INIT_SCALE
    lockstep = False

    def __init__(self, env_id, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None,
                 max_episode_steps=None):
        env_param = dict(env_param or {})
        self.env_id = env_id
        self.env_nums = int(env_nums)
        self.device = torch.device(device)
        self.obs_dim, self.act_dim = 4, 1
        self.first_env = int(first_env)
        self.total_envs = int(total_envs) if total_envs is not None else self.env_nums
        self._max_episode_steps = int(max_episode_steps or MAX_EPISODE_STEPS[env_id])
        self._reward_scale = env_param.get("reward_scale", 1)
        self.obs_norm = bool(env_param.get("obs_norm", False))
        self.training = True
        f32max = float(np.finfo(np.float32).max)
        high = np.array([X_THRESHOLD * 2, f32max, THETA_THRESHOLD * 2, f32max])
        self.observation_space = Box(-high, high)
        self.action_space = Discrete(2)
        N, o, dev = self.env_nums, self.obs_dim, self.device
        self.state = torch.zeros(N, o, dtype=F32, device=dev)       # raw observation
        self.elapsed = torch.zeros(N, dtype=I32, device=dev)
        self.episode = torch.zeros(N, dtype=I32, device=dev)
        self.seeds = torch.zeros(N, dtype=I32, device=dev)
        self.reward = torch.zeros(N, dtype=F32, device=dev)
        self.done = torch.zeros(N, dtype=U8, device=dev)
        self.time_limit = torch.zeros(N, dtype=U8, device=dev)
        self.action_error = torch.zeros(1, dtype=I32, device=dev)
        self.obs_out = torch.zeros(N, o, dtype=F32, device=dev)     # what step() returns (normalised if obs_norm)
        self._partial = torch.zeros(ops.cartpole_num_ctas(N), 2 * o, dtype=F64, device=dev)
        self.batch_sums = torch.zeros(2 * o, dtype=F64, device=dev)
        self._ticket = torch.zeros(1, dtype=I32, device=dev)
        self.any_reset = torch.zeros(2, dtype=I32, device=dev)
        self._obs_normalizer = DeviceNormalizer((o,), device=dev) if self.obs_norm else None
        self._obs = None
        self._host_elapsed = 0
        self._host_mirror_ok = False
        self._dist = None
        self._sums_red = None
        self.seed(0)

    def launch_step(self, actions, step_count=None, max_episode_frames=0, t_ptr=None):
        """Advance all envs one step: state/reward/done/time_limit staging buffers are updated and, with obs_norm,
        `obs_out` receives what env.step would return.  No host sync; an invalid action is reported by
        `check_actions`."""
        update = self.obs_norm and self.training and self._obs_normalizer.should_estimate
        nrm = self._obs_normalizer
        distributed = self.dist is not None and self.dist.active
        rs = float(self._reward_scale) if self.training else 1.0
        moments = (self._partial, self.batch_sums, nrm._mean, nrm._var, nrm._count) if update else (None,) * 5
        ops.cartpole_step(self.state, actions.reshape(-1), self.elapsed, step_count, self.reward, self.done,
                          self.time_limit, self.action_error, *moments, self._ticket, self.any_reset, t_ptr, rs,
                          self._max_episode_steps, int(max_episode_frames) if step_count is not None else (1 << 30),
                          update and not distributed)
        if update and distributed:
            ops.obs_norm_merge(self._reduce_sums(), self.total_envs, nrm._mean, nrm._var, nrm._count)
        if self.obs_norm:
            ops.obs_norm_filt(self.state, nrm._mean, nrm._var, nrm.clip, self.obs_out)
        return self.obs_out

    def check_actions(self):
        """Raise if any step since the last check received an action other than 0 or 1 (one host sync)."""
        if int(self.action_error.item()) != 0:
            self.action_error.zero_()
            raise ValueError("%s takes the actions 0 and 1; another value was passed to step()" % self.env_id)

    def step(self, actions):
        """obs (N,4), reward (N,1), done (N,1) bool, {'time_limit': (N,) bool} -- device tensors."""
        actions = torch.as_tensor(actions, device=self.device).reshape(-1).to(F32).contiguous()
        if actions.numel() != self.env_nums:
            raise ValueError("%s.step: %d actions for %d envs" % (self.env_id, actions.numel(), self.env_nums))
        self.launch_step(actions)
        if not self.obs_norm:
            self.obs_out.copy_(self.state)
        self.check_actions()
        infos = {"time_limit": self.time_limit.bool()}
        return self.obs_out, self.reward.unsqueeze(-1), self.done.bool().unsqueeze(-1), infos
