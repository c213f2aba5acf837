"""Device-resident CartPole-v0 / CartPole-v1 with the vec-env API of DeviceVecEnv.

Stands where ``VecEnv(gym.make("CartPole-v1"))`` stands in the reference (/root/reference/torchrl/env/get_env.py:53,
:70-78): gym's closed-form cart-pole dynamics for all N envs in one launch (csrc/cartpole.cu, defined in
oracle/cartpole.py), reward 1 per step, episodes end when |x| > 2.4, |theta| > 12 degrees or at the time limit
(200 steps for v0, 500 for v1).  Observations are the fp32 state (x, x_dot, theta, theta_dot); actions are 0 (push
left) or 1 (push right).  Resets draw every component from U(-0.05, 0.05) with the counter-hash of the synthetic envs,
so the reset and the collector's in-kernel partial reset are the synthetic envs' own.
"""
import numpy as np

from .. import ops
from ..spaces import Box, Discrete
from .synth import DeviceVecEnv

MAX_EPISODE_STEPS = {"CartPole-v0": 200, "CartPole-v1": 500}
INIT_SCALE = 0.05
X_THRESHOLD = 2.4
THETA_THRESHOLD = 12 * 2 * np.pi / 360


def is_cartpole(env_id):
    return env_id in MAX_EPISODE_STEPS


class CartPoleVecEnv(DeviceVecEnv):
    """N CartPole envs on one GPU.  env_param / first_env / total_envs / dist: as DeviceVecEnv."""

    init_scale = INIT_SCALE
    lockstep = False
    _host_mirror_ok = False
    action_error_msg = "%s takes the actions 0 and 1; another value was passed to step()"

    def __init__(self, env_id, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None,
                 max_episode_steps=None):
        super().__init__(env_id, env_nums, env_param, device, first_env, total_envs,
                         max_episode_steps or MAX_EPISODE_STEPS[env_id], 4, 1, ops.cartpole_num_ctas(int(env_nums)))
        f32max = float(np.finfo(np.float32).max)
        high = np.array([X_THRESHOLD * 2, f32max, THETA_THRESHOLD * 2, f32max])
        self.observation_space = Box(-high, high)
        self.action_space = Discrete(2)

    def _step_kernel(self, actions, step_count, moments, t_ptr, reward_scale, max_episode_frames, merge):
        ops.cartpole_step(self.state, actions.reshape(-1), self.elapsed, step_count, self.reward, self.done,
                          self.time_limit, self.action_error, *moments, self._ticket, self.any_reset, t_ptr,
                          reward_scale, self._max_episode_steps, max_episode_frames, merge)
