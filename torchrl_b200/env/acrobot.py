"""Device-resident Acrobot-v1 with the vec-env API of DeviceVecEnv.

Stands where ``VecEnv(gym.make("Acrobot-v1"))`` stands in the reference (/root/reference/torchrl/env/get_env.py:53,
:70-78): gym's "book" Acrobot (one RK4 step of dt = 0.2 per action, no torque noise) for all N envs in one launch
(csrc/acrobot.cu, defined in oracle/acrobot.py).  Actions are 0, 1, 2 (torque -1, 0, +1); observations are
(cos theta1, sin theta1, cos theta2, sin theta2, dtheta1, dtheta2) in fp32; the reward is -1 per step and 0 on the step
that lifts the tip above the goal line (-cos theta1 - cos(theta1 + theta2) > 1), which ends the episode; the time limit
is 500 steps.  The physical state is fp64 (`phys`).  Resets draw every state component from U(-0.1, 0.1) with the
counter hash of the synthetic envs; the collector's partial reset is the env's own kernel (`resets_itself`), launched
right after the finalize kernel inside the captured step.
"""
import math

import numpy as np
import torch

from .. import ops
from ..spaces import Box, Discrete
from .synth import DeviceVecEnv

ENV_ID = "Acrobot-v1"
MAX_EPISODE_STEPS = 500
MAX_VEL_1 = 4 * math.pi
MAX_VEL_2 = 9 * math.pi


def is_acrobot(env_id):
    return env_id == ENV_ID


class AcrobotVecEnv(DeviceVecEnv):
    """N Acrobot-v1 envs on one GPU.  env_param / first_env / total_envs / dist: as DeviceVecEnv."""

    lockstep = False
    _host_mirror_ok = False
    # the collector's finalize kernel leaves this env's counters and observation to `collector_reset`
    resets_itself = True
    action_error_msg = "%s takes the actions 0, 1 and 2; another value was passed to step()"

    def __init__(self, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None, max_episode_steps=None):
        super().__init__(ENV_ID, env_nums, env_param, device, first_env, total_envs,
                         max_episode_steps or MAX_EPISODE_STEPS, 6, 1, ops.acrobot_num_ctas(int(env_nums)))
        high = np.array([1.0, 1.0, 1.0, 1.0, MAX_VEL_1, MAX_VEL_2])
        self.observation_space = Box(-high, high)
        self.action_space = Discrete(3)
        # theta1, theta2, dtheta1, dtheta2
        self.phys = torch.zeros(self.env_nums, 4, dtype=torch.float64, device=self.device)

    def _reset_kernel(self, mask):
        ops.acrobot_reset(self.phys, self.state, self.elapsed, self.episode, self.seeds, mask=mask)

    def collector_reset(self, step_count, cur_ob, t_ptr, raw_obs_after_reset):
        """The collector's partial reset (one launch, capturable): new episodes for the envs whose `step_count` the
        finalize kernel just zeroed, and their next observation in `cur_ob` by collect_finalize's rules."""
        nrm = self._obs_normalizer if self.obs_norm else None
        ops.acrobot_reset(self.phys, self.state, self.elapsed, self.episode, self.seeds, step_count=step_count,
                          next_norm=self.obs_out, cur_ob=cur_ob, any_reset=self.any_reset, t_ptr=t_ptr,
                          norm_mean=None if nrm is None else nrm._mean, norm_var=None if nrm is None else nrm._var,
                          clip=10.0 if nrm is None else nrm.clip, raw_obs_after_reset=raw_obs_after_reset)

    def _step_kernel(self, actions, step_count, moments, t_ptr, reward_scale, max_episode_frames, merge):
        ops.acrobot_step(self.phys, self.state, actions.reshape(-1), self.elapsed, step_count, self.reward, self.done,
                         self.time_limit, self.action_error, *moments, self._ticket, self.any_reset, t_ptr,
                         reward_scale, self._max_episode_steps, max_episode_frames, merge)
