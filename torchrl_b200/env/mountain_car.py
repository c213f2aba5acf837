"""Device-resident MountainCar-v0 and MountainCarContinuous-v0 with the vec-env API of DeviceVecEnv.

Stands where ``VecEnv(gym.make("MountainCar-v0"))`` and ``NormAct(VecEnv(gym.make("MountainCarContinuous-v0")))`` stand
in the reference (/root/reference/torchrl/env/get_env.py:53, :70-78, env/continuous_wrapper.py:18-20): gym's mountain
car for all N envs in one launch (csrc/mountain_car.cu, defined in oracle/mountain_car.py).  Observations are
(position, velocity) in fp32.
    MountainCar-v0: actions 0, 1, 2 (push left, none, right); reward -1 per step; the episode ends at position >= 0.5
        with velocity >= 0, or at the 200-step time limit.
    MountainCarContinuous-v0: actions in [-1, 1], the force; reward 100 on reaching the goal minus 0.1 force^2 per
        step; the episode ends at position >= 0.45 with velocity >= 0, or at the 999-step time limit.
The physical state is fp64 (`phys`).  Resets draw the position from U(-0.6, -0.4) with the counter hash of the synthetic
envs and set the velocity to 0; the collector's partial reset is the env's own kernel (`resets_itself`), launched right
after the finalize kernel inside the captured step.
"""
import numpy as np
import torch

from .. import ops
from ..spaces import Box, Discrete
from .synth import DeviceVecEnv

# id: (time limit, continuous)
SPECS = {"MountainCar-v0": (200, False), "MountainCarContinuous-v0": (999, True)}
MIN_POSITION, MAX_POSITION, MAX_SPEED = -1.2, 0.6, 0.07


def is_mountain_car(env_id):
    return env_id in SPECS


class MountainCarVecEnv(DeviceVecEnv):
    """N Mountain Car envs of one id on one GPU.  env_param / first_env / total_envs / dist: as DeviceVecEnv."""

    lockstep = False
    _host_mirror_ok = False
    # the collector's finalize kernel leaves this env's counters and observation to `collector_reset`
    resets_itself = True

    def __init__(self, env_id, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None,
                 max_episode_steps=None):
        limit, self.continuous = SPECS[env_id]
        self.action_error_msg = ("%s takes finite actions in [-1, 1]; a NaN or an infinity was passed to step()"
                                 if self.continuous else
                                 "%s takes the actions 0, 1 and 2; another value was passed to step()")
        super().__init__(env_id, env_nums, env_param, device, first_env, total_envs, max_episode_steps or limit, 2, 1,
                         ops.mountain_car_num_ctas(int(env_nums)))
        self.observation_space = Box(np.array([MIN_POSITION, -MAX_SPEED]), np.array([MAX_POSITION, MAX_SPEED]))
        self.action_space = Box(-1.0, 1.0, shape=(1,)) if self.continuous else Discrete(3)
        self.phys = torch.zeros(self.env_nums, 2, dtype=torch.float64, device=self.device)   # position, velocity

    def _reset_kernel(self, mask):
        ops.mountain_car_reset(self.phys, self.state, self.elapsed, self.episode, self.seeds, mask=mask)

    def collector_reset(self, step_count, cur_ob, t_ptr, raw_obs_after_reset):
        """The collector's partial reset (one launch, capturable): new episodes for the envs whose `step_count` the
        finalize kernel just zeroed, and their next observation in `cur_ob` by collect_finalize's rules."""
        nrm = self._obs_normalizer if self.obs_norm else None
        ops.mountain_car_reset(self.phys, self.state, self.elapsed, self.episode, self.seeds, step_count=step_count,
                               next_norm=self.obs_out, cur_ob=cur_ob, any_reset=self.any_reset, t_ptr=t_ptr,
                               norm_mean=None if nrm is None else nrm._mean,
                               norm_var=None if nrm is None else nrm._var, clip=10.0 if nrm is None else nrm.clip,
                               raw_obs_after_reset=raw_obs_after_reset)

    def _step_kernel(self, actions, step_count, moments, t_ptr, reward_scale, max_episode_frames, merge):
        ops.mountain_car_step(self.phys, self.state, actions.reshape(-1), self.elapsed, step_count, self.reward,
                              self.done, self.time_limit, self.action_error, *moments, self._ticket, self.any_reset,
                              t_ptr, reward_scale, self._max_episode_steps, max_episode_frames, merge, self.continuous)
