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

from ..spaces import Box, Discrete
from .synth import SelfResettingVecEnv

# id: (time limit, continuous)
SPECS = {"MountainCar-v0": (200, False), "MountainCarContinuous-v0": (999, True)}
MIN_POSITION, MAX_POSITION, MAX_SPEED = -1.2, 0.6, 0.07


def is_mountain_car(env_id):
    return env_id in SPECS


class MountainCarVecEnv(SelfResettingVecEnv):
    """N Mountain Car envs of one id on one GPU.  env_param / first_env / total_envs / dist: as DeviceVecEnv."""

    lockstep = False
    _host_mirror_ok = False
    kernels = "mountain_car"
    step_extra = ("continuous",)

    def __init__(self, env_id, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None,
                 max_episode_steps=None):
        limit, self.continuous = SPECS[env_id]
        self.action_error_msg = ("%s takes finite actions in [-1, 1]; a NaN or an infinity was passed to step()"
                                 if self.continuous else
                                 "%s takes the actions 0, 1 and 2; another value was passed to step()")
        # phys: position, velocity
        super().__init__(env_id, env_nums, env_param, device, first_env, total_envs, max_episode_steps or limit, 2, 2)
        self.observation_space = Box(np.array([MIN_POSITION, -MAX_SPEED]), np.array([MAX_POSITION, MAX_SPEED]))
        self.action_space = Box(-1.0, 1.0, shape=(1,)) if self.continuous else Discrete(3)
