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

from ..spaces import Box, Discrete
from .synth import SelfResettingVecEnv

ENV_ID = "Acrobot-v1"
MAX_EPISODE_STEPS = 500
MAX_VEL_1 = 4 * math.pi
MAX_VEL_2 = 9 * math.pi


def is_acrobot(env_id):
    return env_id == ENV_ID


class AcrobotVecEnv(SelfResettingVecEnv):
    """N Acrobot-v1 envs on one GPU.  env_param / first_env / total_envs / dist: as DeviceVecEnv."""

    lockstep = False
    _host_mirror_ok = False
    kernels = "acrobot"
    action_error_msg = "%s takes the actions 0, 1 and 2; another value was passed to step()"

    def __init__(self, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None, max_episode_steps=None):
        # phys: theta1, theta2, dtheta1, dtheta2
        super().__init__(ENV_ID, env_nums, env_param, device, first_env, total_envs,
                         max_episode_steps or MAX_EPISODE_STEPS, 6, 4)
        high = np.array([1.0, 1.0, 1.0, 1.0, MAX_VEL_1, MAX_VEL_2])
        self.observation_space = Box(-high, high)
        self.action_space = Discrete(3)
