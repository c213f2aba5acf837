"""Device-resident Pendulum-v1 with the vec-env API of DeviceVecEnv.

Stands where ``NormAct(VecEnv(gym.make("Pendulum-v1")))`` stands in the reference (/root/reference/torchrl/env/get_env.py:53,
:70-78, env/continuous_wrapper.py:18-20): gym's Pendulum-v1 for all N envs in one launch (csrc/pendulum.cu, defined in
oracle/pendulum.py).  Actions are in [-1, 1] and map to a torque in [-2, 2]; observations are (cos theta, sin theta,
theta_dot) in fp32; the reward is minus gym's cost; there is no terminal state, every episode ends at the 200-step time
limit, so all envs run in lock step.  The physical state (theta, theta_dot) is fp64 (`phys`).  Resets draw theta from
U(-pi, pi) and theta_dot from U(-1, 1) with the counter hash of the synthetic envs; the collector's partial reset is the
env's own kernel (`resets_itself`), launched right after the finalize kernel inside the captured step.

Only v1 is served: Pendulum-v0 moves the angle with the unclipped velocity, which this kernel does not compute.
"""
import numpy as np

from ..spaces import Box
from .synth import SelfResettingVecEnv

ENV_ID = "Pendulum-v1"
MAX_EPISODE_STEPS = 200
MAX_SPEED = 8.0


def is_pendulum(env_id):
    return env_id == ENV_ID


class PendulumVecEnv(SelfResettingVecEnv):
    """N Pendulum-v1 envs on one GPU.  env_param / first_env / total_envs / dist: as DeviceVecEnv."""

    lockstep = True
    kernels = "pendulum"
    action_error_msg = "%s takes finite actions in [-1, 1]; a NaN or an infinity was passed to step()"

    def __init__(self, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None, max_episode_steps=None):
        # phys: theta, theta_dot
        super().__init__(ENV_ID, env_nums, env_param, device, first_env, total_envs,
                         max_episode_steps or MAX_EPISODE_STEPS, 3, 2)
        self.observation_space = Box(np.array([-1.0, -1.0, -MAX_SPEED]), np.array([1.0, 1.0, MAX_SPEED]))
        self.action_space = Box(-1.0, 1.0, shape=(1,))
