"""Env factories with the reference's names (/root/reference/torchrl/env/get_env.py:32-87).

Synthetic ids ("SynthHalfCheetah-v0", "SynthAnt-v0") build the device-resident
SynthVecEnv, "SynthAtari-v0" the pixel env, "CartPole-v0" / "CartPole-v1" the device CartPole, "Pendulum-v1" the
device Pendulum, "Acrobot-v1" the device Acrobot and "MountainCar-v0" / "MountainCarContinuous-v0" the device Mountain
Car; any other id (Pendulum-v0 included: its dynamics differ from v1's) needs a real gym + the host-env
bridge (SURVEY.md section 8(f).1), which is outside this round's hot path and raises.
"""
import torch

from . import synth_spec
from .acrobot import AcrobotVecEnv, is_acrobot
from .cartpole import CartPoleVecEnv, is_cartpole
from .mountain_car import MountainCarVecEnv, is_mountain_car
from .pendulum import PendulumVecEnv, is_pendulum
from .synth import SynthVecEnv
from .synth_atari import SynthAtariVecEnv, ENV_ID as ATARI_ID


def _device(device):
    if device is not None:
        return device
    if not torch.cuda.is_available():
        raise RuntimeError("torchrl_b200 envs live on the GPU: no CUDA device available (there is no CPU path)")
    return "cuda"


def get_vec_env(env_id, env_param, vec_env_nums, device=None, **kwargs):
    if synth_spec.is_synth(env_id):
        return SynthVecEnv(env_id, vec_env_nums, env_param, device=_device(device), **kwargs)
    if env_id == ATARI_ID:
        return SynthAtariVecEnv(vec_env_nums, env_param, device=_device(device), **kwargs)
    if is_cartpole(env_id):
        return CartPoleVecEnv(env_id, vec_env_nums, env_param, device=_device(device), **kwargs)
    if is_pendulum(env_id):
        return PendulumVecEnv(vec_env_nums, env_param, device=_device(device), **kwargs)
    if is_acrobot(env_id):
        return AcrobotVecEnv(vec_env_nums, env_param, device=_device(device), **kwargs)
    if is_mountain_car(env_id):
        return MountainCarVecEnv(env_id, vec_env_nums, env_param, device=_device(device), **kwargs)
    raise NotImplementedError("only the synthetic device envs are built in this round: %r" % (env_id,))


def get_subprocvec_env(env_id, env_param, vec_env_nums, proc_nums, device=None, **kwargs):
    """`proc_nums` is accepted for API compatibility: the device env needs no worker processes."""
    return get_vec_env(env_id, env_param, vec_env_nums, device=device, **kwargs)


def get_env(env_id, env_param, device=None):
    return get_vec_env(env_id, env_param, 1, device=device)
