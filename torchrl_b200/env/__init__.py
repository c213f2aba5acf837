from .get_env import get_env, get_vec_env, get_subprocvec_env  # noqa: F401
from .synth import SynthVecEnv, DeviceNormalizer  # noqa: F401
from .synth import SynthVecEnv as VecEnv  # noqa: F401  (the reference exports VecEnv / SubProcVecEnv)
from .synth import SynthVecEnv as SubProcVecEnv  # noqa: F401
from .synth_atari import SynthAtariVecEnv  # noqa: F401
from .cartpole import CartPoleVecEnv  # noqa: F401
from .pendulum import PendulumVecEnv  # noqa: F401
from .acrobot import AcrobotVecEnv  # noqa: F401
from .mountain_car import MountainCarVecEnv  # noqa: F401
from .bridge import HostEnvBridge  # noqa: F401
from ..hostenv import VecEnv as HostVecEnv, SubProcVecEnv as HostSubProcVecEnv  # noqa: F401
