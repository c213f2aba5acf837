"""Host-side (CPU) vectorised envs and per-env wrapper chain for real gym-style environments.
NumPy only -- no torch import here, so spawned env workers start fast."""
from .vecenv import VecEnv, SubProcVecEnv  # noqa: F401
from .wrappers import HostEnv, get_single_env  # noqa: F401
from .atari import AtariHostEnv, get_atari_env  # noqa: F401
