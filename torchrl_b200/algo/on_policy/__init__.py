from .a2c import A2C  # noqa: F401
from .ppo import PPO  # noqa: F401
from .reinforce import Reinforce  # noqa: F401
from .trpo import TRPO  # noqa: F401
from .v_mpo import VMPO  # noqa: F401
