from .twin_sac_q import TwinSACQ  # noqa: F401
from .sac import SAC  # noqa: F401
from .twin_sac import TwinSAC  # noqa: F401
from .td3 import TD3  # noqa: F401
from .dqn import DQN, QRDQN  # noqa: F401
from .bootstrapped_dqn import BootstrappedDQN  # noqa: F401
from .ddpg import DDPG  # noqa: F401
