from .on_policy import A2C, PPO, Reinforce, TRPO, VMPO  # noqa: F401
from .off_policy import TwinSACQ, SAC, TwinSAC, TD3, DQN, BootstrappedDQN, QRDQN, DDPG  # noqa: F401
from .rl_algo import RLAlgo  # noqa: F401

__all__ = ['TwinSACQ', 'SAC', 'TwinSAC', 'TD3', 'DQN', 'BootstrappedDQN', 'QRDQN', 'DDPG', 'A2C', 'PPO', 'Reinforce', 'TRPO', 'VMPO',
           'RLAlgo']
