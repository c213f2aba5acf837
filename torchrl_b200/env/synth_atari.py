"""Device-resident synthetic Atari-shaped pixel env (BASELINE.json config 4): observations (N,4,84,84) uint8,
6 discrete actions.  Same vec-env API as SynthVecEnv; the game is defined in oracle/synth_atari.py (the
reference only wraps real ALE games, /root/reference/torchrl/env/atari_wrapper.py) and implemented in
csrc/atari_env.cu, bit-exact against the oracle (integer arithmetic).  Frames stay uint8 end to end
(env -> replay ring -> gather); `obs_scale` = 1/255 is applied when a batch is fed to the network
(ScaledFloatFrame, atari_wrapper.py:171-180)."""
import copy

import numpy as np
import torch

from .. import ops
from ..spaces import Box, Discrete

F32, U8, I32 = torch.float32, torch.uint8, torch.int32
ENV_ID = "SynthAtari-v0"
MAX_EPISODE_STEPS = 1000


class SynthAtariVecEnv:
    obs_dtype = torch.uint8
    obs_scale = 1.0 / 255.0
    pixel = True
    lockstep = False
    obs_norm = False
    _obs_normalizer = None

    def __init__(self, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None,
                 max_episode_steps=MAX_EPISODE_STEPS):
        self.env_id = ENV_ID
        self.env_nums = int(env_nums)
        self.device = torch.device(device)
        self.first_env = int(first_env)
        self.total_envs = int(total_envs) if total_envs is not None else self.env_nums
        self._max_episode_steps = int(max_episode_steps)
        self._reward_scale = 1
        self.training = True
        self.observation_space = Box(0, 255, (4, 84, 84), dtype=np.uint8)
        self.action_space = Discrete(6)
        N, dev = self.env_nums, self.device
        self.obs = torch.zeros(N, 4, 84, 84, dtype=U8, device=dev)        # current frame stack (in place)
        self.latent = torch.zeros(N, 5, dtype=I32, device=dev)
        self.elapsed = torch.zeros(N, dtype=I32, device=dev)
        self.episode = torch.zeros(N, dtype=I32, device=dev)
        self.seeds = torch.zeros(N, dtype=I32, device=dev)
        self.reward = torch.zeros(N, dtype=F32, device=dev)
        self.done = torch.zeros(N, dtype=U8, device=dev)
        self.time_limit = torch.zeros(N, dtype=U8, device=dev)
        self._host_mirror_ok = False
        self.dist = None
        self.seed(0)

    def train(self):
        self.training = True

    def eval(self):
        self.training = False

    def close(self):
        pass

    def seed(self, seed):
        ops.synth_env_seed(self.seeds, self.episode, seed, self.total_envs, self.first_env)

    def _reset(self, mask=None, zero_is_mask=None, episode_bias=0, bump=1):
        ops.synth_atari_reset(self.obs, self.latent, self.elapsed, self.episode, self.seeds, mask, zero_is_mask,
                              episode_bias, bump)

    def reset(self, **kwargs):
        self._reset()
        return self.obs

    def partial_reset(self, index_mask, **kwargs):
        mask = torch.as_tensor(index_mask, device=self.device).reshape(-1).to(U8).contiguous()
        self._reset(mask=mask)
        return self.obs

    def launch_step(self, actions):
        """actions: (N,) or (N,1) float tensor holding the action index.  Updates obs in place."""
        ops.synth_atari_step(self.obs, self.latent, actions, self.elapsed, self.reward, self.done, self.time_limit,
                             self._max_episode_steps)
        return self.obs

    def step(self, actions):
        act = torch.as_tensor(actions, device=self.device).reshape(-1).to(F32).contiguous()
        self.launch_step(act)
        return self.obs, self.reward.unsqueeze(-1), self.done.bool().unsqueeze(-1), {"time_limit": self.time_limit.bool()}

    def to_float(self, obs_u8, out=None):
        """uint8 frames -> float32 in [0,1] (one launch)."""
        return ops.u8_to_f32(obs_u8, self.obs_scale, out)

    def __deepcopy__(self, memo):
        new = SynthAtariVecEnv.__new__(SynthAtariVecEnv)
        for k, v in self.__dict__.items():
            new.__dict__[k] = v.clone() if torch.is_tensor(v) else copy.deepcopy(v, memo)
        return new
