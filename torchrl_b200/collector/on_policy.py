"""On-policy collectors (API of /root/reference/torchrl/collector/on_policy.py:8-155): adds the
value net, stores V(obs) per step and bootstraps rewards of envs cut by `max_episode_frames`.

`VecOnPolicyCollector(vf, env=<pixel env>, ...)` -- the reference's Atari examples construct it directly -- yields a
PixelVecOnPolicyCollector: uint8 frame stacks from the env to the rollout buffer (collector/pixel.py)."""
from .base import VecCollector
from .pixel import PixelVecCollector


class VecOnPolicyCollector(VecCollector):
    on_policy = True

    def __new__(cls, *args, **kwargs):
        if cls is VecOnPolicyCollector and getattr(kwargs.get("env"), "pixel", False):
            cls = PixelVecOnPolicyCollector
        return super().__new__(cls)

    def __init__(self, vf, discount=0.99, **kwargs):
        self.vf = vf
        self.discount = discount
        super().__init__(**kwargs)

    @property
    def funcs(self):
        return {"pf": self.pf, "vf": self.vf}


class PixelVecOnPolicyCollector(VecOnPolicyCollector, PixelVecCollector):
    """On-policy rollouts of a uint8 pixel env: `_obs` / `_next_obs` are (T, N, C, H, W) uint8, `_acts` (T, N)."""
    on_policy = True


OnPolicyCollectorBase = VecOnPolicyCollector
