"""Frame-de-duplicated replay ring for frame-stacked pixel observations (API of
/root/reference/torchrl/replay_buffers/memory_efficient_replay_buffer.py:5-33).

The reference avoids storing the C-1 shared frames of consecutive observations by keeping LazyFrames objects (lists of
references to the env's frame arrays, /root/reference/torchrl/env/atari_wrapper.py:142-168) in Python lists.  On the
device the same saving is a data layout (csrc/frames.cu): per time row and env the ring holds only the NEWEST frame of
`obs`, the newest frame of `next_obs` and an age byte (2 of the 2C stored frames: 4x less HBM at C = 4);
`gather_rows` rebuilds both stacks for the sampled rows -- exactly, including the rows whose older frames the ring has
already overwritten (a C-1 deep history of overwritten frames) -- and hands them out as float32 scaled by `obs_scale`
(ScaledFloatFrame fused into the gather).  Sampling is BaseReplayBuffer's (np.random.randint row indices, bit-exact).
"""
import torch

from .. import ops
from .base import BaseReplayBuffer

U8, I32, F32 = torch.uint8, torch.int32, torch.float32


class MemoryEfficientReplayBuffer(BaseReplayBuffer):
    frame_dedup = True

    def __init__(self, max_replay_buffer_size, env_nums=1, time_limit_filter=False, device=None, obs_scale=1.0 / 255.0):
        super().__init__(max_replay_buffer_size, env_nums, time_limit_filter, device)
        self.obs_scale = float(obs_scale)
        self._stack = None                   # (C, H, W) of one observation
        self._stack_cache = {}

    # ------------------------------------------------------------------ storage
    def allocate_frames(self, stack_shape):
        """Create the de-duplicated storage for observations of shape (C, H, W)."""
        self._ensure_device()
        C = int(stack_shape[0])
        F = 1
        for d in stack_shape[1:]:
            F *= int(d)
        assert C >= 2 and F % 16 == 0, "frame stacks need C >= 2 frames of a multiple of 16 bytes"
        T, N, dev = self._max_replay_buffer_size, self.env_nums, self.device
        self._stack, self._C, self._F = tuple(int(d) for d in stack_shape), C, F
        self._obs = torch.zeros(T, N, F, dtype=U8, device=dev)           # newest frame of obs
        self._next_obs = torch.zeros(T, N, F, dtype=U8, device=dev)      # newest frame of next_obs
        self._age = torch.zeros(T, N, dtype=U8, device=dev)
        self._hist = torch.zeros(C - 1, N, F, dtype=U8, device=dev)
        self._hist_count = torch.zeros(1, dtype=I32, device=dev)
        for k in ("obs", "next_obs"):
            if k not in self._keys:
                self._keys.append(k)

    def write_obs(self, stack_u8, elapsed):
        """Collector step, before env.step: newest frame of the (N, C, H, W) stack -> row `_top` (+ age, history)."""
        ops.frame_ring_write(stack_u8, self._obs, self._top_dev, age=self._age, elapsed=elapsed, hist=self._hist,
                             hist_count=self._hist_count, size=self._size_dev)
        ops.frame_hist_advance(self._hist_count, self._size_dev, self._max_replay_buffer_size)

    def write_next_obs(self, stack_u8):
        """Collector step, after env.step: newest frame of the new stack -> row `_top`."""
        ops.frame_ring_write(stack_u8, self._next_obs, self._top_dev)

    def add_sample(self, sample_dict, episode_steps=None, **kwargs):
        """Reference-style row insertion with full (N, C, H, W) uint8 stacks under "obs" / "next_obs".
        `episode_steps` (N,) int32: steps since each env's episode began when `obs` was observed (how many of the
        older frames in `obs` are real history rather than repeats of the first frame); default C-1 (mid-episode)."""
        obs, nxt = sample_dict["obs"], sample_dict["next_obs"]
        self._ensure_device(obs if torch.is_tensor(obs) else None)
        obs = torch.as_tensor(obs, device=self.device).to(U8).contiguous()
        nxt = torch.as_tensor(nxt, device=self.device).to(U8).contiguous()
        if self._stack is None:
            self.allocate_frames(tuple(obs.shape[1:]))
        if episode_steps is None:
            episode_steps = torch.full((self.env_nums,), self._C - 1, dtype=I32, device=self.device)
        self.write_obs(obs, torch.as_tensor(episode_steps, device=self.device).to(I32).contiguous())
        self.write_next_obs(nxt)
        rest = {k: v for k, v in sample_dict.items() if k not in ("obs", "next_obs")}
        if rest:
            super().add_sample(rest, **kwargs)          # writes its keys at `_top` and advances
        else:
            ops.counter_advance(None, self._top_dev, self._max_replay_buffer_size, self._size_dev)
            self._advance()

    # ------------------------------------------------------------------ sampling
    def gather_rows(self, indices, sample_key, pos_ptr=None, rows=None):
        rows = int(indices.numel()) if rows is None else int(rows)
        frame_keys = [k for k in sample_key if k in ("obs", "next_obs")]
        other = [k for k in sample_key if k not in ("obs", "next_obs")]
        out = super().gather_rows(indices, other, pos_ptr=pos_ptr, rows=rows) if other else {}
        if frame_keys:
            bufs = self._stack_cache.get(rows)
            if bufs is None:
                shape = (rows * self.env_nums,) + self._stack
                bufs = self._stack_cache[rows] = (torch.empty(shape, dtype=F32, device=self.device),
                                                  torch.empty(shape, dtype=F32, device=self.device))
            ops.frame_stack_gather(self._obs, self._next_obs, self._age, self._hist, self._hist_count, indices, rows,
                                   self._top_dev, self._size_dev, self.obs_scale, bufs[0], bufs[1], pos=pos_ptr)
            if "obs" in frame_keys:
                out["obs"] = bufs[0]
            if "next_obs" in frame_keys:
                out["next_obs"] = bufs[1]
        return out

    def stored_frame_bytes(self):
        """HBM held by the pixel storage (2 frames + 1 byte per (row, env); a full-stack ring holds 2 C frames)."""
        return self._obs.numel() + self._next_obs.numel() + self._age.numel() + self._hist.numel()
