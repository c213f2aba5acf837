"""Prioritised replay over time rows (BASELINE.json config 4).

PARITY UNPINNED: the reference ships no prioritised replay (SURVEY.md fact 7).  This class extends
BaseReplayBuffer (/root/reference/torchrl/replay_buffers/base.py:4-54 API) with proportional
prioritisation at the buffer's own sampling granularity -- the time row: `random_batch` draws
`batch_size // env_nums` rows with probability proportional to the row priority and additionally returns
`weights` (importance weights, one per sample) and `indices` (row ids) for `update_priorities`.
Uniform numbers come from np.random.rand on the host (global legacy RNG, like the reference's
np.random.randint), so the sampled indices are reproducible against the NumPy oracle
(oracle/ref_numpy.per_sample).  Every draw goes through the two-pass sampler (csrc/prioritized.cu:
trl_per_sample_rows), which serves rings of up to 2^24 rows and reads the live size and the draw position on the
device, so the agents' captured update graphs sample too.
"""
import numpy as np
import torch

from .. import ops
from .base import BaseReplayBuffer


class PrioritizedReplayBuffer(BaseReplayBuffer):
    def __init__(self, max_replay_buffer_size, env_nums=1, time_limit_filter=False, device=None, alpha=0.6,
                 beta=0.4, eps=1e-6):
        super().__init__(max_replay_buffer_size, env_nums, time_limit_filter, device)
        if not 1 <= self._max_replay_buffer_size <= ops.PER_MAX_ROWS:
            raise ValueError("a prioritised ring holds 1..%d time rows; %d transitions over %d envs make %d"
                             % (ops.PER_MAX_ROWS, int(max_replay_buffer_size), env_nums, self._max_replay_buffer_size))
        self.alpha, self.beta, self.eps = alpha, beta, eps
        self._priorities = None
        self._max_prio = None
        self._last_idx = None
        self._sampler = None     # the sampler's scratch and device scalars: working memory, not checkpointed

    def _ensure_prio(self):
        self._ensure_device()
        if self._priorities is None:
            self._priorities = torch.zeros(self._max_replay_buffer_size, dtype=torch.float32, device=self.device)
            self._max_prio = torch.ones(1, dtype=torch.float32, device=self.device)
        if self._sampler is None:
            dev = self.device
            self._sampler = {
                "scratch": torch.empty(ops.per_scratch_doubles(self._max_replay_buffer_size), dtype=torch.float64,
                                       device=dev),
                "size": torch.zeros(1, dtype=torch.int32, device=dev),
                "pos": torch.zeros(1, dtype=torch.int32, device=dev),
            }

    def add_sample(self, sample_dict, **kwargs):
        self._ensure_device(next(iter(sample_dict.values())))
        self._ensure_prio()
        ops.per_insert(self._priorities, self._top_dev, self._max_prio)     # new rows get the max priority
        super().add_sample(sample_dict, **kwargs)

    def mark_inserted(self):
        """For collectors that write rows themselves: give the row at `_top` the running max priority."""
        self._ensure_prio()
        ops.per_insert(self._priorities, self._top_dev, self._max_prio)

    def random_batch(self, batch_size, sample_key):
        assert batch_size % self.env_nums == 0, "batch size should be dividable by env_nums"
        b = batch_size // self.env_nums
        self._ensure_prio()
        u = torch.from_numpy(np.random.rand(b)).to(self.device, non_blocking=True)
        self._sampler["size"].fill_(self.num_steps_can_sample())
        idx = torch.empty(b, dtype=torch.int64, device=self.device)
        w = torch.empty(b, dtype=torch.float32, device=self.device)
        self.sample_rows(u, self._sampler["pos"], self._sampler["size"], idx, w)
        out = self.gather_rows(idx, sample_key)
        out["weights"] = w.repeat_interleave(self.env_nums).unsqueeze(-1)
        out["indices"] = idx
        self._last_idx = idx
        return out

    def sample_rows(self, u, pos_ptr, size_ptr, idx, weights):
        """Draw idx.numel() rows (idx, weights) from the first *size_ptr rows with the uniforms u[*pos_ptr * b:][:b];
        all device-side, so the call can be captured in a CUDA graph."""
        self._ensure_prio()
        return ops.per_sample_rows(self._priorities, size_ptr, u, pos_ptr, idx.numel(), self.beta,
                                   self._sampler["scratch"], idx, weights)

    def update_priorities(self, indices, td_errors):
        """td_errors: (b*N,) or (b*N, critics) per-sample TD errors of the batch drawn with `indices`.  The new
        priority of a row is (mean of |TD| over its N transitions and the critics + eps)^alpha."""
        td = td_errors.reshape(indices.numel(), -1).contiguous().float()
        ops.per_update(self._priorities, indices, td, self.alpha, self.eps, self._max_prio)
