"""Epoch loop shared by every agent (API of /root/reference/torchrl/algo/rl_algo.py:14-190)."""
import copy
import os.path as osp
import pathlib
import pickle
import time
from collections import deque

import numpy as np
import torch
import torch.optim as optim

from ..flat import FlatAdam, FlatParams
from ..spaces import is_box
from .. import ops


class _LRGroup(dict):
    """param_group stand-in: assigning ['lr'] forwards to the flat optimizer's device scalar."""

    def __init__(self, owner, seg, lr):
        super().__init__(lr=lr)
        self._owner, self._seg = owner, seg

    def __setitem__(self, k, v):
        super().__setitem__(k, v)
        if k == "lr":
            self._owner.set_lr(self._seg, v)


class SegmentOptimizer:
    """What `agent.pf_optimizer` etc. return: one segment of the agent's FlatAdam, exposing the
    `param_groups[...]['lr']` knob that update_linear_schedule uses."""

    def __init__(self, flat, seg):
        self.flat, self.seg = flat, seg
        self.param_groups = [_LRGroup(flat, seg, flat.initial_lrs[seg])]

    def zero_grad(self):
        self.flat.grad[self.flat.seg_begin[self.seg]:self.flat.seg_begin[self.seg + 1]].zero_()

    def step(self):
        self.flat.step(active_mask=1 << self.seg)


class _Stopwatch:
    """Accumulates wall time per phase between two epoch reports."""

    def __init__(self):
        self.spent = {}

    def add(self, phase, seconds):
        self.spent[phase] = self.spent.get(phase, 0.0) + seconds

    def take(self, phase):
        return self.spent.pop(phase, 0)


class RLAlgo:
    """Owns the epoch loop: collect -> update -> (every eval_interval) evaluate + report -> (every save_interval)
    snapshot.  Subclasses provide `update_per_epoch`, declare their networks through `_init_networks` and optionally
    provide pretrain / start_epoch / finish_epoch hooks."""
    _nets = _targets = ()           # names of the networks and of those with a target: see _init_networks

    def __init__(self, env=None, replay_buffer=None, collector=None, logger=None, grad_clip=None, discount=0.99,
                 num_epochs=3000, batch_size=128, device='cpu', save_interval=100, eval_interval=1, save_dir=None,
                 use_cuda_graph=True, dist=None, resume_checkpoints=False):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("torchrl_b200 agents run on a CUDA device (there is no CPU path); got %r" % (device,))
        self._init_bookkeeping(env, replay_buffer, collector, logger, grad_clip, discount, num_epochs, batch_size,
                               save_interval, eval_interval, save_dir)
        self.use_cuda_graph = bool(use_cuda_graph)
        self.dist = dist                    # None or a torchrl_b200.distributed.DataParallelContext
        self.resume_checkpoints = bool(resume_checkpoints)

    def _init_bookkeeping(self, env, replay_buffer, collector, logger, grad_clip, discount, num_epochs, batch_size,
                          save_interval, eval_interval, save_dir):
        """Everything the epoch loop needs that does not touch the device."""
        self.env, self.replay_buffer, self.collector, self.logger = env, replay_buffer, collector, logger
        self.continuous = is_box(env.action_space)
        self.discount, self.grad_clip = discount, grad_clip
        self.num_epochs, self.batch_size = num_epochs, batch_size
        self.epoch_frames = collector.epoch_frames
        self.training_update_num = 0
        self.sample_key = None
        self.episode_rewards = deque(maxlen=30)              # evaluation returns (running average)
        self.training_episode_rewards = deque(maxlen=30)     # finished training episodes
        self.save_interval, self.eval_interval = save_interval, eval_interval
        self.save_dir = save_dir
        if save_dir is not None:
            pathlib.Path(save_dir).mkdir(parents=True, exist_ok=True)
        self.best_eval = None
        self._watch = _Stopwatch()
        self.start = time.time()
        self.current_epoch = 0
        self.first_epoch = 0                # load_checkpoint moves it past the last finished epoch
        self.use_cuda_graph = True
        self.dist = None
        self.resume_checkpoints = False

    # the two phase timers of the reference, kept as attributes for code that reads them
    @property
    def explore_time(self):
        return self._watch.spent.get("explore", 0)

    @property
    def train_time(self):
        return self._watch.spent.get("train", 0)

    # ------------------------------------------------------------------ resume (absent in the reference)
    def save_checkpoint(self, path):
        """Full training state (weights, Adam moments, targets, collector / env / normaliser state, replay
        ring, every RNG stream): see utils/checkpoint.py."""
        from ..utils.checkpoint import save_checkpoint
        return save_checkpoint(self, path)

    def load_checkpoint(self, path):
        """Restore a `save_checkpoint` file in place; `train()` then continues with the next epoch."""
        from ..utils.checkpoint import load_checkpoint
        self.first_epoch = load_checkpoint(self, path) + 1
        return self.first_epoch

    # ------------------------------------------------------------------ hooks
    def start_epoch(self):
        pass

    def finish_epoch(self):
        return {}

    def pretrain(self):
        pass

    def update_per_epoch(self):
        pass

    def _device_sync(self):
        torch.cuda.synchronize(self.device)

    # ------------------------------------------------------------------ snapshots
    def snapshot(self, prefix, epoch):
        """model_{name}_{epoch}.pth state_dicts + pickled obs normaliser (rl_algo.py:83-94)."""
        if prefix is None:
            return
        normalizer = getattr(self.env, "_obs_normalizer", None)
        if normalizer is not None:
            with open(osp.join(prefix, "_obs_normalizer_{}.pkl".format(epoch)), "wb") as f:
                pickle.dump(normalizer, f)
        for name, network in self.snapshot_networks:
            torch.save(network.state_dict(), osp.join(prefix, "model_{}_{}.pth".format(name, epoch)))

    # ------------------------------------------------------------------ the loop
    def _collect_and_update(self):
        """One epoch of data + learning; returns the collector's summary."""
        t0 = time.time()
        summary = self.collector.train_one_epoch()
        self.training_episode_rewards.extend(summary["train_rewards"])
        t1 = time.time()
        self._watch.add("explore", t1 - t0)
        self.update_per_epoch()
        self._device_sync()
        self._watch.add("train", time.time() - t1)
        return summary

    def _evaluate_and_report(self, epoch, total_frames, summary, extra):
        """Evaluation episodes, best-model snapshot and the epoch row of the log (rl_algo.py:125-157)."""
        t0 = time.time()
        evals = self.collector.eval_one_epoch()
        eval_time = time.time() - t0
        returns = evals.pop("eval_rewards")
        self.episode_rewards.extend(returns)
        score = np.mean(returns)
        if self.best_eval is None or score > self.best_eval:
            self.best_eval = score
            self.snapshot(self.save_dir, 'best')
        trained = self.training_episode_rewards
        row = {
            "Running_Average_Rewards": np.mean(self.episode_rewards),
            "Train_Epoch_Reward": summary["train_epoch_reward"],
            "Running_Training_Average_Rewards": np.mean(trained) if len(trained) else float("nan"),
            "Explore_Time": self._watch.take("explore"),
            "Train___Time": self._watch.take("train"),
            "Eval____Time": eval_time,
        }
        row.update(evals)
        row.update(extra)
        self.logger.add_epoch_info(epoch, total_frames, time.time() - self.start, row)
        self.start = time.time()

    def train(self):
        if self.first_epoch == 0:
            self.pretrain()
            total_frames = getattr(self, "pretrain_frames", 0)
        else:
            # resumed through load_checkpoint: the pretraining data is already in the restored ring and the
            # frame count continues where the interrupted run stopped
            total_frames = getattr(self, "total_frames",
                                   getattr(self, "pretrain_frames", 0) + self.first_epoch * self.epoch_frames)
        self.start_epoch()
        for epoch in range(self.first_epoch, self.num_epochs):
            self.current_epoch = epoch
            self.start_epoch()
            summary = self._collect_and_update()
            extra = self.finish_epoch()
            total_frames += self.epoch_frames
            self.total_frames = total_frames
            if epoch % self.eval_interval == 0:
                self._evaluate_and_report(epoch, total_frames, summary, extra)
            if epoch % self.save_interval == 0:
                self.snapshot(self.save_dir, epoch)
                if self.resume_checkpoints and self.save_dir is not None:
                    self.save_checkpoint(osp.join(self.save_dir, "checkpoint_latest.pt"))
        self.snapshot(self.save_dir, "finish")
        self.collector.terminate()
        self.logger.finish()

    def update(self, batch):
        raise NotImplementedError

    def _record_infos(self, infos):
        """Keep the epoch's per-update info dicts and hand them to the logger."""
        self._last_infos = infos
        if self.logger is not None:
            for info in infos:
                self.logger.add_update_info(info)

    # ------------------------------------------------------------------ networks, the fused optimizer, target networks
    def _init_networks(self, optimizer_class, segments, eps, max_norms, targets=()):
        """The agent's networks, declared once.  `segments`: [(name or None, module or parameter list, lr)] in
        flat-buffer order, with one max grad norm per segment (0: no clipping); `targets`: the names of the segments
        whose network has a target network.  In this order: self.target_<name> = a copy of each such network (before
        anything moves the online weights), the networks move to the device, self.opt = one FlatAdam over the segments
        (a named segment gets the reference's handle `self.<name>_optimizer`), and self._target_flat = one flat buffer
        over the targets.  Returns {name: segment index}.

        Polyak averaging and hard copies read the online networks as one slice of the optimizer's buffer, so the
        segments with a target must be contiguous."""
        if optimizer_class is not optim.Adam:
            raise NotImplementedError("torchrl_b200 fuses clip + Adam in CUDA; only optim.Adam is supported "
                                      "(DESIGN.md section 6, deviation 10)")
        index = {name: i for i, (name, _, _) in enumerate(segments) if name is not None}
        self._nets = [name for name, net, _ in segments if name is not None and isinstance(net, torch.nn.Module)]
        self._targets = [name for name in self._nets if name in targets]
        assert len(self._targets) == len(targets), "a network with a target must be a named optimizer segment"
        for name in self._targets:
            setattr(self, "target_" + name, copy.deepcopy(getattr(self, name)))
        self.to(self.device)
        self.opt = FlatAdam([params for _, params, _ in segments], lrs=[lr for _, _, lr in segments], eps=eps,
                            max_norms=max_norms, device=self.device, dist=self.dist)
        for name, i in index.items():
            setattr(self, name + "_optimizer", SegmentOptimizer(self.opt, i))
        if self._targets:
            segs = [index[name] for name in self._targets]
            assert segs[-1] - segs[0] == len(segs) - 1, "the networks with a target must be contiguous segments"
            self._target_segs = (segs[0], segs[-1] + 1)
            self._target_flat = FlatParams([target for _, target in self.target_networks], device=self.device)
        return index

    @property
    def networks(self):
        """What a checkpoint saves, in its order: the named networks in segment order, then their targets."""
        return [getattr(self, name) for name in self._nets] + [target for _, target in self.target_networks]

    @property
    def target_networks(self):
        return [(getattr(self, name), getattr(self, "target_" + name)) for name in self._targets]

    @property
    def snapshot_networks(self):
        return [(name, getattr(self, name)) for name in self._nets]

    def _optimizer_step(self, active_mask=None):
        """Clip + Adam over the segments in `active_mask` (None: all).  Data parallel (every rank draws the same rows
        from the same host seed): the flat gradient is summed over ranks first and scaled by 1/G inside the Adam
        kernel, before clipping -- what a single process over all envs would apply.  Returns that scale."""
        scale, reduced = self.dist.reduce_grads(self.opt, active_mask) if self.dist is not None else (1.0, False)
        self.opt.step(active_mask=active_mask, grad_scale=scale, reduced=reduced)
        return scale

    def _update_target_networks(self):
        """Polyak update of the target nets (rl_algo.py:169-172) on the flat buffers: one launch,
        captured inside the update graph.  The periodic HARD copy (rl_algo.py:173-176) depends on a
        host counter, so it is applied by `_maybe_hard_update` outside of any captured graph."""
        if self.use_soft_update:
            ops.polyak_update(self._target_flat.data, self.opt.seg_slice(*self._target_segs), self.tau,
                              planes=(self._target_flat.hi, self._target_flat.lo))

    def _maybe_hard_update(self):
        if not self.use_soft_update and self.training_update_num % self.target_hard_update_period == 0:
            self._hard_update_targets()

    def _hard_update_targets(self):
        """Targets <- online networks (copy_model_params_from_to on the flat buffers)."""
        self._target_flat.copy_from(self.opt.seg_slice(*self._target_segs))

    def to(self, device):
        for net in self.networks:
            net.to(device)
