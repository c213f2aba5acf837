"""Off-policy base: uniform row sampling + opt_times updates per epoch, target networks
(API of /root/reference/torchrl/algo/off_policy/off_rl_algo.py:8-84).

Device form of `update_per_epoch`: the row indices of ALL opt_times minibatches are drawn up-front
with the reference's own np.random.randint calls (same global RNG stream, bit-exact indices),
uploaded once, and one captured CUDA graph of {gather, update} is replayed opt_times times reading
its position from a device counter.  Logged scalars accumulate in a device log and are fetched
once per epoch (the reference syncs ~20 times per update).

Prioritised replay (no reference counterpart) has the same structure: the uniforms of ALL opt_times draws come from
one np.random.rand(opt_times * b) (the stream of opt_times calls of rand(b)) and are uploaded once; each update
{draw rows by priority at the device position, gather, weighted update, write the rows' new priorities, log row} is
one captured graph per variant.  Only the critics' TD losses are importance weighted (DESIGN.md deviation 24).
"""
import time

import numpy as np
import torch

from ... import ops
from ...networks import fused
from ..rl_algo import RLAlgo


class OffRLAlgo(RLAlgo):
    INFO_SLOTS = 64
    TD_COLUMNS = 1               # critics whose |TD| per sample the loss writes for the new priorities

    def __init__(self, pretrain_epochs=0, min_pool=0, target_hard_update_period=1000, use_soft_update=True,
                 tau=0.001, opt_times=1, **kwargs):
        super().__init__(**kwargs)
        self.pretrain_epochs = pretrain_epochs
        self.target_hard_update_period = target_hard_update_period
        self.use_soft_update = use_soft_update
        self.tau = tau
        self.opt_times = opt_times
        self.min_pool = min_pool
        self.sample_key = ["obs", "next_obs", "acts", "rewards", "terminals"]
        self._ub = None              # update-loop state (buffers, graphs)
        self._graphs = {}
        self._eager_runs = {}
        self._last_infos = []
        self._td = None              # prioritised replay: (B, TD_COLUMNS) |TD| of the last update, inside self._ub

    # ------------------------------------------------------------------ device update loop
    def _ub_setup(self):
        rb = self.replay_buffer
        N = rb.env_nums
        assert self.batch_size % N == 0, "batch size should be dividable by env_nums"
        b = self.batch_size // N
        dev = self.device
        U = max(int(self.opt_times), 1)
        self._ub = {
            "b": b, "B": b * N, "U": U,
            "idx": torch.zeros(U * b, dtype=torch.int64, device=dev),
            "idx_host": torch.zeros(U * b, dtype=torch.int64).pin_memory(),
            "upd": torch.zeros(1, dtype=torch.int32, device=dev),
            "log_ticket": torch.zeros(1, dtype=torch.int32, device=dev),
            "info": torch.zeros(1, self.INFO_SLOTS, dtype=torch.float32, device=dev),
            "log32": torch.zeros(U, self.INFO_SLOTS, dtype=torch.float32, device=dev),
            "scratch": ops.OffPolicyScratch(b * N, dev),
        }
        self._ub["log_plan"] = ops.RowCopyPlan([self._ub["info"]], [self._ub["log32"]], [self.INFO_SLOTS * 4])
        ub = self._ub
        ub["per"] = hasattr(rb, "update_priorities")
        if ub["per"]:
            ub.update({
                "u": torch.zeros(U * b, dtype=torch.float64, device=dev),
                "u_host": torch.zeros(U * b, dtype=torch.float64).pin_memory(),
                "size": torch.zeros(1, dtype=torch.int32, device=dev),
                "rows": torch.zeros(b, dtype=torch.int64, device=dev),
                "w": torch.zeros(b, dtype=torch.float32, device=dev),
                "w_samples": torch.zeros(b * N, 1, dtype=torch.float32, device=dev),
                "td": torch.zeros((b * N,) if self.TD_COLUMNS == 1 else (b * N, self.TD_COLUMNS), dtype=torch.float32,
                                  device=dev),
            })
            self._td = ub["td"]
        return ub

    def _gather(self):
        ub = self._ub
        rb = self.replay_buffer
        if not ub["per"]:
            return rb.gather_rows(ub["idx"], self.sample_key, pos_ptr=ub["upd"], rows=ub["b"])
        rb.sample_rows(ub["u"], ub["upd"], ub["size"], ub["rows"], ub["w"])
        batch = dict(rb.gather_rows(ub["rows"], self.sample_key))
        ub["w_samples"].view(ub["b"], -1).copy_(ub["w"].view(-1, 1).expand(ub["b"], rb.env_nums))
        batch["weights"] = ub["w_samples"]
        return batch

    def _critic_loss(self, batch, q1, q2, y, info):
        """MSE of one or two critics against y: importance weighted when the batch carries prioritised-replay
        weights, with the unweighted |q - y| of drawn rows into self._td for their new priorities."""
        sc = self._ub["scratch"]
        weights = batch.get("weights")
        if weights is None:
            return ops.twin_mse_loss(q1, q2, y, sc, info=info)
        td = self._td if self._explicit_batch is None else None
        return ops.twin_mse_loss_weighted(q1, q2, y, weights.reshape(-1), sc, info=info, td_out=td)

    def _finish_update(self):
        """New priorities of the drawn rows (prioritised replay), log row of a gathered update, then upd += 1 (an
        explicit batch's info row is read directly)."""
        if self._explicit_batch is not None:
            return
        ub = self._ub
        if ub["per"]:
            self.replay_buffer.update_priorities(ub["rows"], self._td)
        ops.ring_write_advance(ub["log_plan"], ub["upd"], ub["U"], ub["log_ticket"])     # log row, then upd += 1

    def _variant(self):
        """Key of the update-graph variant for the current update (e.g. TD3's delayed actor step)."""
        return 0

    # ------------------------------------------------------------------ data parallel (SURVEY.md 8(e))
    @property
    def _dp(self):
        return self.dist is not None and self.dist.active

    def _all_ranks(self, vec):
        """Concatenation of a per-rank (B,) vector over ranks (rank order), identical on every rank."""
        if not self._dp:
            return vec
        import torch.distributed as tdist
        out = torch.empty(vec.numel() * self.dist.world_size, dtype=vec.dtype, device=vec.device)
        tdist.all_gather_into_tensor(out, vec.contiguous())
        return out

    def _update_body(self, variant):
        raise NotImplementedError

    def _decode_info(self, row, variant):
        raise NotImplementedError

    def _run_update(self):
        self.training_update_num += 1
        v = self._variant()
        if not self.use_cuda_graph:
            self._update_body(v)
        elif v in self._graphs:
            self._graphs[v].replay()
        elif self._eager_runs.get(v, 0) < 3:
            self._eager_runs[v] = self._eager_runs.get(v, 0) + 1
            self._update_body(v)
        else:
            g = ops.CapturedGraph(lambda: self._update_body(v))
            self._graphs[v] = g
            g.replay()
        self._maybe_hard_update()
        return v

    @fused.presplit_scope
    def update_per_epoch(self, flush_infos=True):
        """opt_times x {random_batch; update} (off_rl_algo.py:46-51)."""
        ub = self._ub or self._ub_setup()
        size = self.replay_buffer.num_steps_can_sample()
        staged = ub.get("staged")
        if staged is not None:
            staged.synchronize()          # the last epoch's upload has left the pinned buffer we are about to refill
        if ub["per"]:
            # the uniforms of every draw at once: rand(U * b) is the stream of U calls of rand(b)
            ub["u_host"].copy_(torch.from_numpy(np.random.rand(ub["U"] * ub["b"])))
            ub["u"].copy_(ub["u_host"], non_blocking=True)
            ub["size"].fill_(size)
        else:
            for u in range(ub["U"]):
                idx = np.random.randint(0, size, ub["b"])           # one draw per update, like random_batch
                ub["idx_host"][u * ub["b"]:(u + 1) * ub["b"]].copy_(torch.from_numpy(idx.astype(np.int64)))
            ub["idx"].copy_(ub["idx_host"], non_blocking=True)
        ub["staged"] = torch.cuda.Event()
        ub["staged"].record()
        ub["upd"].zero_()
        variants = [self._run_update() for _ in range(ub["U"])]
        if flush_infos:
            log = ub["log32"][:len(variants)].cpu().numpy()
            self._record_infos([self._decode_info(log[u], variants[u]) for u in range(len(variants))])

    @fused.presplit_scope
    def update(self, batch):
        """Eager single update on an explicit batch dict (reference signature); syncs to return floats."""
        dev = self.device
        ub = self._ub or self._ub_setup()
        conv = {}
        for k in self.sample_key + (["weights"] if "weights" in batch else []):   # weights: prioritised replay
            v = batch[k]
            v = torch.as_tensor(np.asarray(v)) if not torch.is_tensor(v) else v
            dt = torch.uint8 if k in ("terminals", "masks") else torch.float32   # masks: Bootstrapped DQN
            conv[k] = v.to(device=dev, dtype=dt).contiguous()
        variant = self._explicit_update(conv)
        ub["upd"].zero_()
        return self._decode_info(ub["info"][0].cpu().numpy(), variant)

    _explicit_batch = None

    def _explicit_update(self, batch):
        """One eager update on a batch dict of device tensors instead of the gathered rows; returns its variant."""
        self.training_update_num += 1
        variant = self._variant()
        self._explicit_batch = batch
        try:
            self._update_body(variant)
            self._maybe_hard_update()
        finally:
            self._explicit_batch = None
        return variant

    def _batch(self):
        return self._explicit_batch if self._explicit_batch is not None else self._gather()

    # ------------------------------------------------------------------ pieces of the continuous-control updates
    def _transitions(self):
        """The update's batch and its transition fields: obs, acts as (B, -1), next_obs, flat rewards and terminals."""
        batch = self._batch()
        obs, acts, next_obs = batch["obs"], batch["acts"], batch["next_obs"]
        rewards, terminals = batch["rewards"].reshape(-1), batch["terminals"].reshape(-1)
        return batch, obs, acts.reshape(obs.shape[0], -1), next_obs, rewards, terminals

    def _deterministic_policy_step(self, qf, obs, info):
        """DDPG's and TD3's policy loss -mean qf(s, pf(s)): its value into info[6], its gradient into the policy
        segment.  Returns the new actions."""
        new_actions = self.pf(obs)
        q_new = qf([obs, new_actions])
        info[6:7].copy_((-q_new.detach().mean()).reshape(1))
        seed = torch.full_like(q_new, -1.0 / q_new.numel())
        torch.autograd.backward([q_new], [seed], inputs=self.opt.segments[0])
        return new_actions

    def _critic_backward(self, preds, grads, first, last):
        """Backward from the critics' predictions, seeded with the loss kernel's gradients, into the critic segments
        first .. last - 1."""
        torch.autograd.backward(preds, [g.reshape(q.shape) for g, q in zip(grads, preds)],
                                inputs=[p for seg in self.opt.segments[first:last] for p in seg])

    def update_per_timestep(self):
        if self.replay_buffer.num_steps_can_sample() > max(self.min_pool, self.batch_size):
            self.update_per_epoch()

    def pretrain(self):
        """pretrain_epochs of collection with the learning policy, no updates (off_rl_algo.py:53-84)."""
        total_frames = 0
        self.pretrain_frames = self.pretrain_epochs * self.epoch_frames
        for pretrain_epoch in range(self.pretrain_epochs):
            start = time.time()
            self.start_epoch()
            training_epoch_info = self.collector.train_one_epoch()
            for reward in training_epoch_info["train_rewards"]:
                self.training_episode_rewards.append(reward)
            finish_epoch_info = self.finish_epoch()
            total_frames += self.epoch_frames
            infos = {"Train_Epoch_Reward": training_epoch_info["train_epoch_reward"],
                     "Running_Training_Average_Rewards":
                         np.mean(self.training_episode_rewards) if len(self.training_episode_rewards) else float("nan")}
            infos.update(finish_epoch_info)
            if self.logger is not None:
                self.logger.add_epoch_info(pretrain_epoch, total_frames, time.time() - start, infos, csv_write=False)
        if self.logger is not None:
            self.logger.log("Finished Pretrain")
