"""Advantage actor-critic on the device (API of /root/reference/torchrl/algo/on_policy/a2c.py:8-112) and the
minibatch machinery PPO shares with it.

Per minibatch (one captured CUDA graph, replayed T/b times per pass):
  row gather of all keys (1 launch) -> vf forward -> critic loss fwd+bwd kernel -> autograd through vf -> value
  statistics (1) -> pf forward -> actor loss fwd+bwd kernel (policy-gradient mode: L = -mean(logp * adv_norm) -
  c_ent * mean(ent), a2c.py:66-70) -> autograd through pf -> [gradient exchange] -> grad-norm + clip(0.5) + Adam
  (eps 1e-5) for both networks in one step (a2c.py:29-39, 72-80: two optimizers over disjoint parameters) -> info row.
The advantage statistics of every minibatch of the epoch are computed once up-front (`_epoch_adv_stats`).  Nothing
syncs with the host inside the loop: the reference's 12 `.item()` calls per update (a2c.py:82-98) become one device
log fetched per epoch.  The constructor re-homes pf and vf into one flat buffer (flat.FlatAdam).
`update(batch)` runs the same minibatch step (`_step`) on an explicit batch, with that batch's own advantage statistics.
"""
import numpy as np
import torch
import torch.optim as optim

from ... import ops
from ...networks import fused
from ..utils import four_stats
from .on_rl_algo import OnRLAlgo
from .policy_heads import policy_head


class A2C(OnRLAlgo):
    def __init__(self, pf, vf, plr=3e-4, vlr=3e-4, optimizer_class=optim.Adam, entropy_coeff=0.001, **kwargs):
        super().__init__(**kwargs)
        self.pf = pf
        self.vf = vf
        self.plr = plr
        self.vlr = vlr
        self.optimizer_class = optimizer_class
        # segment 0 = policy, segment 1 = value net (each clipped to 0.5), then whatever a subclass optimises besides
        # (unclipped)
        nets = self._net_segments(plr, vlr)
        extra = self._extra_opt_segments()
        self._init_networks(optimizer_class, nets + extra, eps=self.adam_eps,
                            max_norms=[0.5] * len(nets) + [0.0] * len(extra), targets=self._target_segments)
        self.entropy_coeff = entropy_coeff
        self.vf_criterion = torch.nn.MSELoss()
        self.sample_key = ["obs", "acts", "advs", "estimate_returns"]
        self.tanh_action = bool(getattr(pf, "tanh_action", False))
        self._head = policy_head(pf)
        self._mb_graph = None
        self._mb_eager_runs = 0
        self._mb_state = None
        self._last_infos = []
        self._side_stream = torch.cuda.Stream(device=self.device)

    # ------------------------------------------------------------------ what subclasses specialise
    adam_eps = 1e-5
    _target_segments = ()           # the segments whose network has a target network (PPO and V-MPO: "pf")

    def _net_segments(self, plr, vlr):
        """[(name, network, lr)] of the networks the agent trains, each clipped to a gradient norm of 0.5."""
        return [("pf", self.pf, plr), ("vf", self.vf, vlr)]

    def _extra_opt_segments(self):
        """[(name or None, parameter list, lr)] optimised without clipping by the same fused step besides pf and vf."""
        return []

    def _step_mask(self):
        """Bit mask of the optimizer segments that step in the minibatch loop (None: all)."""
        return None

    def _passes(self):
        """Optimisation passes over the epoch's rollout (a2c: one; ppo: opt_epochs)."""
        return 1

    def _gather_keys(self):
        return ["obs", "acts", "advs", "estimate_returns"]

    def _critic_step(self, batch, st, info):
        v = self.vf(batch["obs"])
        g_v, _ = ops.ppo_critic_loss(v.reshape(-1), batch["estimate_returns"].reshape(-1), None, False, 0.0,
                                     st["scratch"], info=info[16:17])
        with fused.backward_fork():
            torch.autograd.backward([v], [g_v.reshape(v.shape)])
        ops.vec_stats(v.detach().reshape(-1), out=info[24:28])          # v_pred/* (a2c.py:85-88)

    def _actor_step(self, batch, st, info):
        std = self._head.actor(self.pf, batch["obs"], batch["acts"], None, batch["advs"].reshape(-1), st["adv_table"],
                               st["upd"], 0.0, self.entropy_coeff, st["scratch"], info)
        self._head.std_row(self.pf, std, info)

    def _pre_update(self):
        """Host-side work of an epoch before the minibatch loop (schedules, target copies)."""

    def _prepare_batch(self, batch, st):
        """For an explicit batch, what the epoch computes once for all of its minibatches (`_epoch_adv_stats`): the
        advantage statistics, here of this batch alone (a2c.py:62)."""
        ops.vec_stats(batch["advs"].reshape(-1), out=st["adv_table"][0])

    def _decode_info(self, row, norms, st):
        info = {'Training/policy_loss': float(row[0]), 'Training/vf_loss': float(row[16])}
        info.update(four_stats('v_pred', row[24:28]))
        info.update(self._head.a2c_std_info(row, st["B"], st["a"]))
        info['ent'] = float(row[11])
        info['log_prob'] = float(row[1])
        return info

    # ------------------------------------------------------------------ helpers
    def _device_path_ok(self):
        """The fused minibatch loop needs a policy its head supports (a Gaussian policy with a shared log-std vector,
        or a categorical policy) over a device rollout buffer; anything else runs `update(batch)` on each minibatch."""
        rb = self.replay_buffer
        return self._head.fused_ok(self.pf) and rb is not None and hasattr(rb, "gather_rows") and hasattr(rb, "_rewards")

    def _step_state(self, B, U, a):
        """What a minibatch step of B samples (a action components) runs against: the loss kernels' scratch, the info
        row, and the (U, 4) advantage statistics table (mean, std, max, min per row) read at row `upd`."""
        dev = self.device
        return {
            "B": B, "U": U, "a": a,
            "n": B,                                                 # samples behind one row of the table
            "upd": torch.zeros(1, dtype=torch.int32, device=dev),
            "info": torch.zeros(1, 64, dtype=torch.float32, device=dev),
            "scratch": self._head.loss_scratch(B, a, dev),
            "adv_table": torch.zeros(U, 4, dtype=torch.float32, device=dev),
        }

    def _mb_setup(self):
        rb = self.replay_buffer
        N = rb.env_nums
        assert self.batch_size % N == 0, "batch size should be dividable by env_nums"
        b = self.batch_size // N
        T = rb._max_replay_buffer_size
        assert T % b == 0, "rows per minibatch must divide the buffer rows"
        n_mb = T // b
        passes = self._passes()
        U = passes * n_mb
        dev = self.device
        W = self.dist.world_size if (self.dist is not None and self.dist.active) else 1
        # one step state for all U minibatches of the epoch: `upd` is the gather position, the statistics row and the
        # log row of minibatch u
        st = self._step_state(b * N, U, int(np.prod(rb._acts.shape[2:])))
        st.update({
            "b": b, "n_mb": n_mb, "passes": passes, "n": b * N * W,     # the table spans every rank's rows
            # every pass' row order is uploaded up-front: (passes, T) indices, minibatch u of the epoch reads
            # perm[u*b : (u+1)*b]
            "perm": torch.zeros(passes * T, dtype=torch.int64, device=dev),
            "perm_host": torch.zeros(passes * T, dtype=torch.int64).pin_memory(),
            "log_ticket": torch.zeros(1, dtype=torch.int32, device=dev),
            "log32": torch.zeros(U, 64, dtype=torch.float32, device=dev),
            "log64": torch.zeros(U, self.opt.sumsq3.numel(), dtype=torch.float64, device=dev),
            "keys": self._gather_keys(),
        })
        st["log_plan"] = ops.RowCopyPlan([st["info"], self.opt.sumsq3.view(1, -1)], [st["log32"], st["log64"]],
                                         [64 * 4, self.opt.sumsq3.numel() * 8])
        self._mb_state = st
        return st

    def _step(self, batch, st):
        """One minibatch update against the step state `st`; returns the gradient scale of the optimizer step.
        `batch` None: the epoch's minibatch, whose row indices are read at device position `upd` and whose log row is
        written before `upd` advances.  Layer gradients go straight into the flat gradient buffer
        (networks.fused.direct_grad): every parameter gets exactly one contribution per minibatch and the optimizer step
        left the buffer zeroed.  The dgrad GEMMs read transposed weight planes, rewritten from the previous optimizer
        step's planes beside the gather and the forward passes."""
        with fused.direct_grad(), fused.deferred_reduces(), fused.transposed_planes(self.opt):
            epoch = batch is None
            if epoch:
                batch = self.replay_buffer.gather_rows(st["perm"], st["keys"], pos_ptr=st["upd"], rows=st["b"])
                batch["obs"] = self._prep_obs(batch["obs"])
            info = st["info"][0]
            # the critic and the actor branch share nothing but their (read-only) inputs: run them on two streams --
            # under capture this becomes two parallel branches of the graph -- so that their many latency-bound
            # launches overlap instead of queueing behind one another
            main = torch.cuda.current_stream(self.device)
            side = self._side_stream
            side.wait_stream(main)
            with torch.cuda.stream(side):
                self._critic_step(batch, st, info)
            self._actor_step(batch, st, info)
            main.wait_stream(side)
            fused.flush_reduces()              # the slab sums of both networks' skinny gradients, one launch
            scale = self._optimizer_step(self._step_mask())
            if epoch:
                # the log row, then upd += 1
                ops.ring_write_advance(st["log_plan"], st["upd"], st["U"], st["log_ticket"])
            return scale

    def _mb_body(self):
        """One minibatch update of the epoch (what the captured graph holds)."""
        self._step(None, self._mb_state)

    def _run_minibatch(self):
        if not self.use_cuda_graph:
            self._mb_body()
        elif self._mb_graph is not None:
            self._mb_graph.replay()
        elif self._mb_eager_runs < 3:
            self._mb_eager_runs += 1
            self._mb_body()
        else:
            g = ops.CapturedGraph(self._mb_body)
            self._mb_graph = g
            g.replay()
        self.training_update_num += 1

    def _epoch_adv_stats(self):
        """a2c.py:62 / ppo.py:141-147 for ALL minibatches of the epoch at once: which time rows form minibatch u is
        known as soon as the permutations are uploaded, so one launch reduces every minibatch's advantages to raw
        moments, (data parallel) ONE exchange gathers the ranks' moments, one launch turns them into the (U,4) table
        the actor loss indexes with the device counter.  Per minibatch this removes a reduction launch and, with
        several ranks, an all-gather."""
        st, rb = self._mb_state, self.replay_buffer
        U, b = st["U"], st["b"]
        dp = self.dist is not None and self.dist.active
        W = self.dist.world_size if dp else 1
        if "mom_all" not in st:
            st["mom_all"] = torch.zeros(W, U, 4, dtype=torch.float64, device=self.device)
            if dp and self.dist.peer is not None:
                st["mom"] = self.dist.peer.region("adv_moments", 32 * U, torch.float64)[0][:4 * U].view(U, 4)
            else:
                st["mom"] = torch.zeros(U, 4, dtype=torch.float64, device=self.device) if dp else st["mom_all"][0]
        advs = rb._advs.reshape(rb._advs.shape[0], -1)
        ops.row_group_moments(advs, st["perm"], U, b, out=st["mom"])
        if dp:
            if self.dist.peer is not None:
                self.dist.peer.all_reduce_f64("adv_moments", 4 * U, st["mom_all"], gather=True)
            else:
                import torch.distributed as tdist
                tdist.all_gather_into_tensor(st["mom_all"].view(-1), st["mom"].view(-1))
        ops.group_stats_from_moments(st["mom_all"], W, U, float(st["n"]), out=st["adv_table"])

    def _flush_infos(self, n_updates):
        """One D2H copy of the epoch's per-update scalars -> list of the reference's info dicts."""
        st = self._mb_state
        log32 = st["log32"][:n_updates].cpu().numpy()
        log32[:, 20:24] = st["adv_table"][:n_updates].cpu().numpy()
        log64 = st["log64"][:n_updates].cpu().numpy()
        # the flat gradient holds the SUM over ranks; the averaged gradient's norm is what one process sees
        gs = 1.0 / self.dist.world_size if (self.dist is not None and self.dist.active) else 1.0
        return [self._decode_info(log32[u], np.sqrt(log64[u][:self.opt.nseg]) * gs, st) for u in range(n_updates)]

    # ------------------------------------------------------------------ reference API
    @fused.presplit_scope
    def update_per_epoch(self, flush_infos=True):
        """on_rl_algo.py:35-42 (a2c) / ppo.py:27-39: advantages, then `passes` sweeps of row-order minibatches.
        flush_infos=False skips the end-of-epoch read-back of the logged scalars (device-only benchmarking)."""
        if not self._device_path_ok():
            return super().update_per_epoch()
        self.process_epoch_samples()
        self._pre_update()
        self._minibatch_epoch(flush_infos)

    def _minibatch_epoch(self, flush_infos):
        """`passes` sweeps of row-order minibatches over the stored rollout, one captured minibatch graph each."""
        st = self._mb_state or self._mb_setup()
        st["upd"].zero_()
        T = self.replay_buffer._max_replay_buffer_size
        # the reference draws one np.random.permutation per pass and nothing else touches np.random in between, so
        # drawing all passes up-front consumes the global RNG identically
        for e in range(st["passes"]):
            order = self.replay_buffer.epoch_order(self.shuffle)
            st["perm_host"][e * T:(e + 1) * T].copy_(torch.from_numpy(np.ascontiguousarray(order, dtype=np.int64)))
        st["perm"].copy_(st["perm_host"], non_blocking=True)
        self._epoch_adv_stats()
        n = st["U"]
        for _ in range(n):
            self._run_minibatch()
        if flush_infos:
            self._record_infos(self._flush_infos(n))

    def _device_batch(self, batch, keys):
        """The `keys` present in an explicit batch as contiguous device tensors: float32, except uint8 frames, which
        `_prep_obs` then scales as the epoch's gather does."""
        out = {}
        for k in keys:
            if k in batch:
                v = batch[k] if torch.is_tensor(batch[k]) else torch.as_tensor(np.asarray(batch[k]))
                dt = torch.uint8 if (k == "obs" and v.dtype == torch.uint8) else torch.float32
                out[k] = v.to(device=self.device, dtype=dt).contiguous()
        out["obs"] = self._prep_obs(out["obs"])
        return out

    @fused.presplit_scope
    def update(self, batch):
        """One minibatch update on an explicit batch (a2c.py:45-112; PPO, V-MPO and REINFORCE likewise): the epoch's
        `_step` against a one-row step state whose advantage statistics are the batch's own.  Syncs to return the
        reference's info dict."""
        self.training_update_num += 1
        batch = self._device_batch(batch, self._gather_keys())
        B = batch["obs"].shape[0]
        st = self._step_state(B, 1, int(np.prod(batch["acts"].shape[1:])) if "acts" in batch else 1)
        self._prepare_batch(batch, st)
        scale = self._step(batch, st)
        row = st["info"][0].cpu().numpy()
        row[20:24] = st["adv_table"][0].cpu().numpy()                   # where _flush_infos puts the epoch's table
        return self._decode_info(row, self.opt.grad_norms().cpu().numpy() * scale, st)
