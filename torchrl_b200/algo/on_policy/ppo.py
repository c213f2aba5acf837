"""PPO on the device (API of /root/reference/torchrl/algo/on_policy/ppo.py:10-160).

The per-minibatch loop (gather -> critic loss -> actor loss -> [gradient exchange] -> clip + Adam -> log row, one
captured CUDA graph replayed opt_epochs * T/b times per epoch, no host sync inside) and the explicit-batch `update` live
in a2c.A2C; PPO adds the clipped surrogate (the actor kernel's ratio mode), the optional clipped value loss, the linear
LR decay and the target policy.

Exactness notes (SURVEY.md section 7):
  * old log-probs are computed once per epoch and gathered with the minibatch -- the reference recomputes
    target_pf(obs) every minibatch (ppo.py:54-56) but target_pf is constant within an epoch, so the cached values are
    the same numbers;
  * critic and actor steps of one minibatch are fused into one optimizer launch: the two networks share no parameters,
    so the result equals the reference's critic-then-actor order;
  * minibatch row order comes from np.random.permutation on the host (bit-exact indexing).
"""
import numpy as np
import torch

from ... import ops
from ...networks import fused
from .. import utils as atu
from .a2c import A2C

# info slots 0-6 of the actor loss kernels; slots 7-10 hold the head's extra keys (log_std/* of a Gaussian policy)
_INFO_KEYS_ACTOR = ['Training/policy_loss', 'logprob/mean', 'logprob/std', 'logprob/max', 'logprob/min',
                    'ratio/max', 'ratio/min']


class PPO(A2C):
    _target_segments = ("pf",)

    def __init__(self, pf, clip_para=0.2, opt_epochs=10, clipped_value_loss=False, **kwargs):
        super().__init__(pf=pf, **kwargs)
        self.clip_para = clip_para
        self.opt_epochs = opt_epochs
        self.clipped_value_loss = clipped_value_loss
        self.sample_key = ["obs", "acts", "advs", "estimate_returns", "values"]

    # ------------------------------------------------------------------ specialisation of the minibatch loop
    def _passes(self):
        return self.opt_epochs

    def _gather_keys(self):
        return ["obs", "acts", "advs", "estimate_returns", "values", "old_logp"]

    def _device_path_ok(self):
        return True

    def _critic_step(self, batch, st, info):
        v = self.vf(batch["obs"])
        g_v, _ = ops.ppo_critic_loss(v.reshape(-1), batch["estimate_returns"].reshape(-1),
                                     batch["values"].reshape(-1), self.clipped_value_loss, self.clip_para,
                                     st["scratch"], info=info[16:17])
        with fused.backward_fork():
            torch.autograd.backward([v], [g_v.reshape(v.shape)])

    def _actor_step(self, batch, st, info):
        self._head.actor(self.pf, batch["obs"], batch["acts"], batch["old_logp"].reshape(-1), batch["advs"].reshape(-1),
                         st["adv_table"], st["upd"], self.clip_para, self.entropy_coeff, st["scratch"], info)

    def _cache_old_logp(self):
        """log pi_old(a|s) for every stored transition, once per epoch (see module docstring).  Chunks of whole time
        rows, sized by the observation so that the chunk's network activations stay small: a 4x84x84 frame stack is
        113 KB per sample in float32."""
        rb = self.replay_buffer
        if not hasattr(rb, "_old_logp"):
            rb.allocate("old_logp", tuple(rb._rewards.shape[1:]))
        T, N = rb._obs.shape[0], rb._obs.shape[1]
        per_sample = int(np.prod(rb._obs.shape[2:])) * 4
        samples = max(1, min(1 << 16, (256 << 20) // (16 * per_sample)))
        rows = max(1, samples // N)
        with torch.no_grad():
            for r0 in range(0, T, rows):
                r1 = min(T, r0 + rows)
                obs = self._prep_obs(rb._obs[r0:r1].reshape((-1,) + tuple(rb._obs.shape[2:])))
                acts = rb._acts[r0:r1].reshape(obs.shape[0], -1)
                self._head.old_log_prob(self.pf, obs, acts, rb._old_logp[r0:r1].reshape(-1))

    def _pre_update(self):
        """ppo.py:29-34: linear LR decay, target <- pf; then the epoch's old log-probs."""
        atu.update_linear_schedule(self.pf_optimizer, self.current_epoch, self.num_epochs, self.plr)
        atu.update_linear_schedule(self.vf_optimizer, self.current_epoch, self.num_epochs, self.vlr)
        self._hard_update_targets()                              # copy_model_params_from_to(pf, target_pf)
        self._cache_old_logp()

    def _prepare_batch(self, batch, st):
        """The batch's advantage statistics, and its old log-probs from the target policy when it brings none
        (ppo.py:54-56)."""
        super()._prepare_batch(batch, st)
        if "old_logp" not in batch:
            with torch.no_grad():
                batch["old_logp"] = self._head.old_log_prob(self.target_pf, batch["obs"], batch["acts"], None)

    def _decode_info(self, row, norms, st):
        info = atu.four_stats('advs', row[20:24])
        info['Training/vf_loss'] = float(row[16])
        info['grad_norm/vf'] = float(norms[1])
        for i, k in enumerate(_INFO_KEYS_ACTOR):
            info[k] = float(row[i])
        for i, k in enumerate(self._head.ppo_extra_keys):
            info[k] = float(row[7 + i])
        info['grad_norm/pf'] = float(norms[0])
        return info
