"""V-MPO on the device (API of /root/reference/torchrl/algo/on_policy/v_mpo.py:11-185).

Same minibatch loop and explicit-batch `update` as A2C / PPO (a2c.A2C: row gather, per-epoch advantage statistics,
fused clip + Adam for every optimised tensor in one step, one captured CUDA graph per minibatch, no host sync inside).
The actor step is the reference's (v_mpo.py:59-125): keep the half of the minibatch with the largest normalised
advantages, weight the log-likelihood by softmax(adv / eta), add alpha * KL(pi || pi_target), learn the temperature
eta and the KL multiplier alpha by their dual losses, clamp both at 1e-8.  The MLPs run on the library's fused
layers; the per-sample loss assembly (sort, softmax, KL) is a handful of elementwise torch ops inside the captured
graph.  eta and alpha live in one 2-element parameter optimised by a third segment of the flat Adam (lr = plr,
eps = 1e-5, no clipping: v_mpo.py:33-37).

With a CategoricalDisPolicy the actor step runs on the library's kernels instead (csrc/categorical.cu): one launch per
epoch selects the top half of every minibatch (`_epoch_adv_stats`), and one launch per minibatch computes the loss,
its gradient wrt the selected rows' logits and the duals' gradient.  reference_quirks=True keeps the reference's
summed KL: for a Categorical, kl_divergence(...).sum(-1, keepdim=True) sums over the rows (one scalar K that enters
every row's loss and the alpha loss); False uses the per-row KL of the Gaussian path and the V-MPO paper.
"""
import torch

from ... import ops
from ..utils import four_stats
from .a2c import A2C
from .policy_heads import CategoricalHead


class VMPO(A2C):
    _target_segments = ("pf",)

    def __init__(self, pf, opt_epochs=10, eta_eps=0.02, alpha_eps=0.1, clipped_value_loss=False,
                 reference_quirks=True, **kwargs):
        self.reference_quirks = reference_quirks
        self.eta_eps, self.alpha_eps = eta_eps, alpha_eps
        self.opt_epochs = opt_epochs
        dev = torch.device(kwargs.get("device", "cuda"))
        self.dual = torch.nn.Parameter(torch.tensor([1.0, 0.1], dtype=torch.float32, device=dev))   # [eta, alpha]
        super().__init__(pf=pf, **kwargs)
        self.sample_key = ["obs", "acts", "advs", "estimate_returns", "values"]
        self._categorical = isinstance(self._head, CategoricalHead)

    @property
    def eta(self):
        return self.dual[0:1]

    @property
    def alpha(self):
        return self.dual[1:2]

    def _extra_opt_segments(self):
        return [(None, [self.dual], self.plr)]

    def _passes(self):
        return self.opt_epochs

    def _gather_keys(self):
        return ["obs", "acts", "advs", "estimate_returns"]

    def _pre_update(self):
        self._hard_update_targets()                              # copy_model_params_from_to(pf, target_pf)

    def _critic_step(self, batch, st, info):
        v = self.vf(batch["obs"])
        g_v, _ = ops.ppo_critic_loss(v.reshape(-1), batch["estimate_returns"].reshape(-1), None, False, 0.0,
                                     st["scratch"], info=info[16:17])
        torch.autograd.backward([v], [g_v.reshape(v.shape)])

    def _actor_loss(self, obs, acts, advn, info):
        """v_mpo.py:59-125 on (B, .) device tensors with already normalised advantages; writes the logged scalars
        into `info` (device) and returns the scalar loss."""
        B = advn.shape[0]
        idx = torch.sort(advn.reshape(-1), dim=0, descending=True)[1][:B - B // 2]      # chunk(2)[0]: ceil(B/2)
        obs, acts, adv = obs[idx], acts[idx], advn.reshape(-1, 1)[idx]
        out = self.pf.update(obs, acts)
        log_probs, mean, std = out["log_prob"], out["mean"], out["std"]
        with torch.no_grad():
            tmean, tstd, _ = self.target_pf(obs)
        eta, alpha = self.dual[0:1], self.dual[1:2]
        phis = torch.softmax(adv / eta.detach(), dim=0)
        eta_loss = eta * self.eta_eps + eta * torch.log(torch.mean(torch.exp(adv / eta)))
        kl = (torch.log(tstd / std) + (std * std + (mean - tmean) ** 2) / (2.0 * tstd * tstd) - 0.5).sum(-1, keepdim=True)
        alpha_loss = alpha * self.alpha_eps - alpha * kl.detach().mean()
        policy_loss = (-phis * log_probs + alpha.detach() * kl).mean()
        info[32:33].copy_(policy_loss.detach().reshape(1))
        info[33:34].copy_(alpha_loss.detach().reshape(1))
        ops.vec_stats(log_probs.detach().reshape(-1).contiguous(), out=info[36:40])
        ops.vec_stats(kl.detach().reshape(-1).contiguous(), out=info[40:44])
        return policy_loss + eta_loss.sum() + alpha_loss.sum()

    def _actor_step(self, batch, st, info):
        if self._categorical:
            sel = st["sel"].index_select(0, st["upd"].long()).reshape(-1)        # this minibatch's top half
            self._head.vmpo_actor(self.pf, self.target_pf, batch["obs"].index_select(0, sel),
                                  batch["acts"].reshape(-1).index_select(0, sel),
                                  batch["advs"].reshape(-1).index_select(0, sel), st["adv_table"], st["upd"], self.dual,
                                  self.eta_eps, self.alpha_eps, not self.reference_quirks, st["vmpo_scratch"],
                                  info[32:44])
            return
        row = st["adv_table"].index_select(0, st["upd"].long())                  # this minibatch's statistics
        advn = (batch["advs"].reshape(-1, 1) - row[:, 0:1]) / (row[:, 1:2] + 1e-5)
        acts = batch["acts"].reshape(advn.shape[0], -1)
        loss = self._actor_loss(batch["obs"], acts, advn, info)
        loss.backward()

    def _step(self, batch, st):
        scale = super()._step(batch, st)
        with torch.no_grad():
            self.dual.clamp_(min=1e-8)                                           # v_mpo.py:101-103
        return scale

    def _mb_body(self):
        super()._mb_body()
        with torch.no_grad():
            self._mb_state["dual_log"].index_copy_(0, self._dual_pos(), self.dual.detach().reshape(1, 2))

    def _dual_pos(self):
        # the counter has already advanced: log the clamped duals of update u at row u through a device index
        st = self._mb_state
        return ((st["upd"].long() - 1) % st["U"]).reshape(1)

    def _step_state(self, B, U, a):
        st = super()._step_state(B, U, a)
        if self._categorical:
            st["sel"] = torch.zeros(U, B - B // 2, dtype=torch.int64, device=self.device)
            st["vmpo_scratch"] = self._head.vmpo_scratch(B, self.device)
        return st

    def _mb_setup(self):
        st = super()._mb_setup()
        st["dual_log"] = torch.zeros(st["U"], 2, dtype=torch.float32, device=self.device)
        return st

    def _prepare_batch(self, batch, st):
        """The batch's advantage statistics and, for a categorical policy, its top half."""
        super()._prepare_batch(batch, st)
        if self._categorical:
            ops.vmpo_select(batch["advs"].reshape(-1), st["adv_table"], 1, st["B"], out=st["sel"])

    def _epoch_adv_stats(self):
        super()._epoch_adv_stats()
        if self._categorical:                  # every minibatch's top half, once per epoch
            st, rb = self._mb_state, self.replay_buffer
            ops.vmpo_select(rb._advs.reshape(rb._advs.shape[0], -1), st["adv_table"], st["U"], st["b"],
                            perm=st["perm"], out=st["sel"])

    def _flush_infos(self, n_updates):
        self._dual_rows = self._mb_state["dual_log"][:n_updates].cpu().numpy()
        infos = super()._flush_infos(n_updates)
        for u, info in enumerate(infos):
            info['Training/eta'], info['Training/alpha'] = float(self._dual_rows[u][0]), float(self._dual_rows[u][1])
        return infos

    def _decode_info(self, row, norms, st):
        info = four_stats('advs', row[20:24])
        info['Training/vf_loss'] = float(row[16])
        info['grad_norm/vf'] = float(norms[1])
        info['Training/policy_loss'] = float(row[32])
        info['Training/alpha_loss'] = float(row[33])
        info['Training/alpha'] = info['Training/eta'] = float("nan")             # filled by the caller
        info.update(four_stats('logprob', row[36:40]))
        info.update(four_stats('KL', row[40:44]))
        info['grad_norm/pf'] = float(norms[0])
        return info

    def update(self, batch):
        info = super().update(batch)
        info['Training/eta'], info['Training/alpha'] = (float(v) for v in self.dual.detach().cpu().numpy())
        return info
