"""DQN and QR-DQN (API of /root/reference/torchrl/algo/off_policy/dqn.py:8-98, qrdqn.py:11-74).

The whole loss -- gather of the taken action's value/quantiles, greedy target selection,
TD target, squared-error / quantile-Huber reduction and its gradient -- is ONE kernel launch
(csrc/offpolicy.cu: qr_loss_kernel).  `acts` are stored (T,N) as in the reference's collector
(collector/base.py:190-191); the reference's DQN.update itself crashes on that shape
(dqn.py:54, SURVEY.md A.4) -- the oracle for DQN is the reference expression with acts (B,1).
"""
import torch
import torch.optim as optim

from ... import ops
from .off_rl_algo import OffRLAlgo


class DQN(OffRLAlgo):
    quantile_num = 1
    _mse = True

    def __init__(self, qf, pf, qlr, optimizer_class=optim.Adam, optimizer_info={}, **kwargs):
        super().__init__(**kwargs)
        self.pf = pf
        self.qf = qf
        self.qlr = qlr
        # no clipping, whatever grad_clip says: the reference's DQN never clips
        self._init_networks(optimizer_class, [("qf", qf, qlr)], eps=optimizer_info.get("eps", 1e-8), max_norms=[0.0],
                            targets=("qf",))
        self.obs_scale = getattr(self.env, "obs_scale", None)

    def _prep_obs(self, x):
        """uint8 frames -> float32 * obs_scale (ScaledFloatFrame) in one launch; float inputs pass through."""
        if x.dtype == torch.uint8:
            if hasattr(self.env, "to_float") and x.is_contiguous() and x.numel() % 4 == 0:
                return self.env.to_float(x)
            x = x.float()
            if self.obs_scale:
                x = x * self.obs_scale
        return x

    # info: 0 loss 1 q_s_a 2 Reward_Mean
    def _update_body(self, variant):
        ub = self._ub
        batch = self._batch()
        info = ub["info"][0]
        obs, next_obs = self._prep_obs(batch["obs"]), self._prep_obs(batch["next_obs"])
        acts = batch["acts"].reshape(-1).float()
        rewards, terminals = batch["rewards"].reshape(-1), batch["terminals"].reshape(-1)
        q_pred = self.qf(obs)
        with torch.no_grad():
            next_q = self.target_qf(next_obs).contiguous()
        A = q_pred.shape[-1] // self.quantile_num
        pred = q_pred if q_pred.is_contiguous() else q_pred.contiguous()
        weights = batch.get("weights")                 # prioritised replay: importance weights, TD magnitudes out
        td = self._td if weights is not None and self._explicit_batch is None else None
        grad, _ = ops.qr_dqn_loss(pred, next_q, acts.contiguous(), rewards, terminals, self.discount, ub["scratch"],
                                  A, self.quantile_num, mse=self._mse, info=info[0:3],
                                  weights=None if weights is None else weights.reshape(-1).contiguous(),
                                  td_out=td)
        torch.autograd.backward([pred], [grad])
        self._optimizer_step()
        self._update_target_networks()
        self._finish_update()

    def _decode_info(self, row, variant):
        return {'Reward_Mean': float(row[2]), 'Training/qf_loss': float(row[0]),
                'epsilon': float(getattr(self.pf, "epsilon", float("nan"))), 'q_s_a': float(row[1])}

    @property
    def snapshot_networks(self):
        return [("pf", self.qf)]         # the reference names the Q-network's snapshot files model_pf_*


class QRDQN(DQN):
    _mse = False

    def __init__(self, quantile_num=100, **kwargs):
        super().__init__(**kwargs)
        self.quantile_num = quantile_num
        self.quantile_coefficient = ((2 * torch.arange(quantile_num, dtype=torch.float32) + 1)
                                     / (2.0 * quantile_num)).view(1, -1).to(self.device)
