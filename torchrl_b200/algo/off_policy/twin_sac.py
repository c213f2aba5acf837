"""Twin-Q soft actor-critic with a state-value network V
(API of /root/reference/torchrl/algo/off_policy/twin_sac.py:10-254): SAC's update (sac.py here) with
min(Q1, Q2) in the value target and the policy loss, and one MSE per critic."""
import torch.optim as optim

from .sac import SAC


class TwinSAC(SAC):
    _critic_names = ("qf1", "qf2")
    TD_COLUMNS = 2

    def __init__(self, pf, vf, qf1, qf2, plr, vlr, qlr, optimizer_class=optim.Adam, policy_std_reg_weight=1e-3,
                 policy_mean_reg_weight=1e-3, reparameterization=True, automatic_entropy_tuning=True,
                 target_entropy=None, **kwargs):
        super().__init__(pf, vf, [qf1, qf2], plr, vlr, qlr, optimizer_class, policy_std_reg_weight,
                         policy_mean_reg_weight, reparameterization, automatic_entropy_tuning, target_entropy, **kwargs)
