"""Learning on the device CartPole-v1: with fixed seeds, REINFORCE with config/reinforce_cartpole.json's
hyperparameters and categorical PPO reach a mean greedy evaluation return far above a uniformly random policy's (about
22) within a fixed frame budget.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), seed 0, evaluating every 10 epochs: REINFORCE returned 500
(the v1 maximum) at every evaluation from epoch 70 to 150, PPO returned 500 at epoch 100 and 291-500 at epochs 80-120.
The budget is 100 epochs (102,400 frames) for both and the threshold 100, a fifth of the return measured there."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# epochs of 1024 frames (8 envs x 128 steps) and the evaluation threshold per agent
BUDGET = {"reinforce": 100, "ppo": 100}
THRESHOLD = {"reinforce": 100.0, "ppo": 100.0}


def train(kind, epochs, seed=0, report=None):
    """Train `kind` on CartPole-v1 for `epochs` epochs; returns the mean greedy return of the 8 evaluation envs after
    the last epoch.  report(epoch, mean return) is called every 10 epochs when given."""
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import PPO, Reinforce
    from torchrl_b200.collector import VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    from torchrl_b200.utils import NullLogger
    cfg = json.load(open(os.path.join(ROOT, "config", "reinforce_cartpole.json")))
    g = cfg["general_setting"]
    N = 8
    dev = torch.device("cuda:0")
    env, eval_env = get_vec_env("CartPole-v1", cfg["env"], N), get_vec_env("CartPole-v1", cfg["env"], N)
    env.seed(seed); eval_env.seed(seed + 1000); torch.manual_seed(seed); np.random.seed(seed)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=g["epoch_frames"], time_limit_filter=True)
    net = dict(input_shape=4, append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=torch.nn.Tanh)
    pf = policies.CategoricalDisPolicy(output_shape=2, hidden_shapes=cfg["net"]["hidden_shapes"], **net)
    vf = networks.ZeroNet() if kind == "reinforce" else networks.Net(output_shape=1, hidden_shapes=[64, 64], **net)
    col = VecOnPolicyCollector(vf, env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev,
                               epoch_frames=g["epoch_frames"], max_episode_frames=g["max_episode_frames"],
                               discount=g["discount"])
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=g["discount"],
                  num_epochs=epochs, batch_size=g["batch_size"], device=dev, save_dir=None)
    if kind == "reinforce":
        agent = Reinforce(pf=pf, **cfg["reinforce"], **common)
    else:
        agent = PPO(pf=pf, vf=vf, plr=1e-3, vlr=1e-3, opt_epochs=4, clip_para=0.2, entropy_coeff=0.0, tau=0.95,
                    gae=True, shuffle=True, **common)
    ret = None
    for epoch in range(epochs):
        agent.current_epoch = epoch
        col.train_one_epoch()
        agent.update_per_epoch()
        if report is not None and (epoch + 1) % 10 == 0 or epoch == epochs - 1:
            ret = float(np.mean(col.eval_one_epoch()["eval_rewards"]))
            if report is not None:
                report(epoch + 1, ret)
    return ret


@pytest.mark.parametrize("kind", ["reinforce", "ppo"])
def test_agent_learns_to_balance(kind):
    ret = train(kind, BUDGET[kind])
    assert ret >= THRESHOLD[kind], (kind, ret)
