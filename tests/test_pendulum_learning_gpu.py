"""Learning on the device Pendulum-v1: with fixed seeds, TD3 and TwinSAC-Q with config/td3_pendulum.json and
config/twin_sac_q_pendulum.json reach a mean greedy evaluation return far above a uniformly random policy's (about -1230,
tests/test_pendulum_cpu.py::test_random_policy_baseline) within a fixed frame budget.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), seed 0, 16 envs, one pretraining epoch, then evaluating every
5 epochs of 1600 frames on 16 evaluation envs (`python -m tests.test_pendulum_learning_gpu`):
    TD3        epochs 5-40: -793, -500, -148, -241, -157, -119, -169, -152
    TwinSAC-Q  epochs 5-40: -176, -255, -147, -159, -163, -119, -168, -151
The budget is 25 epochs (40,000 frames plus 1,600 of pretraining) for TD3 and 20 (32,000 + 1,600) for TwinSAC-Q; the
threshold is -500 for both: more than twice the worst return measured from epoch 15 on, and 730 above the random
policy's -1230."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N = 16
# epochs of 1600 frames after one pretraining epoch, and the evaluation threshold per agent
BUDGET = {"td3": 25, "twin_sac_q": 20}
THRESHOLD = {"td3": -500.0, "twin_sac_q": -500.0}


def train(kind, epochs, seed=0, report=None):
    """Train `kind` on Pendulum-v1 for `epochs` epochs; returns the mean greedy return of the N evaluation envs after
    the last epoch.  report(epoch, mean return) is called every 5 epochs when given."""
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import TD3, TwinSACQ
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer
    from torchrl_b200.utils import NullLogger
    cfg = json.load(open(os.path.join(ROOT, "config", "%s_pendulum.json" % kind)))
    g = cfg["general_setting"]
    dev = torch.device("cuda:0")
    env, eval_env = get_vec_env("Pendulum-v1", cfg["env"], N), get_vec_env("Pendulum-v1", cfg["env"], N)
    env.seed(seed); eval_env.seed(seed + 1000); torch.manual_seed(seed); np.random.seed(seed)
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=int(cfg["replay_buffer"]["size"]),
                           time_limit_filter=cfg["replay_buffer"]["time_limit_filter"])
    net = dict(cfg["net"], base_type=networks.MLPBase, activation_func=torch.nn.ReLU)
    if kind == "td3":
        pf = policies.FixGuassianContPolicy(input_shape=3, output_shape=1, **net, **cfg["policy"])
    else:
        pf = policies.GuassianContPolicy(input_shape=3, output_shape=2, **net, **cfg["policy"])
    qf1 = networks.QNet(input_shape=4, output_shape=1, **net)
    qf2 = networks.QNet(input_shape=4, output_shape=1, **net)
    col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, **cfg["collector"])
    common = dict(g, num_epochs=epochs, env=env, replay_buffer=buf, collector=col, logger=NullLogger(), device=dev,
                  save_dir=None)
    for k in ("eval_interval", "save_interval"):
        common.pop(k)
    if kind == "td3":
        agent = TD3(pf=pf, qf1=qf1, qf2=qf2, **cfg["td3"], **common)
    else:
        agent = TwinSACQ(pf=pf, qf1=qf1, qf2=qf2, **cfg["twin_sac_q"], **common)
    agent.pretrain()
    ret = None
    for epoch in range(epochs):
        agent.current_epoch = epoch
        col.train_one_epoch()
        agent.update_per_epoch()
        if (report is not None and (epoch + 1) % 5 == 0) or epoch == epochs - 1:
            ret = float(np.mean(col.eval_one_epoch()["eval_rewards"]))
            if report is not None:
                report(epoch + 1, ret)
    return ret


@pytest.mark.parametrize("kind", ["td3", "twin_sac_q"])
def test_agent_learns_to_swing_up(kind):
    ret = train(kind, BUDGET[kind])
    assert ret >= THRESHOLD[kind], (kind, ret)


if __name__ == "__main__":
    import sys
    import time
    for kind in sys.argv[1:] or ["td3", "twin_sac_q"]:
        t0 = time.time()
        train(kind, 40, report=lambda e, r: print("%s epoch %d return %.1f (%.0f s)" % (kind, e, r, time.time() - t0),
                                                  flush=True))
