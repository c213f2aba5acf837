"""Time of one captured off-policy update at BASELINE config-3 sizes for SAC, TwinSAC and TwinSAC-Q.

  1024 SynthAnt envs (obs 111, act 8), batch 4096, MLP(256,256), opt_times 64, 1M-transition ring.
Each agent collects one pretrain epoch into its own ring and runs two update epochs (eager warm-up and graph capture).
Then the three update graphs are replayed in alternating rounds (ROUNDS x REPLAYS replays each) between CUDA events.
Prints the card's name and power limit with the numbers, one JSON line.

    python scripts/sac_v_bench.py [--rounds 4] [--replays 100]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchrl_b200.networks as networks  # noqa: E402
import torchrl_b200.policies as policies  # noqa: E402
from torchrl_b200.algo import SAC, TwinSAC, TwinSACQ  # noqa: E402
from torchrl_b200.collector import VecCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import BaseReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402

N, U = 1024, 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def build(kind, dev):
    env = get_vec_env("SynthAnt-v0", {"reward_scale": 1, "obs_norm": False}, N)
    ev_env = get_vec_env("SynthAnt-v0", {"obs_norm": False}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    o, a = env.observation_space.shape[0], env.action_space.shape[0]
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=int(1e6))
    net = dict(hidden_shapes=[256, 256], append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=nn.ReLU)
    pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, tanh_action=True, **net)
    qfs = [networks.QNet(input_shape=o + a, output_shape=1, **net) for _ in range(1 if kind == "SAC" else 2)]
    col = VecCollector(env=env, eval_env=ev_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=U * N,
                       max_episode_frames=999)
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, batch_size=4 * N,
                  device=dev, save_dir=None, tau=0.005, opt_times=U, num_epochs=10, plr=3e-4, qlr=3e-4,
                  policy_std_reg_weight=0, policy_mean_reg_weight=0)
    if kind == "TwinSACQ":
        agent = TwinSACQ(pf=pf, qf1=qfs[0], qf2=qfs[1], **common)
    else:
        vf = networks.Net(input_shape=o, output_shape=1, **net)
        agent = SAC(pf=pf, vf=vf, qf=qfs[0], vlr=3e-4, **common) if kind == "SAC" else \
            TwinSAC(pf=pf, vf=vf, qf1=qfs[0], qf2=qfs[1], vlr=3e-4, **common)
    col.train_one_epoch()
    for e in range(2):                       # 3 eager updates, then capture; every shape warmed
        agent.current_epoch = e
        agent.update_per_epoch()
    torch.cuda.synchronize()
    assert 0 in agent._graphs, "update graph not captured"
    return agent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--replays", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sac_v_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    kinds = ("SAC", "TwinSAC", "TwinSACQ")
    agents = {k: build(k, dev) for k in kinds}
    total = {k: 0.0 for k in kinds}
    per_round = {k: [] for k in kinds}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k in kinds:                      # alternate the three agents within every round
            g = agents[k]._graphs[0]
            g.replay()
            torch.cuda.synchronize()
            s.record()
            for _ in range(args.replays):
                g.replay()
            e.record()
            torch.cuda.synchronize()
            ms = s.elapsed_time(e)
            total[k] += ms
            per_round[k].append(ms * 1e3 / args.replays)
    n = args.rounds * args.replays
    print(json.dumps({"card": card(), "envs": N, "batch": 4 * N, "mlp": [256, 256], "replays_per_agent": n,
                      "us_per_update": {k: total[k] * 1e3 / n for k in kinds},
                      "us_per_update_by_round": per_round}), flush=True)


if __name__ == "__main__":
    main()
