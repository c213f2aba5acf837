"""Bootstrapped DQN next to DQN at the same sizes, in one run: 512 SynthAtari envs (4x84x84 uint8), the Nature CNN
with a 512-wide head, H = 10 heads, batch 1024, a ring of 100 rows x 512 envs.

Prints one JSON line per algorithm: env-steps/s of collection (the captured collector step) and updates/s (the
captured update), each from CUDA events around whole epochs after two warm-up epochs, plus the card's name and power
limit.  Not part of bench.py.

    python scripts/bootstrapped_dqn_bench.py
"""
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
from torchrl_b200.algo import DQN, BootstrappedDQN  # noqa: E402
from torchrl_b200.collector import PixelVecCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import BaseReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402

N, H, STEPS, UPDATES, EPOCHS = 512, 10, 32, 16, 5
NET = dict(input_shape=(4, 84, 84), hidden_shapes=[[16, [8, 8], [4, 4], [0, 0]], [32, [4, 4], [2, 2], [0, 0]],
                                                   [64, [3, 3], [1, 1], [0, 0]]],
           append_hidden_shapes=[512], base_type=networks.CNNBase, activation_func=nn.ReLU)
dev = torch.device("cuda:0")


def card():
    name = torch.cuda.get_device_name(dev)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "unknown (%s)" % e
    return name, out


def build(kind):
    env, ev_env = get_vec_env("SynthAtari-v0", {}, N), get_vec_env("SynthAtari-v0", {}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=100 * N)
    common = dict(qlr=2.5e-4, optimizer_info={"eps": 0.01}, env=env, replay_buffer=buf, logger=NullLogger(),
                  discount=0.99, batch_size=2 * N, device=dev, save_dir=None, opt_times=UPDATES,
                  use_soft_update=False, target_hard_update_period=10000, num_epochs=10)
    if kind == "dqn":
        qf = networks.Net(output_shape=6, **NET)
        pf = policies.EpsilonGreedyDQNDiscretePolicy(qf=qf, start_epsilon=0.1, end_epsilon=0.1, decay_frames=1000000,
                                                     action_shape=6)
    else:
        qf = networks.BootstrappedNet(output_shape=6, head_num=H, **NET)
        pf = policies.BootstrappedDQNDiscretePolicy(qf=qf, head_num=H, action_shape=6)
    col = PixelVecCollector(env=env, eval_env=ev_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=STEPS * N,
                            max_episode_frames=50000)
    agent = DQN(qf=qf, pf=pf, collector=col, **common) if kind == "dqn" else \
        BootstrappedDQN(head_num=H, bernoulli_p=0.5, qf=qf, pf=pf, collector=col, **common)
    return agent, col


def timeit(agent, col):
    for e in range(2):
        agent.current_epoch = e
        col.train_one_epoch()
        agent.update_per_epoch()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tc, tu = [], []
    for _ in range(EPOCHS):
        ev[0].record(); col.rollout_no_sync(); ev[1].record(); agent.update_per_epoch(flush_infos=False); ev[2].record()
        torch.cuda.synchronize()
        tc.append(ev[0].elapsed_time(ev[1])); tu.append(ev[1].elapsed_time(ev[2]))
    return tc, tu


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    for kind in ("dqn", "bootstrapped_dqn"):
        agent, col = build(kind)
        tc, tu = timeit(agent, col)
        mc, mu = float(np.median(tc)), float(np.median(tu))
        print(json.dumps({"algo": kind, "envs": N, "heads": H if kind != "dqn" else 1, "batch": 2 * N,
                          "collect_env_steps_per_s": STEPS * N / mc * 1e3, "updates_per_s": UPDATES / mu * 1e3,
                          "ms_collect_%d_steps" % STEPS: tc, "ms_%d_updates" % UPDATES: tu,
                          "card": name, "power_limit_max_sm_clock": limit}), flush=True)
        del agent, col
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
