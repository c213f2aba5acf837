"""Throughput of the device Pendulum-v1 under TD3: the captured TD3 collector step plus the TD3 update at a few thousand
envs (scripts/classic_control_bench.py times the bare env-step kernel).  Prints the card and its power limit and one
JSON line.

    python scripts/pendulum_bench.py --envs 4096
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torchrl_b200.networks as networks  # noqa: E402
import torchrl_b200.policies as policies  # noqa: E402
from torchrl_b200.algo import TD3  # noqa: E402
from torchrl_b200.collector import VecCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import BaseReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    """(name, power limit in W or None): the limit is read with nvidia-smi's query mode when it is available."""
    name = torch.cuda.get_device_properties(0).name
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:                                   # noqa: BLE001 -- the number is reported as unknown
        return name, None


def td3_rate(N, T, epochs, hidden, opt_times, batch):
    env = get_vec_env("Pendulum-v1", {}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=8 * T * N, time_limit_filter=False)
    net = dict(hidden_shapes=[hidden, hidden], append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=torch.nn.ReLU)
    pf = policies.FixGuassianContPolicy(input_shape=3, output_shape=1, tanh_action=True, norm_std_explore=0.1, **net)
    qf1 = networks.QNet(input_shape=4, output_shape=1, **net)
    qf2 = networks.QNet(input_shape=4, output_shape=1, **net)
    col = VecCollector(env=env, pf=pf, replay_buffer=buf, device=torch.device("cuda:0"), epoch_frames=T * N,
                       max_episode_frames=200)
    agent = TD3(pf=pf, qf1=qf1, qf2=qf2, plr=1e-3, qlr=1e-3, env=env, replay_buffer=buf, collector=col,
                logger=NullLogger(), discount=0.99, batch_size=batch, device=torch.device("cuda:0"), save_dir=None,
                tau=0.005, use_soft_update=True, opt_times=opt_times, pretrain_epochs=1, num_epochs=epochs)
    agent.pretrain()
    for _ in range(3):
        col.train_one_epoch()
        agent.update_per_epoch()
    torch.cuda.synchronize()
    t_col = t_upd = 0.0
    for _ in range(epochs):
        t0 = time.perf_counter()
        col.rollout_no_sync()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        agent.update_per_epoch(flush_infos=False)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        t_col += t1 - t0
        t_upd += t2 - t1
    return epochs * T * N / t_col, epochs * T * N / (t_col + t_upd), 1e3 * t_upd / (epochs * opt_times)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=50, help="collector steps per epoch")
    p.add_argument("--epochs", type=int, default=5, help="timed epochs (after 3 warm-up epochs)")
    p.add_argument("--hidden", type=int, default=256)
    p.add_argument("--opt-times", type=int, default=50, help="TD3 updates per epoch")
    p.add_argument("--batch", type=int, default=4096)
    a = p.parse_args()
    name, limit = card()
    print("card: %s, power limit: %s W" % (name, "unknown" if limit is None else "%.0f" % limit), flush=True)
    col_rate, epoch_rate, upd_ms = td3_rate(a.envs, a.steps, a.epochs, a.hidden, a.opt_times, a.batch)
    print(json.dumps({
        "gpu": name, "power_limit_w": limit, "envs": a.envs, "hidden": a.hidden, "steps_per_epoch": a.steps, "opt_times": a.opt_times, "batch": a.batch,
        "td3_collector_env_steps_per_s": round(col_rate), "td3_epoch_env_steps_per_s": round(epoch_rate),
        "td3_update_ms": round(upd_ms, 3),
    }))


if __name__ == "__main__":
    main()
