"""Throughput of the device CartPole: the bare env-step kernel, the on-policy collector (categorical MLP policy, captured
step graph) at N envs, and one REINFORCE epoch (collection + discounted returns + minibatch updates).  Prints one JSON
line.  Timings are CUDA-event or synchronised wall-clock measurements after a warm-up.

    python scripts/cartpole_bench.py --envs 4096 --steps 128
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torchrl_b200.networks as networks  # noqa: E402
import torchrl_b200.policies as policies  # noqa: E402
from torchrl_b200.algo import Reinforce  # noqa: E402
from torchrl_b200.collector import VecOnPolicyCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import OnPolicyReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402


def kernel_us(env, iters):
    """Mean time of one env-step launch (CUDA events over `iters` launches)."""
    act = (torch.arange(env.env_nums, device="cuda") % 2).float()
    for _ in range(20):
        env.launch_step(act)
        env.partial_reset(env.done)
    env.reset()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(iters):
        env.launch_step(act)
    ev1.record()
    torch.cuda.synchronize()
    return 1000.0 * ev0.elapsed_time(ev1) / iters


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=128, help="collector steps per epoch")
    p.add_argument("--epochs", type=int, default=10, help="timed epochs (after 3 warm-up epochs)")
    p.add_argument("--hidden", type=int, default=32)
    a = p.parse_args()
    dev = torch.device("cuda:0")
    N, T = a.envs, a.steps
    env = get_vec_env("CartPole-v1", {}, N, device=dev)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    t_kernel = kernel_us(get_vec_env("CartPole-v1", {}, N, device=dev), 2000)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    pf = policies.CategoricalDisPolicy(input_shape=4, output_shape=2, hidden_shapes=[a.hidden, a.hidden],
                                       append_hidden_shapes=[], base_type=networks.MLPBase,
                                       activation_func=torch.nn.Tanh)
    col = VecOnPolicyCollector(networks.ZeroNet(), env=env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=T * N,
                               max_episode_frames=1000)
    agent = Reinforce(pf=pf, plr=3e-3, entropy_coeff=0.001, env=env, replay_buffer=buf, collector=col,
                      logger=NullLogger(), discount=0.99, num_epochs=a.epochs, batch_size=T * N // 4, device=dev,
                      save_dir=None, shuffle=True)
    for _ in range(3):
        col.train_one_epoch()
        agent.update_per_epoch()
    torch.cuda.synchronize()
    t_col = t_upd = 0.0
    for _ in range(a.epochs):
        t0 = time.perf_counter()
        col.rollout_no_sync()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        agent.update_per_epoch(flush_infos=False)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        t_col += t1 - t0
        t_upd += t2 - t1
    props = torch.cuda.get_device_properties(dev)
    print(json.dumps({
        "gpu": props.name, "envs": N, "steps_per_epoch": T, "hidden": a.hidden,
        "cartpole_step_kernel_us": round(t_kernel, 2),
        "collector_env_steps_per_s": round(a.epochs * T * N / t_col),
        "reinforce_epoch_ms": round(1000 * (t_col + t_upd) / a.epochs, 2),
        "reinforce_update_ms": round(1000 * t_upd / a.epochs, 2),
        "minibatches_per_epoch": 4,
    }))


if __name__ == "__main__":
    main()
