"""Throughput of the device classic-control envs (CartPole-v1, Pendulum-v1, Acrobot-v1, MountainCar-v0,
MountainCarContinuous-v0): each bare env-step kernel at N = 2^20 (CUDA events over a captured graph of many launches, bytes per env from the operand shapes, bandwidth against
the H100 SXM's 3.35 TB/s), and the captured DQN collector step (Q-network forward, epsilon-greedy, env step, finalize,
the env's own reset, ring advance) at a few thousand Acrobot envs.  Prints the card and its power limit and one JSON
line.

    python scripts/classic_control_bench.py --kernel-envs 1048576 --envs 4096
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torchrl_b200.networks as networks  # noqa: E402
import torchrl_b200.policies as policies  # noqa: E402
from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.collector import VecCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import BaseReplayBuffer  # noqa: E402
from scripts.pendulum_bench import HBM_BYTES_PER_S, card  # noqa: E402


def bytes_per_env(P, D):
    """Per env and step: phys (P fp64) + action (fp32) + elapsed (int32) read; phys + obs (D fp32) + reward (fp32) +
    done + time_limit (uint8) + elapsed written.  P = 0 (CartPole): the state is the fp32 observation, read too."""
    state = P * 8 if P else D * 4
    return (state + 4 + 4) + (P * 8 + D * 4 + 4 + 1 + 1 + 4)


def kernel_us(env_id, N, launches, reps, actions):
    """Mean time of one step launch over N envs, from a captured graph of `launches` launches."""
    env = get_vec_env(env_id, {}, N)
    env.reset()
    for _ in range(10):
        env.launch_step(actions)
    g = ops.CapturedGraph(lambda: [env.launch_step(actions) for _ in range(launches)])
    g.replay()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        ev0.record()
        g.replay()
        ev1.record()
        torch.cuda.synchronize()
        times.append(1000.0 * ev0.elapsed_time(ev1) / launches)
    return float(np.median(times))


def dqn_collector_rate(N, T, epochs, hidden):
    """Env steps per second of the captured DQN collector step on Acrobot-v1 (device events over whole epochs)."""
    env = get_vec_env("Acrobot-v1", {}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=4 * T * N, time_limit_filter=True)
    qf = networks.Net(input_shape=(6,), output_shape=3, hidden_shapes=[hidden, hidden], append_hidden_shapes=[],
                      base_type=networks.MLPBase, activation_func=torch.nn.ReLU)
    pf = policies.EpsilonGreedyDQNDiscretePolicy(qf=qf, start_epsilon=1.0, end_epsilon=0.05, decay_frames=10 * T * N,
                                                 action_shape=3)
    col = VecCollector(env=env, pf=pf, replay_buffer=buf, device=torch.device("cuda:0"), epoch_frames=T * N,
                       max_episode_frames=1000)
    for _ in range(2):
        col.train_one_epoch()
    assert False in col._graphs
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(epochs):
        col.rollout_no_sync()
    ev1.record()
    torch.cuda.synchronize()
    return epochs * T * N / (ev0.elapsed_time(ev1) / 1000.0), col._graphs[False].launches


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--kernel-envs", type=int, default=1 << 20)
    p.add_argument("--launches", type=int, default=200)
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=100, help="collector steps per epoch")
    p.add_argument("--epochs", type=int, default=10, help="timed epochs (after 2 warm-up epochs)")
    p.add_argument("--hidden", type=int, default=128)
    a = p.parse_args()
    name, limit = card()
    print("card: %s, power limit: %s W" % (name, "unknown" if limit is None else "%.0f" % limit), flush=True)
    N = a.kernel_envs
    binary = (torch.arange(N, device="cuda") % 2).float()
    discrete = (torch.arange(N, device="cuda") % 3).float()
    continuous = torch.linspace(-1, 1, N, device="cuda")
    out = {"gpu": name, "power_limit_w": limit, "kernel_envs": N}
    for key, env_id, P, D, act in (("cartpole", "CartPole-v1", 0, 4, binary),
                                   ("pendulum", "Pendulum-v1", 2, 3, continuous),
                                   ("acrobot", "Acrobot-v1", 4, 6, discrete),
                                   ("mountain_car", "MountainCar-v0", 2, 2, discrete),
                                   ("mountain_car_continuous", "MountainCarContinuous-v0", 2, 2, continuous)):
        us = kernel_us(env_id, N, a.launches, 5, act)
        bw = bytes_per_env(P, D) * N / (us * 1e-6)
        out.update({key + "_step_kernel_us": round(us, 2), key + "_bytes_per_env": bytes_per_env(P, D),
                    key + "_achieved_tb_per_s": round(bw / 1e12, 3),
                    key + "_fraction_of_3_35_tb_per_s": round(bw / HBM_BYTES_PER_S, 3)})
    rate, launches = dqn_collector_rate(a.envs, a.steps, a.epochs, a.hidden)
    out.update({"envs": a.envs, "hidden": a.hidden, "dqn_acrobot_collector_env_steps_per_s": round(rate),
                "dqn_collector_step_library_launches": launches})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
