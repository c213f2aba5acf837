"""Discrete on-policy measurement (not the bench.py headline): PPO with CategoricalDisPolicy on 512 SynthAtari envs
(4x84x84 uint8 frames, 6 actions), horizon 128, the ppo_pong.json CNN (conv 16/32/64 + 512, Tanh), minibatches of
4 * 512 rows, 10 optimisation passes per epoch.

Device-timed with CUDA events around whole phases after two warm-up epochs: rollout (collector step graphs), GAE
(bootstrap value + scan) and update (old log-probs + the captured minibatch loop).  Also the categorical actor loss
kernel alone at the minibatch shape: many launches replayed from a captured CUDA graph (kernel time plus the graph's
launch gap), and the same launches issued one Python call at a time (per-call time including dispatch).  Prints one
JSON line with the card's name and power limit, read in the same run.

    python scripts/ppo_atari_bench.py [--epochs 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchrl_b200.networks as networks  # noqa: E402
import torchrl_b200.policies as policies  # noqa: E402
from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.algo import PPO  # noqa: E402
from torchrl_b200.collector import VecOnPolicyCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import OnPolicyReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402

PONG_CNN = [[16, [8, 8], [4, 4], [0, 0]], [32, [4, 4], [2, 2], [0, 0]], [64, [3, 3], [1, 1], [0, 0]]]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:                                  # noqa: BLE001
        return torch.cuda.get_device_name(0), "not measured"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=512)
    ap.add_argument("--horizon", type=int, default=128)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--loss-launches", type=int, default=2000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda:0")
    N, T = args.envs, args.horizon
    env = get_vec_env("SynthAtari-v0", {}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    net = dict(input_shape=(4, 84, 84), hidden_shapes=PONG_CNN, append_hidden_shapes=[512], base_type=networks.CNNBase,
               activation_func=torch.nn.Tanh)
    pf = policies.CategoricalDisPolicy(output_shape=6, **net)
    vf = networks.Net(output_shape=1, **net)
    col = VecOnPolicyCollector(vf, env=env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=T * N,
                               max_episode_frames=128, eval_episodes=1)
    agent = PPO(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, clip_para=0.1, opt_epochs=10, tau=0.95, shuffle=True,
                entropy_coeff=0.01, env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99,
                num_epochs=4880, batch_size=4 * N, gae=True, device=dev, save_dir=None)
    for e in range(2):                                 # warm-up: graph captures, cuDNN algorithm choice
        agent.current_epoch = e
        col.train_one_epoch()
        agent.update_per_epoch()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t_roll = t_gae = t_upd = 0.0
    for e in range(args.epochs):
        agent.current_epoch = 2 + e
        ev[0].record()
        col.rollout_no_sync()
        ev[1].record()
        agent.process_epoch_samples()
        ev[2].record()
        # update_per_epoch recomputes the (cheap, in-place) advantages first; its time is counted in GAE above and
        # again here, so the update phase is the whole update_per_epoch minus one GAE
        agent.update_per_epoch(flush_infos=False)
        ev[3].record()
        torch.cuda.synchronize()
        t_roll += ev[0].elapsed_time(ev[1])
        t_gae += ev[1].elapsed_time(ev[2])
        t_upd += ev[2].elapsed_time(ev[3]) - ev[1].elapsed_time(ev[2])
    n = args.epochs
    t_roll, t_gae, t_upd = t_roll / n, t_gae / n, t_upd / n
    # the categorical loss kernel alone at the minibatch shape (B = 4 N rows, 6 actions)
    B = 4 * N
    rs = np.random.RandomState(0)
    logits = torch.tensor(rs.randn(B, 6).astype(np.float32), device=dev)
    acts = torch.tensor(rs.randint(0, 6, B).astype(np.float32), device=dev)
    advs = torch.tensor(rs.randn(B).astype(np.float32), device=dev)
    old = torch.tensor(rs.randn(B).astype(np.float32) - 1.8, device=dev)
    stats = torch.tensor([[0.0, 1.0, 0.0, 0.0]], device=dev)
    pos = torch.zeros(1, dtype=torch.int32, device=dev)
    scratch = ops.LossScratch(B, 6, dev, categorical=True)
    g = torch.empty_like(logits)
    info = torch.zeros(16, device=dev)

    def launches(n):
        for _ in range(n):
            ops.ppo_categorical_actor_loss(logits, acts, old, advs, stats, 0.1, 0.01, scratch, g_logits=g, info=info,
                                           stats_pos=pos)
    # the launches are replayed from a captured CUDA graph so that the Python / ctypes dispatch of each call (about as
    # long as this small kernel) is not part of the figure; what remains is kernel time plus the graph's node-to-node
    # launch gap
    per_graph = 200
    launches(50)                                       # warm-up outside the graph
    torch.cuda.synchronize()
    graph = ops.CapturedGraph(lambda: launches(per_graph))
    graph.replay()
    torch.cuda.synchronize()
    reps = max(1, args.loss_launches // per_graph)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        graph.replay()
    e.record()
    torch.cuda.synchronize()
    loss_us = s.elapsed_time(e) * 1e3 / (reps * per_graph)
    # the same launches issued one Python call at a time (what an eager caller pays per call)
    s.record()
    launches(args.loss_launches)
    e.record()
    torch.cuda.synchronize()
    call_us = s.elapsed_time(e) * 1e3 / args.loss_launches
    name, power = card()
    frames = T * N
    print(json.dumps({
        "workload": "PPO CategoricalDisPolicy, SynthAtari-v0 4x84x84 uint8, ppo_pong.json CNN",
        "envs": N, "horizon": T, "batch": B, "opt_epochs": 10, "timed_epochs": n,
        "env_steps_per_s": frames / (t_roll + t_gae + t_upd) * 1e3,
        "rollout_env_steps_per_s": frames / t_roll * 1e3,
        "ms_rollout": t_roll, "ms_gae": t_gae, "ms_update": t_upd,
        "categorical_loss_kernel_us_graph_replay": loss_us, "categorical_loss_launches": reps * per_graph,
        "categorical_loss_us_per_python_call": call_us,
        "gpu": name, "power_limit": power,
        "not_measured": "per-kernel breakdown of rollout and update phases; multi-GPU",
    }), flush=True)


if __name__ == "__main__":
    main()
