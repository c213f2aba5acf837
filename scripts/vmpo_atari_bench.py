"""Discrete V-MPO measurement (not the bench.py headline): VMPO with CategoricalDisPolicy on 512 SynthAtari envs
(4x84x84 uint8 frames, 6 actions), horizon 128, the ppo_pong.json CNN (conv 16/32/64 + 512, Tanh), minibatches of
4 * 512 rows, 10 optimisation passes per epoch -- the workload of scripts/ppo_atari_bench.py with V-MPO's actor step.

Device-timed with CUDA events around whole phases after two warm-up epochs: rollout, GAE and update (the per-epoch
top-half selection and the captured minibatch loop).  Then the V-MPO loss kernel alone on the k = B - B // 2 selected
rows, replayed from a captured CUDA graph, against the same minibatch actor step written in torch ops (sort of the
normalised advantages, softmax, torch's Categorical KL, the loss and its autograd wrt the logits), also replayed from
a captured graph.  Prints one JSON line with the card's name and power limit, read in the same run.

    python scripts/vmpo_atari_bench.py [--epochs 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torchrl_b200.networks as networks  # noqa: E402
import torchrl_b200.policies as policies  # noqa: E402
from ppo_atari_bench import PONG_CNN, card  # noqa: E402
from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.algo import VMPO  # noqa: E402
from torchrl_b200.collector import VecOnPolicyCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import OnPolicyReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402


def graph_us(fn, per_graph, reps):
    """Microseconds per call of fn, replayed from a captured CUDA graph of per_graph calls."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = ops.CapturedGraph(lambda: [fn() for _ in range(per_graph)])
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / (reps * per_graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=512)
    ap.add_argument("--horizon", type=int, default=128)
    ap.add_argument("--epochs", type=int, default=3)
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
    agent = VMPO(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, opt_epochs=10, alpha_eps=0.1, tau=0.95, shuffle=True, env=env,
                 replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, num_epochs=4880,
                 batch_size=4 * N, gae=True, device=dev, save_dir=None)
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
        agent.update_per_epoch(flush_infos=False)     # recomputes the advantages: one GAE is subtracted below
        ev[3].record()
        torch.cuda.synchronize()
        t_roll += ev[0].elapsed_time(ev[1])
        t_gae += ev[1].elapsed_time(ev[2])
        t_upd += ev[2].elapsed_time(ev[3]) - ev[1].elapsed_time(ev[2])
    n = args.epochs
    t_roll, t_gae, t_upd = t_roll / n, t_gae / n, t_upd / n
    # the minibatch actor step alone: B = 4 N rows, k = B - B // 2 selected, 6 actions
    B = 4 * N
    k = B - B // 2
    rs = np.random.RandomState(0)
    logits = torch.tensor(rs.randn(k, 6).astype(np.float32), device=dev, requires_grad=True)
    tlogits = torch.tensor(rs.randn(k, 6).astype(np.float32), device=dev)
    acts = torch.tensor(rs.randint(0, 6, k).astype(np.float32), device=dev)
    advs = torch.tensor(rs.randn(k).astype(np.float32), device=dev)
    stats = torch.tensor([[0.0, 1.0, 0.0, 0.0]], device=dev)
    pos = torch.zeros(1, dtype=torch.int32, device=dev)
    dual = torch.tensor([1.0, 0.1], device=dev, requires_grad=True)
    g_dual = torch.zeros(2, device=dev)
    info = torch.zeros(12, device=dev)
    scratch = ops.VMPOScratch(k, dev)
    g = torch.empty(k, 6, device=dev)
    kernel_us = graph_us(lambda: ops.vmpo_categorical_loss(logits.detach(), tlogits, acts, advs, stats, dual.detach(),
                                                           0.02, 0.1, False, scratch, g_dual, info, stats_pos=pos,
                                                           g_logits=g), 200, 10)
    full_advs = torch.tensor(rs.randn(B, 1).astype(np.float32), device=dev)
    full_logits = torch.tensor(rs.randn(B, 6).astype(np.float32), device=dev, requires_grad=True)
    full_t = torch.tensor(rs.randn(B, 6).astype(np.float32), device=dev)
    full_acts = torch.tensor(rs.randint(0, 6, B).astype(np.float32), device=dev)

    def torch_step():
        """The same actor step in torch ops, as the Gaussian path writes it: sort, gather, softmax, KL, backward."""
        advn = (full_advs - stats[0, 0]) / (stats[0, 1] + 1e-5)
        idx = torch.sort(advn.reshape(-1), dim=0, descending=True)[1][:k]
        z, zq, a, adv = full_logits[idx], full_t[idx], full_acts[idx], advn[idx]
        dis = torch.distributions.Categorical(torch.softmax(z, -1))
        tdis = torch.distributions.Categorical(torch.softmax(zq, -1))
        logp = dis.log_prob(a).unsqueeze(-1)
        kl = torch.distributions.kl.kl_divergence(dis, tdis).sum(-1, keepdim=True)
        eta, alpha = dual[0:1], dual[1:2]
        phis = torch.softmax(adv / eta.detach(), dim=0)
        eta_loss = eta * 0.02 + eta * torch.log(torch.mean(torch.exp(adv / eta)))
        alpha_loss = alpha * 0.1 - alpha * kl.detach().mean()
        policy_loss = (-phis * logp + alpha.detach() * kl).mean()
        (policy_loss + eta_loss.sum() + alpha_loss.sum()).backward()
    torch.distributions.Distribution.set_default_validate_args(False)   # argument checks sync with the host
    torch_us = graph_us(torch_step, 20, 20)
    name, power = card()
    frames = T * N
    print(json.dumps({
        "workload": "V-MPO CategoricalDisPolicy, SynthAtari-v0 4x84x84 uint8, ppo_pong.json CNN",
        "envs": N, "horizon": T, "batch": B, "selected": k, "opt_epochs": 10, "timed_epochs": n,
        "env_steps_per_s": frames / (t_roll + t_gae + t_upd) * 1e3,
        "rollout_env_steps_per_s": frames / t_roll * 1e3,
        "ms_rollout": t_roll, "ms_gae": t_gae, "ms_update": t_upd,
        "vmpo_loss_kernel_us_graph_replay": kernel_us,
        "torch_ops_actor_step_us_graph_replay": torch_us,
        "gpu": name, "power_limit": power,
        "not_measured": "per-kernel breakdown of rollout and update phases; the selection kernel alone; multi-GPU",
    }), flush=True)


if __name__ == "__main__":
    main()
