"""Discrete TRPO measurement (not the bench.py headline): TRPO with CategoricalDisPolicy on SynthAtari (4x84x84 uint8
frames, 6 actions), the ppo_pong.json CNN (conv 16/32/64 + 512, Tanh), one natural-gradient step per epoch on the
whole rollout (default 128 envs x horizon 64 = 8192 rows), 10 CG iterations, 2 value sweeps of 4 * envs rows.

Device-timed with CUDA events after two warm-up epochs: the rollout, the whole update, and inside it the surrogate
gradient, one Fisher-vector product, the conjugate-gradient solve, the line search and the value sweeps (each phase is
bracketed by events and a synchronisation, so the phases add up to slightly more than the unbracketed update).  Then
each new kernel's time per launch, replayed from a captured CUDA graph, at the workload's sizes.  Prints one JSON
line with torch.cuda.max_memory_allocated and the card's name and power limit, read in the same run.

    python scripts/trpo_atari_bench.py [--envs 128 --horizon 64 --epochs 3]
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
from vmpo_atari_bench import graph_us  # noqa: E402
from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.algo import TRPO  # noqa: E402
from torchrl_b200.collector import VecOnPolicyCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import OnPolicyReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402


class PhaseTimer:
    """Wraps agent methods so that every call is bracketed by CUDA events; ms per phase accumulate in `ms`."""

    def __init__(self):
        self.ms, self.calls = {}, {}
        self.active = False

    def wrap(self, owner, name, phase):
        fn = getattr(owner, name)

        def timed(*a, **kw):
            if not self.active:
                return fn(*a, **kw)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*a, **kw)
            e.record()
            torch.cuda.synchronize()
            self.ms[phase] = self.ms.get(phase, 0.0) + s.elapsed_time(e)
            self.calls[phase] = self.calls.get(phase, 0) + 1
            return out
        setattr(owner, name, timed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=128)
    ap.add_argument("--horizon", type=int, default=64)
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
    agent = TRPO(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, max_kl=0.01, cg_damping=0.1, cg_iters=10, residual_tol=1e-10,
                 entropy_coeff=0.01, v_opt_times=2, tau=0.95, shuffle=True, env=env, replay_buffer=buf, collector=col,
                 logger=NullLogger(), discount=0.99, num_epochs=4880, batch_size=4 * N, gae=True, device=dev,
                 save_dir=None)
    timer = PhaseTimer()
    timer.wrap(agent._head, "trpo_actor", "surrogate_gradient")
    timer.wrap(agent._head, "trpo_score", "candidate")
    timer.wrap(agent, "_fvp", "fisher_vector_product")
    timer.wrap(agent, "_conjugate_gradient", "conjugate_gradient")
    timer.wrap(agent, "_linesearch", "line_search")
    timer.wrap(agent, "_minibatch_epoch", "value_sweeps")
    for e in range(2):                                 # warm-up: graph captures, cuDNN algorithm choice
        agent.current_epoch = e
        col.train_one_epoch()
        agent.update_per_epoch()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_roll = t_upd = 0.0
    timer.active = True
    for e in range(args.epochs):
        agent.current_epoch = 2 + e
        ev[0].record()
        col.rollout_no_sync()
        ev[1].record()
        agent.update_per_epoch(flush_infos=False)
        ev[2].record()
        torch.cuda.synchronize()
        t_roll += ev[0].elapsed_time(ev[1])
        t_upd += ev[1].elapsed_time(ev[2])
    timer.active = False
    peak = torch.cuda.max_memory_allocated()
    n = args.epochs
    t_roll, t_upd = t_roll / n, t_upd / n
    phases = {k: v / n for k, v in timer.ms.items()}
    # a CG iteration's products are inside the CG phase; one product alone, averaged over every product timed
    phases["fisher_vector_product"] = timer.ms["fisher_vector_product"] / timer.calls["fisher_vector_product"]
    # each new kernel per launch at the workload's sizes (M = T * N rows, 6 actions; the first conv's activations)
    M = T * N
    rs = np.random.RandomState(0)
    z = torch.tensor(rs.randn(M, 6).astype(np.float32), device=dev)
    t6 = torch.tensor(rs.randn(M, 6).astype(np.float32), device=dev)
    g6 = torch.empty_like(z)
    acts = torch.tensor(rs.randint(0, 6, M).astype(np.float32), device=dev)
    advn = torch.tensor(rs.randn(M).astype(np.float32), device=dev)
    old = ops.categorical_log_prob(z, acts)
    sc = ops.SurrogateScratch(M, dev)
    out = torch.empty(1, device=dev)
    fisher_us = graph_us(lambda: ops.categorical_fisher_vp(z, t6, 1.0 / M, out=g6), 50, 10)
    surrogate_us = graph_us(lambda: ops.categorical_surrogate(z, acts, old, advn, sc, out=out), 50, 10)
    c1 = (M, PONG_CNN[0][0], 20, 20)
    tc = torch.randn(c1, device=dev)
    yc = torch.tanh(torch.randn(c1, device=dev))
    db = torch.randn(c1[1], device=dev)
    tba_us = graph_us(lambda: ops.tangent_bias_act(tc, db, yc, 1), 10, 10)
    tba_gbs = 3 * tc.numel() * 4 / (tba_us * 1e-6) / 1e9
    del tc, yc
    name, power = card()
    frames = T * N
    print(json.dumps({
        "workload": "TRPO CategoricalDisPolicy, SynthAtari-v0 4x84x84 uint8, ppo_pong.json CNN (Tanh)",
        "envs": N, "horizon": T, "rows_per_policy_step": frames, "cg_iters": 10, "v_opt_times": 2,
        "timed_epochs": n,
        "env_steps_per_s": frames / (t_roll + t_upd) * 1e3,
        "ms_rollout": t_roll, "ms_update": t_upd,
        "ms_per_epoch": {k: phases[k] for k in ("surrogate_gradient", "conjugate_gradient", "line_search",
                                                 "value_sweeps")},
        "ms_one_fisher_vector_product": phases["fisher_vector_product"],
        "line_search_candidates_per_epoch": timer.calls.get("candidate", 0) / n,
        "fisher_vp_kernel_us": fisher_us, "surrogate_kernel_us": surrogate_us,
        "tangent_bias_act_us_first_conv": tba_us, "tangent_bias_act_first_conv_shape": list(c1),
        "tangent_bias_act_effective_GBps": tba_gbs,
        "max_memory_allocated_GiB": peak / 2 ** 30,
        "gpu": name, "power_limit": power,
        "not_measured": "multi-GPU; the phases' launch overheads separately from their kernels",
    }), flush=True)


if __name__ == "__main__":
    main()
