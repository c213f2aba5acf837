"""Prioritised replay on the device: the sampler's time over ring sizes and batch sizes, and updates/s of the agents
with uniform vs prioritised replay.  Prints one JSON line per measurement, first the card and its power limit.

    python scripts/per_bench.py            # everything (about a minute on one GPU)
    python scripts/per_bench.py sampler    # only the sampler table

Sampler: CUDA events around a captured graph of REPS launches (kernel time plus launch gaps), per call.  Bytes are
what the two passes move at least: the priorities read (4 B/row) and the in-chunk prefix written (8 B/row) by the chunk
pass, and one 8 B prefix load per binary-search probe of each draw; the HBM bound divides them by 3.35 TB/s.
Updates/s: CUDA events around whole `update_per_epoch` calls after two warm epochs (graphs captured).
QR-DQN: the eager prioritised loop of earlier versions (per update: host uniforms, an eager update body, the priority
write and a read-back of the info row) restated here, alternated with the captured epoch on the same agent.
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
from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.algo import QRDQN, TD3, TwinSACQ  # noqa: E402
from torchrl_b200.collector import PixelVecCollector, VecCollector  # noqa: E402
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.replay_buffers import BaseReplayBuffer, PrioritizedReplayBuffer  # noqa: E402
from torchrl_b200.utils import NullLogger  # noqa: E402

HBM = 3.35e12
REPS = 50


def emit(d):
    print(json.dumps(d), flush=True)


def card():
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                          # noqa: BLE001
        limit = "unknown (%r)" % e
    return {"card": torch.cuda.get_device_name(0), "power_limit": limit}


def time_graph(fn):
    fn()
    torch.cuda.synchronize()
    g = ops.CapturedGraph(lambda: [fn() for _ in range(REPS)])
    g.replay()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / REPS)
    return best


def sampler_table():
    rs = np.random.RandomState(0)
    for lg in (12, 14, 16, 18, 20, 22, 24):
        rows = 1 << lg
        prio = torch.from_numpy((rs.rand(rows) + 0.01).astype(np.float32)).cuda()
        sc = torch.empty(ops.per_scratch_doubles(rows), dtype=torch.float64, device="cuda")
        size = torch.tensor([rows], dtype=torch.int32, device="cuda")
        pos = torch.zeros(1, dtype=torch.int32, device="cuda")
        for b in (64, 256, 1024):
            u = torch.rand(b, dtype=torch.float64, device="cuda")
            idx = torch.empty(b, dtype=torch.int64, device="cuda")
            w = torch.empty(b, dtype=torch.float32, device="cuda")
            us = time_graph(lambda: ops.per_sample_rows(prio, size, u, pos, b, 0.4, sc, idx, w))
            probes = int(np.ceil(np.log2(max(2, min(rows, 4096))))) + int(np.ceil(np.log2(max(2, rows // 4096))))
            nbytes = 12 * rows + 8 * b * probes
            row = {"kind": "sampler_rows", "rows": rows, "b": b, "us": round(us, 2), "bytes": nbytes,
                   "hbm_bound_us": round(nbytes / HBM * 1e6, 2)}
            if rows <= 4096:
                row["one_cta_us"] = round(time_graph(lambda: ops.per_sample(prio, rows, u, 0.4, idx, w)), 2)
            emit(row)


def updates_per_s(agent, col, epochs=3):
    for e in range(2):
        agent.current_epoch = e
        col.train_one_epoch()
        agent.update_per_epoch()
    torch.cuda.synchronize()
    ms = 0.0
    for _ in range(epochs):
        col.rollout_no_sync()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        agent.update_per_epoch(flush_infos=False)
        b.record()
        torch.cuda.synchronize()
        ms += a.elapsed_time(b)
    return agent.opt_times * epochs / ms * 1e3


def td3_pendulum(per):
    N = 16
    env, ev = get_vec_env("Pendulum-v1", {"obs_norm": False}, N), get_vec_env("Pendulum-v1", {"obs_norm": False}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    cls = PrioritizedReplayBuffer if per else BaseReplayBuffer
    buf = cls(env_nums=N, max_replay_buffer_size=100000)
    net = dict(hidden_shapes=[256, 256], append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=nn.ReLU)
    pf = policies.FixGuassianContPolicy(input_shape=3, output_shape=1, tanh_action=True, norm_std_explore=0.1, **net)
    qf1, qf2 = (networks.QNet(input_shape=4, output_shape=1, **net) for _ in range(2))
    col = VecCollector(env=env, eval_env=ev, pf=pf, replay_buffer=buf, device="cuda", epoch_frames=1600,
                       max_episode_frames=200)
    agent = TD3(pf=pf, qf1=qf1, qf2=qf2, plr=1e-3, qlr=1e-3, env=env, replay_buffer=buf, collector=col,
                logger=NullLogger(), discount=0.99, batch_size=256, device="cuda", save_dir=None, tau=0.005,
                opt_times=200, num_epochs=10)
    for _ in range(4):                                       # fill past 4096 rows: 6,250 rows in all
        col.train_one_epoch()
    return updates_per_s(agent, col)


def twin_sac_q_config3(per):
    N = 1024
    env = get_vec_env("SynthAnt-v0", {"reward_scale": 1, "obs_norm": False}, N)
    ev = get_vec_env("SynthAnt-v0", {"obs_norm": False}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    cls = PrioritizedReplayBuffer if per else BaseReplayBuffer
    buf = cls(env_nums=N, max_replay_buffer_size=int(1e6))
    net = dict(hidden_shapes=[256, 256], append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=nn.ReLU)
    pf = policies.GuassianContPolicy(input_shape=111, output_shape=16, tanh_action=True, **net)
    qf1, qf2 = (networks.QNet(input_shape=119, output_shape=1, **net) for _ in range(2))
    col = VecCollector(env=env, eval_env=ev, pf=pf, replay_buffer=buf, device="cuda", epoch_frames=64 * N,
                       max_episode_frames=999)
    agent = TwinSACQ(pf=pf, qf1=qf1, qf2=qf2, plr=3e-4, qlr=3e-4, policy_std_reg_weight=0, policy_mean_reg_weight=0,
                     env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99,
                     batch_size=4 * N, device="cuda", save_dir=None, tau=0.005, opt_times=64, num_epochs=10)
    return updates_per_s(agent, col)


def eager_prioritised_epoch(agent):
    """The per-update host loop the captured prioritised epoch replaced."""
    rb = agent.replay_buffer
    infos = []
    for _ in range(agent.opt_times):
        batch = rb.random_batch(agent.batch_size, agent.sample_key)
        agent._batch = lambda: batch                        # the body reads this batch instead of the gather
        agent.training_update_num += 1
        variant = agent._variant()
        try:
            agent._update_body(variant)
        finally:
            del agent._batch
        agent._maybe_hard_update()
        rb.update_priorities(batch["indices"], agent._eager_td)
        infos.append(agent._decode_info(agent._ub["info"][0].cpu().numpy(), variant))
    return infos


def qr_dqn_config4():
    N, Q = 512, 200
    env = get_vec_env("SynthAtari-v0", {}, N)
    ev = get_vec_env("SynthAtari-v0", {}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    buf = PrioritizedReplayBuffer(env_nums=N, max_replay_buffer_size=100 * N)
    qf = networks.Net(input_shape=(4, 84, 84), output_shape=6 * Q,
                      hidden_shapes=[[16, [8, 8], [4, 4], [0, 0]], [32, [4, 4], [2, 2], [0, 0]], [64, [3, 3], [1, 1], [0, 0]]],
                      append_hidden_shapes=[512], base_type=networks.CNNBase, activation_func=nn.ReLU)
    pf = policies.EpsilonGreedyQRDQNDiscretePolicy(quantile_num=Q, qf=qf, start_epsilon=0.1, end_epsilon=0.1,
                                                   decay_frames=1000000, action_shape=6)
    col = PixelVecCollector(env=env, eval_env=ev, pf=pf, replay_buffer=buf, device="cuda", epoch_frames=32 * N,
                            max_episode_frames=50000)
    agent = QRDQN(quantile_num=Q, qf=qf, pf=pf, qlr=5e-5, optimizer_info={"eps": 0.0003125}, env=env,
                  replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, batch_size=2 * N,
                  device="cuda", save_dir=None, opt_times=16, use_soft_update=False, target_hard_update_period=10000,
                  num_epochs=10)
    for e in range(2):
        col.train_one_epoch()
        agent.update_per_epoch()
    # the eager loop writes its |TD| into a buffer of its own, as the old loop allocated one per update
    agent._eager_td = torch.empty(agent.batch_size, device="cuda")
    real_td = agent._td
    res = {"eager": [], "captured": []}
    for _ in range(3):
        for kind in ("eager", "captured"):
            col.rollout_no_sync()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            if kind == "eager":
                agent._td = agent._eager_td
                agent._ub["per"] = False                     # no device sampling or priority write in the body
                try:
                    eager_prioritised_epoch(agent)
                finally:
                    agent._td = real_td
                    agent._ub["per"] = True
            else:
                agent.update_per_epoch(flush_infos=True)
            b.record()
            torch.cuda.synchronize()
            res[kind].append(agent.opt_times / a.elapsed_time(b) * 1e3)
    return {k: round(float(np.median(v)), 1) for k, v in res.items()}


def main():
    what = sys.argv[1:] or ["sampler", "agents"]
    emit(card())
    if "sampler" in what:
        sampler_table()
    if "agents" in what:
        emit({"kind": "td3_pendulum_16_envs_6250_rows", "uniform_updates_per_s": round(td3_pendulum(False), 1),
              "prioritised_updates_per_s": round(td3_pendulum(True), 1)})
        emit({"kind": "twin_sac_q_config3_1024_envs", "uniform_updates_per_s": round(twin_sac_q_config3(False), 1),
              "prioritised_updates_per_s": round(twin_sac_q_config3(True), 1)})
        emit(dict({"kind": "qr_dqn_config4_updates_per_s"}, **qr_dqn_config4()))


if __name__ == "__main__":
    main()
