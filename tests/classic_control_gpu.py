"""What the GPU tests of the self-resetting classic-control envs (Pendulum-v1, Acrobot-v1, MountainCar-v0,
MountainCarContinuous-v0) share: the tolerance checks, one kernel step from given fp64 states, a stub policy that runs
the scripted controller inside the collector's step, and the off- and on-policy agents of the one-epoch tests.  Each
env's test module holds a `Case` naming its oracle, kernel and controller."""
from dataclasses import dataclass
from typing import Callable

import numpy as np


@dataclass
class Case:
    env_id: str
    P: int                                  # fp64 state width
    D: int                                  # observation width
    step: Callable                          # oracle step(phys, actions, elapsed, reward_scale=...) -> 6-tuple
    reset_phys: Callable                    # oracle reset_phys(seeds, episodes)
    observe: Callable                       # oracle observe(phys)
    controller: Callable                    # torch: raw-or-normalised obs (N, D) -> actions (N,) float32
    ops_step: Callable                      # ops.<env>_step(phys, obs, actions, elapsed, ...) with trailing extras
    extra: tuple = ()                       # trailing arguments of ops_step (MountainCar's `continuous`)
    near_goal: Callable = None              # oracle states whose done flag may differ by rounding (or None)


def check_phys(got, want, ulps):
    """|got - want| <= ulps fp64 ulps of max(|want|, 1), per component; returns the largest error in those ulps."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    unit = np.spacing(np.maximum(np.abs(want), 1.0))
    err = np.abs(got - want) / unit
    assert np.all(err <= ulps), (np.max(err), np.unravel_index(np.argmax(err), err.shape))
    return float(np.max(err)) if err.size else 0.0


def check_obs(got, want):
    """Equal, or one fp32 ulp apart (the fp64 values on either side of a rounding boundary)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    ulp = np.spacing(np.abs(want)).astype(np.float64)
    diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert np.all(diff <= np.maximum(ulp, 1e-45)), np.max(diff)


def step_kernel(case, phys, actions, elapsed, reward_scale=1.0, max_steps=None, obs=None):
    """One launch of the case's step kernel from fp64 states; returns host copies of (phys, obs, reward, done,
    time_limit, elapsed, action_error, any_reset)."""
    import torch
    N = phys.shape[0]
    dev = "cuda"
    ph = torch.as_tensor(phys, dtype=torch.float64, device=dev).contiguous()
    ob = (torch.zeros(N, case.D, device=dev) if obs is None
          else torch.as_tensor(obs, dtype=torch.float32, device=dev).contiguous())
    el = torch.as_tensor(elapsed, dtype=torch.int32, device=dev).contiguous()
    reward, done = torch.zeros(N, device=dev), torch.zeros(N, dtype=torch.uint8, device=dev)
    tl, err = torch.zeros(N, dtype=torch.uint8, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    ticket, any_reset = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)
    case.ops_step(ph, ob, torch.as_tensor(actions, dtype=torch.float32, device=dev).contiguous(), el, None, reward, done,
                  tl, err, None, None, None, None, None, ticket, any_reset, None, reward_scale, max_steps or (1 << 30),
                  1 << 30, False, *case.extra)
    return (ph.cpu().numpy(), ob.cpu().numpy(), reward.cpu().numpy(), done.cpu().numpy().astype(bool),
            tl.cpu().numpy().astype(bool), el.cpu().numpy(), int(err.item()), any_reset.cpu().numpy())


class ScriptedPolicy:
    """A policy stub for the collectors: the scripted controller on the observation the collector holds, written by
    torch ops (so the collector's captured step graph captures it too)."""

    def __init__(self, controller):
        self.controller = controller

    def act_only(self, ob, eps=None, action_out=None, nan_flag=None):
        action_out.copy_(self.controller(ob).reshape(action_out.shape))

    def eval_act(self, ob):
        return self.controller(ob)

    def to(self, device):
        return self


def collector(case, use_graph, quirks, obs_norm, N=24, T=48, seed=3, max_frames=10000, env_param=None):
    import torch
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer
    env = get_vec_env(case.env_id, dict(env_param or {}, obs_norm=obs_norm), N)
    env.seed(seed)
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=False)
    col = VecCollector(env=env, pf=ScriptedPolicy(case.controller), replay_buffer=buf, device=torch.device("cuda:0"),
                       epoch_frames=T * N, max_episode_frames=max_frames, use_cuda_graph=use_graph,
                       reference_quirks=quirks)
    return col, buf, env


def collector_graph_equals_eager(case, quirks, obs_norm, epochs=3, **kw):
    """Epochs with the captured step and with eager steps store bit-identical rows and leave the same env state;
    returns the graph run's rows."""
    import torch
    runs = []
    for use_graph in (False, True):
        col, buf, env = collector(case, use_graph, quirks, obs_norm, **kw)
        rows = []
        for _ in range(epochs):
            col.train_one_epoch()
            rows.append({k: getattr(buf, "_" + k).clone() for k in ("obs", "next_obs", "acts", "rewards",
                                                                   "terminals", "time_limits")})
        if use_graph:
            assert False in col._graphs
        runs.append((rows, col.current_ob.clone(), env.phys.clone(), env.episode.clone(), env.elapsed.clone(),
                     col.current_step.clone()))
    (r0, *s0), (r1, *s1) = runs
    for a, b in zip(r0, r1):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    for a, b in zip(s0, s1):
        assert torch.equal(a, b)
    return r1


def collector_rows_match_the_oracle(case, steps, ulps, N=24, seed=5):
    """Eager collector steps one at a time: each stored row (reward, terminal, time limit, next observation) is the
    oracle's step from the device's state before it under the stored actions, and every env the step ended is reset
    to the oracle's reset of its next episode.  Returns the number of rows that ended at a terminal state."""
    col, buf, env = collector(case, False, True, False, N=N, T=steps, seed=seed)
    seeds = seed * N + np.arange(N)
    episode = env.episode.cpu().numpy().astype(np.int64)
    n_term = 0
    for _ in range(steps):
        row = buf._top
        phys, el = env.phys.cpu().numpy().copy(), env.elapsed.cpu().numpy().copy()
        col.take_actions()
        acts = buf._acts[row].cpu().numpy().reshape(-1)
        wph, wobs, wr, wd, wtl, _ = case.step(phys, acts, el)
        term = buf._terminals[row].cpu().numpy().reshape(-1).astype(bool)
        tl = buf._time_limits[row].cpu().numpy().reshape(-1).astype(bool)
        ok = np.ones(N, bool) if case.near_goal is None else ~case.near_goal(wph)
        np.testing.assert_array_equal(term[ok], wd[ok])             # done, the time limit included (gym's done)
        np.testing.assert_array_equal(tl, wtl)
        np.testing.assert_array_equal(buf._rewards[row].cpu().numpy().reshape(-1)[ok], wr[ok])
        check_obs(buf._next_obs[row].cpu().numpy(), wobs)
        after = env.phys.cpu().numpy()
        wd = term                                                   # the device's episode ends decide the resets
        check_phys(after[~wd], wph[~wd], ulps)
        np.testing.assert_array_equal(after[wd], case.reset_phys(seeds[wd], episode[wd]))
        check_obs(col.current_ob.cpu().numpy()[wd], case.observe(after[wd]))
        episode[wd] += 1
        n_term += int((wd & ~wtl).sum())
    np.testing.assert_array_equal(env.episode.cpu().numpy(), episode)
    return n_term


def collector_launch_count(case):
    """The captured step holds the env step, the finalize, the env's own reset and the ring advance (the stub policy is
    torch ops), and replaying it counts as many library launches as one eager step."""
    from torchrl_b200 import _lib
    col, buf, env = collector(case, True, True, False)
    col.train_one_epoch()
    g = col._graphs[False]
    before = _lib.launch_count()
    col._step_body(False)
    eager = _lib.launch_count() - before
    assert eager == g.launches == 4
    before = _lib.launch_count()
    g.replay()
    assert _lib.launch_count() - before == g.launches


def discrete_agent(env_id, kind, obs_dim, N=16, T=40, seed=0, use_graph=True):
    """One of DQN, QR-DQN, PPO, A2C, REINFORCE on a discrete env with three actions."""
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import A2C, DQN, PPO, QRDQN, Reinforce
    from torchrl_b200.collector import VecCollector, VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer, OnPolicyReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device("cuda:0")
    env, eval_env = get_vec_env(env_id, {}, N), get_vec_env(env_id, {}, N)
    env.seed(seed); eval_env.seed(seed + 1000); torch.manual_seed(seed); np.random.seed(seed)
    if kind in ("dqn", "qrdqn"):
        Q = 8 if kind == "qrdqn" else 1
        buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=4 * T * N)
        qf = networks.Net(input_shape=(obs_dim,), output_shape=3 * Q, hidden_shapes=[64, 64], append_hidden_shapes=[],
                          base_type=networks.MLPBase, activation_func=nn.ReLU)
        kw = dict(qf=qf, start_epsilon=1.0, end_epsilon=0.1, decay_frames=4 * T * N, action_shape=3)
        pf = (policies.EpsilonGreedyQRDQNDiscretePolicy(quantile_num=Q, **kw) if kind == "qrdqn"
              else policies.EpsilonGreedyDQNDiscretePolicy(**kw))
        col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=T * N,
                           max_episode_frames=10000, use_cuda_graph=use_graph)
        common = dict(qf=qf, pf=pf, qlr=1e-3, env=env, replay_buffer=buf, collector=col, logger=NullLogger(),
                      discount=0.99, batch_size=4 * N, device=dev, save_dir=None, opt_times=4, use_soft_update=True,
                      tau=0.005, pretrain_epochs=1, num_epochs=3, use_cuda_graph=use_graph)
        agent = QRDQN(quantile_num=Q, **common) if kind == "qrdqn" else DQN(**common)
        return agent, col, buf, env
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    net = dict(input_shape=obs_dim, hidden_shapes=[32, 32], append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=torch.nn.Tanh)
    pf = policies.CategoricalDisPolicy(output_shape=3, **net)
    vf = networks.ZeroNet() if kind == "reinforce" else networks.Net(output_shape=1, **net)
    col = VecOnPolicyCollector(vf, env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=T * N,
                               max_episode_frames=10000, use_cuda_graph=use_graph)
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, num_epochs=10,
                  batch_size=8 * N, device=dev, save_dir=None, shuffle=True, use_cuda_graph=use_graph)
    if kind == "reinforce":
        agent = Reinforce(pf=pf, plr=3e-3, **common)
    elif kind == "ppo":
        agent = PPO(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, opt_epochs=2, tau=0.95, gae=True, clip_para=0.2, **common)
    else:
        agent = A2C(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, tau=0.95, gae=True, **common)
    return agent, col, buf, env


def one_epoch(agent, col, kind, off_policy):
    """Pretrain (off-policy), one collector epoch and one update epoch; every logged number is finite."""
    if off_policy:
        agent.pretrain()
    agent.current_epoch = 0
    out = col.train_one_epoch()
    agent.update_per_epoch()
    assert agent._last_infos
    for info in agent._last_infos:
        for k, v in info.items():
            if kind == "ppo" and k == "log_std/std":      # the reference's torch std of PPO's one log-std: NaN
                assert np.isnan(v)
            else:
                assert np.isfinite(v), k
    return out


def continuous_agent(env_id, kind, obs_dim, max_episode_frames, time_limit_filter, use_graph=True, N=16, T=40, seed=0):
    """One of TD3, DDPG, SAC, TwinSAC-Q, PPO on a continuous env with one action; `time_limit_filter` is the
    off-policy replay buffer's (PPO's buffer always filters)."""
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import DDPG, PPO, SAC, TD3, TwinSACQ
    from torchrl_b200.collector import VecCollector, VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer, OnPolicyReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device("cuda:0")
    env = get_vec_env(env_id, {"reward_scale": 1, "obs_norm": kind == "ppo"}, N)
    eval_env = get_vec_env(env_id, {"reward_scale": 1, "obs_norm": kind == "ppo"}, N)
    env.seed(seed); eval_env.seed(seed + 1000); torch.manual_seed(seed); np.random.seed(seed)
    o, a = obs_dim, 1
    net = dict(hidden_shapes=[64, 64], append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=nn.ReLU)
    if kind == "ppo":
        buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
        pf = policies.GuassianContPolicyBasicBias(input_shape=o, output_shape=a, tanh_action=True, **net)
        vf = networks.Net(input_shape=o, output_shape=1, **net)
        col = VecOnPolicyCollector(vf, env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev,
                                   epoch_frames=T * N, max_episode_frames=max_episode_frames, use_cuda_graph=use_graph)
        return PPO(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, clip_para=0.2, opt_epochs=2, tau=0.95, shuffle=True, env=env,
                   replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, num_epochs=3,
                   batch_size=10 * N, gae=True, device=dev, save_dir=None, use_cuda_graph=use_graph), col, buf, env
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=4 * T * N, time_limit_filter=time_limit_filter)
    if kind in ("sac", "twin_sac_q"):
        pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, tanh_action=True, **net)
    elif kind == "ddpg":
        pf = policies.DetContPolicy(input_shape=o, output_shape=a, tanh_action=True, **net)
    else:
        pf = policies.FixGuassianContPolicy(input_shape=o, output_shape=a, tanh_action=True, norm_std_explore=0.1,
                                            **net)
    qf1 = networks.QNet(input_shape=o + a, output_shape=1, **net)
    col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=T * N,
                       max_episode_frames=max_episode_frames, use_cuda_graph=use_graph)
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, batch_size=8 * N,
                  device=dev, save_dir=None, tau=0.005, use_soft_update=True, opt_times=8, pretrain_epochs=1,
                  num_epochs=3, use_cuda_graph=use_graph)
    if kind == "td3":
        agent = TD3(pf=pf, qf1=qf1, qf2=networks.QNet(input_shape=o + a, output_shape=1, **net), plr=1e-3, qlr=1e-3,
                    **common)
    elif kind == "ddpg":
        agent = DDPG(pf=pf, qf=qf1, plr=1e-3, qlr=1e-3, **common)
    elif kind == "twin_sac_q":
        agent = TwinSACQ(pf=pf, qf1=qf1, qf2=networks.QNet(input_shape=o + a, output_shape=1, **net), plr=3e-4,
                         qlr=3e-4, policy_std_reg_weight=0, policy_mean_reg_weight=0, **common)
    else:
        vf = networks.Net(input_shape=o, output_shape=1, **net)
        agent = SAC(pf=pf, vf=vf, qf=qf1, plr=3e-4, vlr=3e-4, qlr=3e-4, policy_std_reg_weight=1e-3,
                    policy_mean_reg_weight=1e-3, **common)
    return agent, col, buf, env
