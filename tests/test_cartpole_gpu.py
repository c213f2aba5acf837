"""The device CartPole (csrc/cartpole.cu, torchrl_b200/env/cartpole.py) against its NumPy statement (oracle/cartpole.py):
single steps over ragged batch sizes and states within a few ulps of the thresholds, resets, a long rollout checked
step by step, the NormObs moments, sharded seeding, invalid actions, and the collectors' discrete-action path on float
observations (epsilon-greedy DQN / QR-DQN and the categorical on-policy agents) through the captured step graph."""
import numpy as np
import pytest

from oracle import cartpole as C

pytestmark = pytest.mark.gpu


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def _check_states(got, want):
    """Equal after fp32 rounding for >= 99.99 % of the components and within one fp32 ulp for all."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert np.all(diff <= _ulp(want)), np.max(diff / np.maximum(_ulp(want), 1e-45))
    assert np.mean(got == want) >= 0.9999, np.mean(got == want)


def _near_threshold(state):
    s = np.asarray(state, np.float32).astype(np.float64)
    return ((np.abs(np.abs(s[:, 0]) - C.X_THRESHOLD) <= _ulp(s[:, 0])) |
            (np.abs(np.abs(s[:, 2]) - C.THETA_THRESHOLD) <= _ulp(s[:, 2])))


def _check_flags(got, want, state):
    bad = (np.asarray(got, bool) != np.asarray(want, bool)) & ~_near_threshold(state)
    assert not bad.any(), np.flatnonzero(bad)[:10]


def _states(N, rs):
    """Random states; a quarter of them sit within a few ulps of +-2.4 or +-12 degrees with zero velocity, so the next
    state keeps that position exactly."""
    s = np.stack([rs.uniform(-2.4, 2.4, N), rs.randn(N), rs.uniform(-0.2, 0.2, N), 1.5 * rs.randn(N)], 1)
    s = s.astype(np.float32)
    edge = rs.rand(N) < 0.25
    for i in np.flatnonzero(edge):
        j = rs.randint(2)
        thr = np.float32(C.X_THRESHOLD if j == 0 else C.THETA_THRESHOLD)
        v = thr
        for _ in range(rs.randint(-3, 4) + 3):
            v = np.nextafter(v, np.float32(np.inf))
        for _ in range(3):
            v = np.nextafter(v, np.float32(-np.inf))
        s[i, 2 * j] = v * (1 if rs.rand() < 0.5 else -1)
        s[i, 2 * j + 1] = 0.0
    return s


def _step_kernel(state, actions, elapsed, max_steps, reward_scale=1.0, step_count=None, max_frames=1 << 30):
    import torch
    from torchrl_b200 import ops
    dev = "cuda"
    N = state.shape[0]
    st = torch.as_tensor(state, device=dev).contiguous()
    el = torch.as_tensor(elapsed, dtype=torch.int32, device=dev).contiguous()
    out = dict(reward=torch.zeros(N, device=dev), done=torch.zeros(N, dtype=torch.uint8, device=dev),
               time_limit=torch.zeros(N, dtype=torch.uint8, device=dev))
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ticket = torch.zeros(1, dtype=torch.int32, device=dev)
    any_reset = torch.zeros(2, dtype=torch.int32, device=dev)
    sc = None if step_count is None else torch.as_tensor(step_count, dtype=torch.int32, device=dev)
    ops.cartpole_step(st, torch.as_tensor(actions, dtype=torch.float32, device=dev), el, sc, out["reward"],
                      out["done"], out["time_limit"], err, None, None, None, None, None, ticket, any_reset, None,
                      reward_scale, max_steps, max_frames, False)
    return (st.cpu().numpy(), out["reward"].cpu().numpy(), out["done"].cpu().numpy().astype(bool),
            out["time_limit"].cpu().numpy().astype(bool), el.cpu().numpy(), int(err.item()), any_reset.cpu().numpy())


@pytest.mark.parametrize("N", [1, 33, 4099])
@pytest.mark.parametrize("max_steps", [200, 500])
@pytest.mark.parametrize("reward_scale", [1.0, 0.5])
def test_step_matches_oracle(N, max_steps, reward_scale):
    rs = np.random.RandomState(N + max_steps)
    s = _states(N, rs)
    a = rs.randint(0, 2, N).astype(np.float32)
    el = rs.randint(0, max_steps, N)
    late = rs.rand(N) < 0.5                             # a step or three before the time limit
    el[late] = rs.randint(max_steps - 3, max_steps, int(late.sum()))
    st, r, d, tl, el2, err, any_reset = _step_kernel(s, a, el, max_steps, reward_scale)
    ws, wr, wd, wtl, wel = C.step(s, a, el, max_steps, reward_scale)
    assert err == 0
    _check_states(st, ws)
    np.testing.assert_array_equal(r, wr)
    np.testing.assert_array_equal(el2, wel)
    _check_flags(d, wd, ws)
    _check_flags(tl, wtl, ws)
    assert any_reset[0] == int(d.any())
    if N == 4099:
        assert _near_threshold(ws).sum() > 10          # the edge states reach the thresholds


def test_step_from_the_zero_state():
    s = np.zeros((2, 4), np.float32)
    st = _step_kernel(s, [1.0, 0.0], [0, 0], 500)[0]
    want = np.float32([[0.0, 0.1951219512195122, 0.0, -0.2926829268292683]])
    np.testing.assert_array_equal(st, np.concatenate([want, -want]))


def test_reset_seeding_and_sharding():
    import torch
    from torchrl_b200.env import get_vec_env
    N = 37
    env = get_vec_env("CartPole-v1", {}, 2 * N)
    env.seed(5)
    full = env.reset().cpu().numpy()
    seeds = 5 * 2 * N + np.arange(2 * N)
    np.testing.assert_array_equal(full, C.reset_state(seeds, np.zeros(2 * N)))
    assert np.abs(full).max() <= 0.05 and np.abs(full).max() > 0.04
    parts = []
    for r in range(2):
        e = get_vec_env("CartPole-v1", {}, N, first_env=r * N, total_envs=2 * N)
        e.seed(5)
        parts.append(e.reset().cpu().numpy())
    np.testing.assert_array_equal(np.concatenate(parts), full)
    # a second reset is the next episode of every env
    np.testing.assert_array_equal(env.reset().cpu().numpy(), C.reset_state(seeds, np.ones(2 * N)))
    # partial reset: only the masked envs move to their next episode
    mask = torch.zeros(2 * N, dtype=torch.bool, device="cuda")
    mask[::3] = True
    before = env.state.cpu().numpy().copy()
    env.partial_reset(mask)
    after = env.state.cpu().numpy()
    m = mask.cpu().numpy()
    np.testing.assert_array_equal(after[~m], before[~m])
    np.testing.assert_array_equal(after[m], C.reset_state(seeds[m], np.full(m.sum(), 2)))


@pytest.mark.parametrize("env_id", ["CartPole-v0", "CartPole-v1"])
def test_rollout_tracks_the_oracle_step_by_step(env_id):
    """1000 steps under a fixed action sequence: every step against the oracle from the device's state, every reset
    against the oracle's reset of that env's episode.  Rewards are 1 on every step, the terminating one included."""
    import torch
    from torchrl_b200.env import get_vec_env
    N, steps = 64, 1000
    limit = C.MAX_EPISODE_STEPS[env_id]
    env = get_vec_env(env_id, {}, N)
    env.seed(11)
    seeds = 11 * N + np.arange(N)
    episode = np.zeros(N, np.int64)
    s = env.reset().cpu().numpy().copy()
    episode += 1
    el = np.zeros(N, np.int64)
    rs = np.random.RandomState(0)
    # a balancing controller for most envs (episodes reach the time limit), random pushes for the rest
    n_done = n_tl = 0
    for t in range(steps):
        a = np.where(np.arange(N) < N // 2, (s[:, 2] + 0.5 * s[:, 3] > 0), rs.randint(0, 2, N)).astype(np.float32)
        obs, r, done, info = env.step(torch.as_tensor(a, device="cuda"))
        got = obs.cpu().numpy().copy()
        ws, wr, wd, wtl, wel = C.step(s, a, el, limit)
        _check_states(got, ws)
        np.testing.assert_array_equal(r.cpu().numpy().reshape(-1), wr)
        d = done.cpu().numpy().reshape(-1)
        _check_flags(d, wd, ws)
        _check_flags(info["time_limit"].cpu().numpy(), wtl, ws)
        n_done += int(d.sum())
        n_tl += int(info["time_limit"].cpu().numpy().sum())
        el = wel
        if d.any():
            env.partial_reset(done.reshape(-1))
            got = env.state.cpu().numpy().copy()
            np.testing.assert_array_equal(got[d], C.reset_state(seeds[d], episode[d]))
            episode[d] += 1
            el[d] = 0
        s = env.state.cpu().numpy().copy()
    assert n_done > 100 and n_tl > 0, (n_done, n_tl)


def test_normobs_moments_match_the_synth_formula():
    import torch
    from torchrl_b200.env import get_vec_env
    N = 1000
    env = get_vec_env("CartPole-v1", {"obs_norm": True}, N)
    env.seed(2)
    env.reset()
    nrm = env._obs_normalizer
    mean, var, count = (t.cpu().numpy().astype(np.float64).copy() for t in (nrm._mean, nrm._var, nrm._count))
    for _ in range(3):
        s = env.state.cpu().numpy().copy()
        act = (np.arange(N) % 2).astype(np.float32)
        obs, *_ = env.step(torch.as_tensor(act, device="cuda"))
        x = env.state.cpu().numpy().astype(np.float64)
        ws, _ = C.dynamics(s, act)
        _check_states(x, ws)
        sums = env.batch_sums.cpu().numpy()
        np.testing.assert_allclose(sums[:4], x.sum(0), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sums[4:], (x * x).sum(0), rtol=1e-12)
        # Chan merge, as base_wrapper.py:44-60 and the synth env
        bm, bv = x.mean(0), x.var(0)
        tot = count + N
        delta = bm - mean
        var = (var * count + bv * N + delta ** 2 * count * N / tot) / tot
        mean = mean + delta * N / tot
        count = tot
        np.testing.assert_allclose(nrm._mean.cpu().numpy(), mean, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(nrm._var.cpu().numpy(), var, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(nrm._count.cpu().numpy(), count)
        want = np.clip((x - mean) / (np.sqrt(var) + 1e-4), -10, 10)
        np.testing.assert_allclose(obs.cpu().numpy(), want, rtol=1e-5, atol=1e-5)


def test_invalid_action_raises_at_the_next_sync():
    import torch
    from torchrl_b200.env import get_vec_env
    env = get_vec_env("CartPole-v0", {}, 8)
    env.reset()
    before = env.state.clone()
    with pytest.raises(ValueError, match="actions 0 and 1"):
        env.step(torch.tensor([0, 1, 0.5, 1, 0, 0, 1, 1], device="cuda"))
    assert torch.equal(env.state[2], before[2])              # the env with the bad action did not move
    env.step(torch.ones(8, device="cuda"))                    # the flag was cleared: valid actions go through
    with pytest.raises(ValueError):
        env.step(torch.full((8,), 2.0, device="cuda"))


def test_spaces_and_routing():
    from torchrl_b200.env import CartPoleVecEnv, get_vec_env
    for env_id, limit in (("CartPole-v0", 200), ("CartPole-v1", 500)):
        env = get_vec_env(env_id, {}, 3)
        assert isinstance(env, CartPoleVecEnv) and env._max_episode_steps == limit and not env.lockstep
        assert env.action_space.n == 2 and env.observation_space.shape == (4,)
        np.testing.assert_array_equal(env.observation_space.high,
                                      [4.8, np.finfo(np.float32).max, 0.41887902047863906, np.finfo(np.float32).max])


# ------------------------------------------------------------------------------------------ collectors
def _dqn(kind, N=16, use_graph=True):
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import DQN, QRDQN
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device("cuda:0")
    env = get_vec_env("CartPole-v1", {}, N)
    env.seed(0); torch.manual_seed(0); np.random.seed(0)
    Q = 8 if kind == "qrdqn" else 1
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=64 * N)
    qf = networks.Net(input_shape=(4,), output_shape=2 * Q, hidden_shapes=[128, 128], append_hidden_shapes=[],
                      base_type=networks.MLPBase, activation_func=nn.ReLU)
    kw = dict(qf=qf, start_epsilon=1.0, end_epsilon=0.1, decay_frames=40, action_shape=2)
    pf = (policies.EpsilonGreedyQRDQNDiscretePolicy(quantile_num=Q, **kw) if kind == "qrdqn"
          else policies.EpsilonGreedyDQNDiscretePolicy(**kw))
    col = VecCollector(env=env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=8 * N, max_episode_frames=1000,
                       use_cuda_graph=use_graph)
    common = dict(qf=qf, pf=pf, qlr=1e-3, env=env, replay_buffer=buf, collector=col, logger=NullLogger(),
                  discount=0.99, batch_size=4 * N, device=dev, save_dir=None, opt_times=4, use_soft_update=True,
                  tau=0.005, pretrain_epochs=1, num_epochs=3, use_cuda_graph=use_graph)
    agent = QRDQN(quantile_num=Q, **common) if kind == "qrdqn" else DQN(**common)
    return agent, col, buf, env


@pytest.mark.parametrize("kind", ["dqn", "qrdqn"])
def test_off_policy_collector_on_cartpole(kind):
    agent, col, buf, env = _dqn(kind)
    agent.pretrain()
    for epoch in range(3):
        agent.current_epoch = epoch
        col.train_one_epoch()
        agent.update_per_epoch()
        for info in agent._last_infos:
            assert np.isfinite(info["Training/qf_loss"])
    assert False in col._graphs                                        # the step was captured
    acts = buf._acts.cpu().numpy()
    assert buf._acts.shape == (64, 16) and set(np.unique(acts[:buf._size])) <= {0.0, 1.0}
    assert 0.1 <= agent.pf.epsilon < 1.0                               # the schedule advanced outside the graph
    obs, nxt = buf._obs.cpu().numpy(), buf._next_obs.cpu().numpy()
    n = buf._size
    a = acts[:n].reshape(-1)
    ws, _ = C.dynamics(obs[:n].reshape(-1, 4), a)
    _check_states(nxt[:n].reshape(-1, 4), ws)                          # every stored transition is a CartPole step
    ev = col.eval_one_epoch()
    assert len(ev["eval_rewards"]) == 16 and all(1 <= r <= 500 for r in ev["eval_rewards"])


def _on_policy(kind, N=16, T=32, use_graph=True, seed=0):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import A2C, PPO, Reinforce
    from torchrl_b200.collector import VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device("cuda:0")
    env = get_vec_env("CartPole-v1", {}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    net = dict(input_shape=4, hidden_shapes=[32, 32], append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=torch.nn.Tanh)
    pf = policies.CategoricalDisPolicy(output_shape=2, **net)
    vf = networks.ZeroNet() if kind == "reinforce" else networks.Net(output_shape=1, **net)
    col = VecOnPolicyCollector(vf, env=env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=T * N,
                               max_episode_frames=1000, use_cuda_graph=use_graph)
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, num_epochs=10,
                  batch_size=8 * N, device=dev, save_dir=None, shuffle=True, use_cuda_graph=use_graph)
    if kind == "reinforce":
        agent = Reinforce(pf=pf, plr=3e-3, **common)
    elif kind == "ppo":
        agent = PPO(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, opt_epochs=2, tau=0.95, gae=True, clip_para=0.2, **common)
    else:
        agent = A2C(pf=pf, vf=vf, plr=3e-4, vlr=3e-4, tau=0.95, gae=True, **common)
    return agent, col, buf, env


@pytest.mark.parametrize("kind", ["ppo", "a2c", "reinforce"])
def test_on_policy_collector_on_cartpole(kind):
    from torchrl_b200 import _lib
    agent, col, buf, env = _on_policy(kind)
    for epoch in range(3):
        agent.current_epoch = epoch
        col.train_one_epoch()
        agent.update_per_epoch()
        assert all(np.isfinite(v) for info in agent._last_infos for v in info.values())
    assert True in col._graphs and agent._mb_graph is not None
    acts = buf._acts.cpu().numpy()
    assert buf._acts.shape == (32, 16) and set(np.unique(acts)) <= {0.0, 1.0}
    ws, _ = C.dynamics(buf._obs.cpu().numpy().reshape(-1, 4), acts.reshape(-1))
    _check_states(buf._next_obs.cpu().numpy().reshape(-1, 4), ws)    # every stored transition is a CartPole step
    vals = buf._values.cpu().numpy()
    if kind == "reinforce":
        assert not vals.any()                                          # V = 0 without a launch
        g = col._graphs[True]
        before = _lib.launch_count()
        g.replay()
        assert _lib.launch_count() - before == g.launches
    else:
        assert vals.any()


def test_reinforce_step_graph_has_no_value_launches():
    """A ZeroNet value function adds nothing to the collector's captured step: the same graph as without any value
    net, i.e. policy forward + sampler + env step + finalize + ring advance."""
    agent, col, buf, env = _on_policy("reinforce")
    col.train_one_epoch()
    ppo, pcol, _, _ = _on_policy("ppo")
    pcol.train_one_epoch()
    assert col._graphs[True].launches < pcol._graphs[True].launches
