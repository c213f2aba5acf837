"""The device Pendulum-v1 (csrc/pendulum.cu, torchrl_b200/env/pendulum.py) against its NumPy statement
(oracle/pendulum.py): single steps over ragged batch sizes with actions at, beyond and between the ends of [-1, 1], a long
rollout checked step by step, resets, sharded seeding, the NormObs moments, non-finite actions, the collector's reset
hook inside the captured step (graph == eager, episode cuts, launch counts), one epoch of each continuous agent, and a
TD3 resume.

Tolerance of the fp64 state: the kernel and NumPy differ only in `sin` / `cos` (CUDA's fp64 sin is within 2 ulp, glibc's
within 1).  sin(theta) enters the new velocity as 15 * sin * 0.05, so its error is 0.75 of an ulp of a number <= 1 before
the roundings of the sum; one or two last-bit flips of theta_dot and theta follow.  The check allows 4 ulp of
max(|x|, 1) in fp64 and one fp32 ulp in the observation; over 64 envs about 90 % of the fp64 components were
bit-identical on an H100, and at least 75 % must be.  The cost uses no sin / cos, so rewards must be bit-identical."""
import math

import numpy as np
import pytest

from oracle import pendulum as P
from tests import classic_control_gpu as cc

pytestmark = pytest.mark.gpu


def _case():
    from torchrl_b200 import ops
    return cc.Case("Pendulum-v1", 2, 3, P.step, P.reset_phys, P.observe, None, ops.pendulum_step)


def _check_phys(got, want):
    cc.check_phys(got, want, 4)
    if np.size(got) >= 128:
        assert np.mean(got == want) >= 0.75, np.mean(got == want)        # most components agree to the last bit


@pytest.mark.parametrize("N", [1, 33, 4099])
@pytest.mark.parametrize("reward_scale", [1.0, 0.5])
def test_step_matches_oracle(N, reward_scale):
    rs = np.random.RandomState(N)
    phys = np.stack([rs.uniform(-3 * math.pi, 3 * math.pi, N), rs.uniform(-8, 8, N)], 1)
    fast = rs.rand(N) < 0.2                                   # near the speed limit: the clip decides
    phys[fast, 1] = np.sign(rs.randn(int(fast.sum()))) * rs.uniform(7.5, 8.0, int(fast.sum()))
    a = rs.uniform(-1, 1, N).astype(np.float32)
    pick = rs.randint(0, 6, N)
    a = np.where(pick == 0, 1.0, np.where(pick == 1, -1.0, np.where(pick == 2, 0.0, a))).astype(np.float32)
    a[pick == 3] = rs.choice([1.5, -1.5, 3.0, -7.0], int((pick == 3).sum()))
    el = rs.randint(0, 200, N)
    el[rs.rand(N) < 0.3] = 199
    ph, obs, r, d, tl, el2, err, any_reset = cc.step_kernel(_case(), phys, a, el, reward_scale, 200)
    wph, wobs, wr, wd, wtl, wel = P.step(phys, a, el, reward_scale=reward_scale)
    assert err == 0
    _check_phys(ph, wph)
    cc.check_obs(obs, wobs)
    cc.check_obs(obs, P.observe(ph))
    np.testing.assert_array_equal(r, wr)
    np.testing.assert_array_equal(el2, wel)
    np.testing.assert_array_equal(d, wd)
    np.testing.assert_array_equal(tl, wtl)
    assert any_reset[0] == int(d.any())
    if N == 4099:
        assert (np.abs(ph[:, 1]) == 8.0).sum() > 50             # the clip was exercised


def test_step_from_the_rest_state():
    ph, obs, r, *_ = cc.step_kernel(_case(), np.zeros((3, 2)), [1.0, -1.0, 0.0], [0, 0, 0], max_steps=200)
    assert ph.tolist() == [[0.30000000000000004 * 0.05, 0.30000000000000004], [-0.015000000000000003,
                                                                               -0.30000000000000004], [0.0, 0.0]]
    assert r.tolist() == np.float32([-0.004, -0.004, 0.0]).tolist()


def test_reset_seeding_and_sharding():
    import torch
    from torchrl_b200.env import get_vec_env
    N = 37
    env = get_vec_env("Pendulum-v1", {}, 2 * N)
    env.seed(5)
    full = env.reset().cpu().numpy()
    seeds = 5 * 2 * N + np.arange(2 * N)
    want = P.reset_phys(seeds, np.zeros(2 * N))
    np.testing.assert_array_equal(env.phys.cpu().numpy(), want)
    cc.check_obs(full, P.observe(want))
    parts, pphys = [], []
    for r in range(2):
        e = get_vec_env("Pendulum-v1", {}, N, first_env=r * N, total_envs=2 * N)
        e.seed(5)
        parts.append(e.reset().cpu().numpy())
        pphys.append(e.phys.cpu().numpy())
    np.testing.assert_array_equal(np.concatenate(parts), full)
    np.testing.assert_array_equal(np.concatenate(pphys), env.phys.cpu().numpy())
    env.reset()                                                  # the next episode of every env
    np.testing.assert_array_equal(env.phys.cpu().numpy(), P.reset_phys(seeds, np.ones(2 * N)))
    mask = torch.zeros(2 * N, dtype=torch.bool, device="cuda")
    mask[::3] = True
    before, before_obs = env.phys.cpu().numpy().copy(), env.state.cpu().numpy().copy()
    raw = env.partial_reset(mask).cpu().numpy()
    after = env.phys.cpu().numpy()
    m = mask.cpu().numpy()
    np.testing.assert_array_equal(after[~m], before[~m])
    np.testing.assert_array_equal(raw[~m], before_obs[~m])
    np.testing.assert_array_equal(after[m], P.reset_phys(seeds[m], np.full(m.sum(), 2)))
    cc.check_obs(raw[m], P.observe(after[m]))


def test_rollout_tracks_the_oracle_step_by_step():
    """1000 steps (five episodes) of a mixed controller: every step against the oracle from the device's state, every
    reset against the oracle's reset of that env's next episode."""
    import torch
    from torchrl_b200.env import get_vec_env
    N, steps = 64, 1000
    env = get_vec_env("Pendulum-v1", {"reward_scale": 0.1}, N)
    env.seed(11)
    seeds = 11 * N + np.arange(N)
    env.reset()
    episode = np.ones(N, np.int64)
    phys = env.phys.cpu().numpy().copy()
    el = np.zeros(N, np.int64)
    rs = np.random.RandomState(0)
    n_done = 0
    for t in range(steps):
        ctrl = np.clip(-(np.sin(phys[:, 0]) * 2 + 0.5 * phys[:, 1]), -1, 1)
        a = np.where(np.arange(N) < N // 2, ctrl, rs.uniform(-1.2, 1.2, N)).astype(np.float32)
        obs, r, done, info = env.step(torch.as_tensor(a, device="cuda"))
        wph, wobs, wr, wd, wtl, wel = P.step(phys, a, el, reward_scale=0.1)
        got = env.phys.cpu().numpy().copy()
        _check_phys(got, wph)
        cc.check_obs(obs.cpu().numpy(), wobs)
        np.testing.assert_array_equal(r.cpu().numpy().reshape(-1), wr)
        d = done.cpu().numpy().reshape(-1)
        np.testing.assert_array_equal(d, wd)
        np.testing.assert_array_equal(info["time_limit"].cpu().numpy(), wtl)
        el = wel
        if d.any():
            n_done += int(d.sum())
            env.partial_reset(done.reshape(-1))
            got = env.phys.cpu().numpy().copy()
            np.testing.assert_array_equal(got[d], P.reset_phys(seeds[d], episode[d]))
            episode[d] += 1
            el[d] = 0
        phys = got
    assert n_done == 5 * N


def test_normobs_moments_match_the_chan_formula():
    import torch
    from torchrl_b200.env import get_vec_env
    N = 1000
    env = get_vec_env("Pendulum-v1", {"obs_norm": True}, N)
    env.seed(2)
    env.reset()
    nrm = env._obs_normalizer
    mean, var, count = (t.cpu().numpy().astype(np.float64).copy() for t in (nrm._mean, nrm._var, nrm._count))
    for k in range(3):
        act = np.linspace(-1, 1, N).astype(np.float32) * (1 - 2 * (k % 2))
        obs, *_ = env.step(torch.as_tensor(act, device="cuda"))
        x = env.state.cpu().numpy().astype(np.float64)
        sums = env.batch_sums.cpu().numpy()
        np.testing.assert_allclose(sums[:3], x.sum(0), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sums[3:], (x * x).sum(0), rtol=1e-12)
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


def test_non_finite_action_raises_at_the_next_sync():
    import torch
    from torchrl_b200.env import get_vec_env
    env = get_vec_env("Pendulum-v1", {}, 8)
    env.reset()
    before, before_obs = env.phys.clone(), env.state.clone()
    with pytest.raises(ValueError, match="finite actions"):
        env.step(torch.tensor([0, 1, float("nan"), 1, 0, float("inf"), 1, 1], device="cuda"))
    for i in (2, 5):
        assert torch.equal(env.phys[i], before[i]) and torch.equal(env.state[i], before_obs[i])
    assert not torch.equal(env.phys[0], before[0])
    env.step(torch.ones(8, device="cuda"))                    # the flag was cleared: finite actions go through
    with pytest.raises(ValueError):
        env.step(torch.full((8,), float("-inf"), device="cuda"))


def test_spaces_and_routing():
    from torchrl_b200.env import PendulumVecEnv, get_vec_env
    env = get_vec_env("Pendulum-v1", {}, 3)
    assert isinstance(env, PendulumVecEnv) and env._max_episode_steps == 200 and env.lockstep
    assert env.observation_space.shape == (3,) and env.action_space.shape == (1,)
    np.testing.assert_array_equal(env.observation_space.high, [1, 1, 8])
    np.testing.assert_array_equal(env.action_space.low, [-1])


# ------------------------------------------------------------------------------------------ collector hook
def _collector(use_graph, quirks, obs_norm, N=24, T=12, max_frames=200, seed=3, steps_per_epoch=None):
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer
    env = get_vec_env("Pendulum-v1", {"reward_scale": 1, "obs_norm": obs_norm}, N, max_episode_steps=None)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=False)
    net = dict(hidden_shapes=[32, 32], append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=nn.ReLU)
    pf = policies.FixGuassianContPolicy(input_shape=3, output_shape=1, tanh_action=True, norm_std_explore=0.3, **net)
    col = VecCollector(env=env, pf=pf, replay_buffer=buf, device=torch.device("cuda:0"),
                       epoch_frames=(steps_per_epoch or T) * N, max_episode_frames=max_frames,
                       use_cuda_graph=use_graph, reference_quirks=quirks)
    return col, buf, env


def _short_episodes(env, limit):
    env._max_episode_steps = limit


@pytest.mark.parametrize("quirks", [True, False])
@pytest.mark.parametrize("obs_norm", [False, True])
def test_collector_graph_equals_eager(quirks, obs_norm):
    """Epochs with the captured step and with eager steps store bit-identical rows and carry the same current_ob.
    Episodes are shortened to 7 steps so that resets (and quirk A.1's all-raw step) happen inside the epochs."""
    import torch
    runs = []
    for use_graph in (False, True):
        col, buf, env = _collector(use_graph, quirks, obs_norm)
        _short_episodes(env, 7)
        rows = []
        for _ in range(3):
            col.train_one_epoch()
            rows.append({k: getattr(buf, "_" + k).clone() for k in ("obs", "next_obs", "acts", "rewards",
                                                                   "terminals", "time_limits")})
        if use_graph:
            assert False in col._graphs
        runs.append((rows, col.current_ob.clone(), env.phys.clone(), env.episode.clone(), env.elapsed.clone()))
    (r0, c0, p0, e0, l0), (r1, c1, p1, e1, l1) = runs
    for a, b in zip(r0, r1):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert torch.equal(c0, c1) and torch.equal(p0, p1) and torch.equal(e0, e1) and torch.equal(l0, l1)
    assert int(r1[-1]["time_limits"].sum()) > 0


@pytest.mark.parametrize("quirks", [True, False])
def test_collector_resets_cut_episodes(quirks):
    """max_episode_frames = 5 < 200 cuts every episode after 5 steps: the next observation of a cut env is its next
    episode's reset observation (raw, or normalised without quirk A.1), the env's elapsed and episode counters follow,
    and no cut is stored as a terminal or a time limit."""
    import torch
    N, T = 16, 12
    col, buf, env = _collector(True, quirks, False, N=N, T=T, max_frames=5)
    seeds = np.arange(N)                                         # seed 0: seeds[i] = i
    env.seed(0)
    col.current_ob.copy_(env.reset())
    col.train_one_epoch()
    obs, nxt = buf._obs.cpu().numpy(), buf._next_obs.cpu().numpy()
    assert not buf._terminals.cpu().numpy().any() and not buf._time_limits.cpu().numpy().any()
    ep = 1
    for t in range(T - 1):
        if (t + 1) % 5 == 0:                                      # rows 4, 9: the step that cut every env
            want = P.observe(P.reset_phys(seeds, np.full(N, ep)))
            cc.check_obs(obs[t + 1], want)
            ep += 1
        else:
            np.testing.assert_array_equal(obs[t + 1], nxt[t])
    assert env.episode.cpu().numpy().tolist() == [3] * N
    assert env.elapsed.cpu().numpy().tolist() == [2] * N == col.current_step.cpu().numpy().tolist()


def test_collector_step_graph_launch_count():
    from torchrl_b200 import _lib
    col, buf, env = _collector(True, True, True)
    col.train_one_epoch()
    g = col._graphs[False]
    before = _lib.launch_count()
    col._step_body(False)                                       # one eager step: the same launches as the graph
    eager = _lib.launch_count() - before
    assert eager == g.launches
    before = _lib.launch_count()
    g.replay()
    assert _lib.launch_count() - before == g.launches


# ------------------------------------------------------------------------------------------ agents
@pytest.mark.parametrize("kind", ["td3", "ddpg", "sac", "twin_sac_q", "ppo"])
def test_one_epoch_of_each_agent(kind):
    agent, col, buf, env = cc.continuous_agent("Pendulum-v1", kind, 3, 200, False)
    out = cc.one_epoch(agent, col, kind, kind != "ppo")
    assert all(-16.3 * 200 <= r <= 0 for r in out["train_rewards"])     # the cost is at most pi^2 + 6.4 + 0.004
    acts = buf._acts.cpu().numpy()
    assert np.all(np.abs(acts[:buf._size]) <= 1.0)
    ev = col.eval_one_epoch()
    assert len(ev["eval_rewards"]) == 16 and ev["eval_traj_length"] == 200.0


def test_td3_resume_continues_identically(tmp_path):
    import torch
    path = str(tmp_path / "ck.pt")

    def epochs(agent, col, first, n):
        out = []
        for e in range(first, first + n):
            agent.current_epoch = e
            out.append(col.train_one_epoch()["train_epoch_reward"])
            agent.update_per_epoch()
        return out

    agent, col, buf, env = cc.continuous_agent("Pendulum-v1", "td3", 3, 200, False, use_graph=False, seed=1)
    agent.pretrain()
    epochs(agent, col, 0, 3)                                      # 3 x 40 steps: mid-episode at the checkpoint
    agent.save_checkpoint(path)
    want_r = epochs(agent, col, 3, 3)
    want, want_t, want_phys = agent.opt.data.clone(), agent._target_flat.data.clone(), env.phys.clone()
    agent2, col2, buf2, env2 = cc.continuous_agent("Pendulum-v1", "td3", 3, 200, False, use_graph=False, seed=77)
    assert agent2.load_checkpoint(path) == 3
    got_r = epochs(agent2, col2, 3, 3)
    np.testing.assert_allclose(got_r, want_r, rtol=1e-6)
    assert torch.equal(env2.phys, want_phys)
    torch.testing.assert_close(agent2.opt.data, want, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(agent2._target_flat.data, want_t, rtol=1e-5, atol=1e-7)
