"""The device MountainCar-v0 and MountainCarContinuous-v0 (csrc/mountain_car.cu, torchrl_b200/env/mountain_car.py)
against their NumPy statement (oracle/mountain_car.py): single steps from random and boundary states over ragged batch
sizes, a long rollout re-synchronised every step, resets, sharded seeding, the NormObs moments, refused actions, the
collector with the env's own reset inside the captured step (graph == eager, rows against the oracle, launch counts),
evaluation with the scripted controller against the oracle's episodes, and one epoch of each agent.

Tolerance of the fp64 state: the kernel and NumPy differ only in cos(3x) (CUDA's fp64 cos is within 2 ulp, NumPy's
within 1), which enters the velocity scaled by 0.0025: at most a last-bit flip of the velocity and the position.  The
check allows 4 ulp of max(|x|, 1).  fp32 observations must be equal or one ulp apart, and rewards and done flags
identical except within 1e-12 of the goal."""
import numpy as np
import pytest

from oracle import mountain_car as M
from tests import classic_control_gpu as cc

pytestmark = pytest.mark.gpu

V0, CONT = "MountainCar-v0", "MountainCarContinuous-v0"
ULPS = 4


def _controller(env_id):
    def push(ob):
        import torch
        hi, lo = (1.0, -1.0) if env_id == CONT else (2.0, 0.0)
        return torch.where(ob[:, 1] >= 0, hi, lo).float()
    return push


def _case(env_id):
    from torchrl_b200 import ops

    def step(phys, actions, elapsed, reward_scale=1.0):
        return M.step(phys, actions, elapsed, env_id, reward_scale=reward_scale)
    return cc.Case(env_id, 2, 2, step, M.reset_phys, M.observe, _controller(env_id), ops.mountain_car_step,
                   (env_id == CONT,))


def _states(N, rs, env_id):
    goal = M.SPECS[env_id][0]
    phys = np.stack([rs.uniform(-1.2, 0.6, N), rs.uniform(-0.07, 0.07, N)], 1)
    pick = rs.randint(0, 6, N)
    phys[pick == 0, 0] = rs.choice([-1.2, 0.6, goal, -0.5], int((pick == 0).sum()))
    phys[pick == 1, 1] = rs.choice([-0.07, 0.07, 0.0], int((pick == 1).sum()))
    wall = pick == 2                                          # against the left wall, moving left
    phys[wall] = np.stack([rs.uniform(-1.2, -1.15, int(wall.sum())), rs.uniform(-0.07, -0.01, int(wall.sum()))], 1)
    near = pick == 3                                          # just short of the goal
    phys[near, 0] = goal - rs.uniform(0.0, 0.07, int(near.sum()))
    return phys


def _actions(N, rs, env_id):
    if env_id == V0:
        return rs.randint(0, 3, N).astype(np.float32)
    a = rs.uniform(-1, 1, N).astype(np.float32)
    pick = rs.randint(0, 5, N)
    a[pick == 0] = rs.choice([1.0, -1.0, 0.0, 1.5, -3.0], int((pick == 0).sum()))
    return a


def _near_goal(phys, env_id):
    return (np.abs(phys[:, 0] - M.SPECS[env_id][0]) < 1e-12) | (np.abs(phys[:, 1]) < 1e-12)


@pytest.mark.parametrize("env_id", [V0, CONT])
@pytest.mark.parametrize("N", [1, 255, 256, 257, 100003])
def test_step_matches_oracle(N, env_id):
    rs = np.random.RandomState(N)
    phys = _states(N, rs, env_id)
    a = _actions(N, rs, env_id)
    limit = M.SPECS[env_id][1]
    el = rs.randint(0, limit, N)
    el[rs.rand(N) < 0.3] = limit - 1
    reward_scale = 0.5 if N % 2 else 1.0
    ph, obs, r, d, tl, el2, err, any_reset = cc.step_kernel(_case(env_id), phys, a, el, reward_scale, limit)
    wph, wobs, wr, wd, wtl, wel = M.step(phys, a, el, env_id, reward_scale=reward_scale)
    assert err == 0
    cc.check_phys(ph, wph, ULPS)
    cc.check_obs(obs, wobs)
    np.testing.assert_array_equal(obs, M.observe(ph))
    ok = ~_near_goal(wph, env_id)
    np.testing.assert_array_equal(d[ok], wd[ok])
    if env_id == V0:
        np.testing.assert_array_equal(r, wr)
    else:
        np.testing.assert_array_equal(r[ok], wr[ok])
    np.testing.assert_array_equal(tl, wtl)
    np.testing.assert_array_equal(el2, wel)
    assert any_reset[0] == int(d.any())
    if N == 100003:
        assert (ph[:, 0] == -1.2).sum() > 1000 and (ph[ph[:, 0] == -1.2, 1] >= 0).all()      # the wall was hit
        assert (wd & ~wtl).sum() > 1000 and (np.abs(ph[:, 1]) == 0.07).sum() > 100


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_goal_and_wall_boundaries(env_id):
    """States that land exactly on the goal with zero velocity, and on the wall moving left."""
    goal = M.SPECS[env_id][0]
    # at the goal position with v = 0 and no net push: x stays, v becomes -0.0025 cos(3 goal) +- the push
    phys = np.array([[goal, 0.0], [-1.19, -0.07], [0.59, 0.07]])
    a = np.float32([1.0, 0.0, 2.0]) if env_id == V0 else np.float32([0.0, -1.0, 1.0])
    ph, obs, r, d, *_ = cc.step_kernel(_case(env_id), phys, a, [0, 0, 0])
    wph, _, wr, wd, _, _ = M.step(phys, a, [0, 0, 0], env_id)
    cc.check_phys(ph, wph, ULPS)
    assert ph[1].tolist() == [-1.2, 0.0] and ph[2].tolist() == [0.6, 0.07]
    np.testing.assert_array_equal(d, wd)
    np.testing.assert_array_equal(r, wr)
    assert d[2] and not d[1]


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_reset_seeding_and_sharding(env_id):
    import torch
    from torchrl_b200.env import get_vec_env
    N = 37
    env = get_vec_env(env_id, {}, 2 * N)
    env.seed(5)
    full = env.reset().cpu().numpy()
    seeds = 5 * 2 * N + np.arange(2 * N)
    want = M.reset_phys(seeds, np.zeros(2 * N))
    np.testing.assert_array_equal(env.phys.cpu().numpy(), want)
    np.testing.assert_array_equal(full, M.observe(want))
    parts = []
    for r in range(2):
        e = get_vec_env(env_id, {}, N, first_env=r * N, total_envs=2 * N)
        e.seed(5)
        parts.append(e.reset().cpu().numpy())
    np.testing.assert_array_equal(np.concatenate(parts), full)
    mask = torch.zeros(2 * N, dtype=torch.bool, device="cuda")
    mask[1::4] = True
    before = env.phys.cpu().numpy().copy()
    env.partial_reset(mask)
    after, m = env.phys.cpu().numpy(), mask.cpu().numpy()
    np.testing.assert_array_equal(after[~m], before[~m])
    np.testing.assert_array_equal(after[m], M.reset_phys(seeds[m], np.ones(m.sum())))


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_rollout_tracks_the_oracle_step_by_step(env_id):
    """1000 steps, the scripted controller on half the envs and random actions on the other half: every step against
    the oracle from the device's state, every reset where the oracle ends the episode."""
    import torch
    from torchrl_b200.env import get_vec_env
    N, steps = 64, 1000
    env = get_vec_env(env_id, {"reward_scale": 0.1}, N)
    env.seed(11)
    seeds = 11 * N + np.arange(N)
    env.reset()
    episode = np.ones(N, np.int64)
    phys = env.phys.cpu().numpy().copy()
    el = np.zeros(N, np.int64)
    rs = np.random.RandomState(0)
    n_term = n_limit = 0
    for t in range(steps):
        a = np.where(np.arange(N) < N // 2, M.push(phys, env_id), _actions(N, rs, env_id)).astype(np.float32)
        obs, r, done, info = env.step(torch.as_tensor(a, device="cuda"))
        wph, wobs, wr, wd, wtl, wel = M.step(phys, a, el, env_id, reward_scale=0.1)
        got = env.phys.cpu().numpy().copy()
        cc.check_phys(got, wph, ULPS)
        cc.check_obs(obs.cpu().numpy(), wobs)
        d = done.cpu().numpy().reshape(-1)
        ok = ~_near_goal(wph, env_id)
        np.testing.assert_array_equal(r.cpu().numpy().reshape(-1)[ok], wr[ok])
        np.testing.assert_array_equal(d[ok], wd[ok])
        np.testing.assert_array_equal(info["time_limit"].cpu().numpy(), wtl)
        el = wel
        if d.any():
            n_term += int((d & ~wtl).sum())
            n_limit += int(wtl.sum())
            env.partial_reset(done.reshape(-1))
            got = env.phys.cpu().numpy().copy()
            np.testing.assert_array_equal(got[d], M.reset_phys(seeds[d], episode[d]))
            episode[d] += 1
            el[d] = 0
        phys = got
    assert n_term >= 7 * (N // 2)                                  # the controller reaches the goal every ~110-125 steps
    assert n_limit >= (N // 2 if env_id == V0 else 0)


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_normobs_moments_match_the_chan_formula(env_id):
    import torch
    from torchrl_b200.env import get_vec_env
    N = 1000
    env = get_vec_env(env_id, {"obs_norm": True}, N)
    env.seed(2)
    env.reset()
    nrm = env._obs_normalizer
    mean, var, count = (t.cpu().numpy().astype(np.float64).copy() for t in (nrm._mean, nrm._var, nrm._count))
    for k in range(3):
        act = (np.arange(N) % 3).astype(np.float32) if env_id == V0 else np.linspace(-1, 1, N).astype(np.float32)
        obs, *_ = env.step(torch.as_tensor(act, device="cuda"))
        x = env.state.cpu().numpy().astype(np.float64)
        sums = env.batch_sums.cpu().numpy()
        np.testing.assert_allclose(sums[:2], x.sum(0), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sums[2:], (x * x).sum(0), rtol=1e-12)
        bm, bv = x.mean(0), x.var(0)
        tot = count + N
        delta = bm - mean
        var = (var * count + bv * N + delta ** 2 * count * N / tot) / tot
        mean = mean + delta * N / tot
        count = tot
        np.testing.assert_allclose(nrm._mean.cpu().numpy(), mean, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(nrm._var.cpu().numpy(), var, rtol=1e-9, atol=1e-15)
        np.testing.assert_allclose(nrm._count.cpu().numpy(), count)
        want = np.clip((x - mean) / (np.sqrt(var) + 1e-4), -10, 10)
        np.testing.assert_allclose(obs.cpu().numpy(), want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_refused_action_raises_at_the_next_sync(env_id):
    import torch
    from torchrl_b200.env import get_vec_env
    env = get_vec_env(env_id, {}, 8)
    env.reset()
    before, before_obs = env.phys.clone(), env.state.clone()
    bad = ([0, 1, 0.5, 2, 0, 3, 1, -1] if env_id == V0 else [0, 1, float("nan"), 1, 0, float("inf"), 1, float("-inf")])
    with pytest.raises(ValueError, match="actions 0, 1 and 2" if env_id == V0 else "finite actions"):
        env.step(torch.tensor(bad, device="cuda"))
    for i in (2, 5, 7):
        assert torch.equal(env.phys[i], before[i]) and torch.equal(env.state[i], before_obs[i])
    assert not torch.equal(env.phys[0], before[0])
    env.step(torch.ones(8, device="cuda"))                    # the flag was cleared: valid actions go through
    with pytest.raises(ValueError):
        env.step(torch.full((8,), 7.0 if env_id == V0 else float("nan"), device="cuda"))


def test_spaces_and_routing():
    from torchrl_b200.env import MountainCarVecEnv, get_vec_env
    for env_id, limit in ((V0, 200), (CONT, 999)):
        env = get_vec_env(env_id, {}, 3)
        assert isinstance(env, MountainCarVecEnv) and env._max_episode_steps == limit and not env.lockstep
        np.testing.assert_array_equal(env.observation_space.low, [-1.2, -0.07])
        np.testing.assert_array_equal(env.observation_space.high, [0.6, 0.07])
    assert get_vec_env(V0, {}, 2).action_space.n == 3
    assert get_vec_env(CONT, {}, 2).action_space.shape == (1,)


# ------------------------------------------------------------------------------------------ collector
@pytest.mark.parametrize("env_id", [V0, CONT])
@pytest.mark.parametrize("quirks", [True, False])
@pytest.mark.parametrize("obs_norm", [False, True])
def test_collector_graph_equals_eager(env_id, quirks, obs_norm):
    """The scripted controller ends episodes at different steps in different envs; the captured step and eager steps
    store bit-identical rows, and both leave the envs and the collector in the same state."""
    rows = cc.collector_graph_equals_eager(_case(env_id), quirks, obs_norm, T=100)
    if not obs_norm:
        assert sum(int(r["terminals"].sum()) for r in rows) >= 24          # every env reached the goal at least once


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_collector_rows_match_the_oracle(env_id):
    n_term = cc.collector_rows_match_the_oracle(_case(env_id), 260, ULPS)
    assert n_term >= 2 * 24


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_collector_step_graph_launch_count(env_id):
    cc.collector_launch_count(_case(env_id))


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_eval_returns_the_oracles_episode_returns(env_id):
    col, buf, env = cc.collector(_case(env_id), True, True, False, N=16)
    col.eval_env.seed(42)
    ev = col.eval_one_epoch()
    ret, length, reached = M.episodes(lambda s: M.push(s, env_id), M.reset_phys(42 * 16 + np.arange(16),
                                                                                 np.zeros(16)), env_id)
    assert reached.all()
    np.testing.assert_allclose(ev["eval_rewards"], ret, rtol=1e-6, atol=1e-4)
    if env_id == V0:
        assert ev["eval_rewards"] == ret.tolist()
    assert ev["eval_traj_length"] == float(length.mean())


# ------------------------------------------------------------------------------------------ agents
@pytest.mark.parametrize("kind", ["dqn", "qrdqn", "ppo", "a2c", "reinforce"])
def test_one_epoch_of_each_discrete_agent(kind):
    agent, col, buf, env = cc.discrete_agent(V0, kind, 2)
    out = cc.one_epoch(agent, col, kind, kind in ("dqn", "qrdqn"))
    assert all(-200 <= r <= 0 for r in out["train_rewards"])
    acts = buf._acts.cpu().numpy()
    assert set(np.unique(acts[:buf._size])) <= {0.0, 1.0, 2.0}
    ev = col.eval_one_epoch()
    assert len(ev["eval_rewards"]) == 16 and all(-200 <= r <= 0 for r in ev["eval_rewards"])


@pytest.mark.parametrize("kind", ["td3", "ddpg", "sac", "twin_sac_q", "ppo"])
def test_one_epoch_of_each_continuous_agent(kind):
    agent, col, buf, env = cc.continuous_agent(CONT, kind, 2, 999, True)
    out = cc.one_epoch(agent, col, kind, kind != "ppo")
    assert all(-0.1 * 999 - 1e-3 <= r <= 100 for r in out["train_rewards"])
    acts = buf._acts.cpu().numpy()
    assert np.all(np.abs(acts[:buf._size]) <= 1.0)
    ev = col.eval_one_epoch()
    assert len(ev["eval_rewards"]) == 16 and 1 <= ev["eval_traj_length"] <= 999
