"""The device Acrobot-v1 (csrc/acrobot.cu, torchrl_b200/env/acrobot.py) against its NumPy statement (oracle/acrobot.py):
single steps from random and boundary states over ragged batch sizes, a long rollout re-synchronised every step,
resets, sharded seeding, the NormObs moments, invalid actions, the collector with the env's own reset inside the
captured step (graph == eager, rows against the oracle, launch counts), evaluation, one epoch of each discrete agent,
and a DQN resume.

Tolerance of the fp64 state: the kernel and NumPy differ only in `sin` / `cos` (CUDA's fp64 sin / cos are within 2 ulp,
NumPy's within 1).  One Acrobot step evaluates them 16 times inside RK4, and each stage feeds its error into the next:
the accelerations hold dtheta^2 sin(theta2) terms, so at the velocity bounds (9 pi: dtheta^2 near 800) a last-bit
difference in a sine becomes a difference in the acceleration hundreds of times larger, which dt / 2 carries into the
next stage's state, three times over.  On an H100 the largest difference seen was 206 ulp of max(|x|, 1) over the 257
random states and 46,728 ulp (1.6e-10 absolute, in dtheta2 near 27) over the 100,003 states that include envs at the
velocity bounds; about 89 % of the components were bit-identical.  The check allows ULPS = 2^17 ulp and requires 85 %
bit-identical components.  A state error of 1.6e-10 moves the tip's height by less than 1e-9, so rewards and done
flags must be identical except within 1e-9 of the goal line; fp32 observations must be equal or one ulp apart."""
import math

import numpy as np
import pytest

from oracle import acrobot as A
from tests import classic_control_gpu as cc

pytestmark = pytest.mark.gpu

ULPS = 1 << 17


def _controller(ob):
    """oracle/acrobot.py's pump on the fp32 observation: torque along dtheta2 - dtheta1 - sin theta2."""
    import torch
    return (1.0 + torch.sign(ob[:, 5] - ob[:, 4] - ob[:, 3])).float()


def _case():
    from torchrl_b200 import ops
    return cc.Case("Acrobot-v1", 4, 6, A.step, A.reset_phys, A.observe, _controller, ops.acrobot_step,
                   near_goal=_near_goal)


def _states(N, rs):
    """Random states with boundary cases: the angle ends, the velocity bounds, fast states whose angles wrap more than
    once, states near the goal line, and resets."""
    pi = math.pi
    phys = np.stack([rs.uniform(-pi, pi, N), rs.uniform(-pi, pi, N), rs.uniform(-4 * pi, 4 * pi, N),
                     rs.uniform(-9 * pi, 9 * pi, N)], 1)
    pick = rs.randint(0, 6, N)
    phys[pick == 0, :2] = rs.choice([pi, -pi, 0.0], (int((pick == 0).sum()), 2))
    phys[pick == 1, 2:] = rs.choice([-1, 1], (int((pick == 1).sum()), 2)) * np.array([4 * pi, 9 * pi])
    phys[pick == 2] = rs.uniform(-0.1, 0.1, (int((pick == 2).sum()), 4))
    near = pick == 3                                         # link 1 near upright: the tip near the goal line
    phys[near, 0] = pi + rs.uniform(-0.6, 0.6, int(near.sum()))
    phys[near, 1] = rs.uniform(-1.5, 1.5, int(near.sum()))
    return phys


def _near_goal(phys):
    return np.abs(A.goal_height(phys) - 1.0) < 1e-9


@pytest.mark.parametrize("N", [1, 255, 256, 257, 100003])
def test_step_matches_oracle(N):
    rs = np.random.RandomState(N)
    phys = _states(N, rs)
    a = rs.randint(0, 3, N).astype(np.float32)
    el = rs.randint(0, 500, N)
    el[rs.rand(N) < 0.3] = 499
    reward_scale = 0.5 if N % 2 else 1.0
    ph, obs, r, d, tl, el2, err, any_reset = cc.step_kernel(_case(), phys, a, el, reward_scale, 500)
    wph, wobs, wr, wd, wtl, wel = A.step(phys, a, el, reward_scale=reward_scale)
    assert err == 0
    worst = cc.check_phys(ph, wph, ULPS)
    print("acrobot step N=%d: largest state error %.1f ulp, bit-identical %.3f" % (N, worst, np.mean(ph == wph)))
    if N >= 255:
        assert np.mean(ph == wph) >= 0.85
    cc.check_obs(obs, wobs)
    cc.check_obs(obs, A.observe(ph))
    ok = ~_near_goal(wph)
    np.testing.assert_array_equal(r[ok], wr[ok])
    np.testing.assert_array_equal(d[ok], wd[ok])
    np.testing.assert_array_equal(tl, wtl)
    np.testing.assert_array_equal(el2, wel)
    assert any_reset[0] == int(d.any())
    assert np.all(np.abs(ph[:, :2]) <= math.pi)
    if N == 100003:
        assert (np.abs(ph[:, 3]) == 9 * math.pi).sum() > 100 and (wd & ~wtl).sum() > 1000


def test_step_from_rest_moves_by_the_cosine_residue():
    ph, obs, r, d, *_ = cc.step_kernel(_case(), np.zeros((2, 4)), [1.0, 2.0], [0, 0])
    want, _ = A.dynamics(np.zeros((2, 4)), [1.0, 2.0])
    cc.check_phys(ph, want, 4)
    assert np.all(ph[0] != 0.0) and np.abs(ph[0]).max() < 1e-15 and ph[0, 0] < 0
    assert r.tolist() == [-1.0, -1.0] and not d.any()


def test_reset_seeding_and_sharding():
    import torch
    from torchrl_b200.env import get_vec_env
    N = 37
    env = get_vec_env("Acrobot-v1", {}, 2 * N)
    env.seed(5)
    full = env.reset().cpu().numpy()
    seeds = 5 * 2 * N + np.arange(2 * N)
    want = A.reset_phys(seeds, np.zeros(2 * N))
    np.testing.assert_array_equal(env.phys.cpu().numpy(), want)
    cc.check_obs(full, A.observe(want))
    parts, pphys = [], []
    for r in range(2):
        e = get_vec_env("Acrobot-v1", {}, N, first_env=r * N, total_envs=2 * N)
        e.seed(5)
        parts.append(e.reset().cpu().numpy())
        pphys.append(e.phys.cpu().numpy())
    np.testing.assert_array_equal(np.concatenate(parts), full)
    np.testing.assert_array_equal(np.concatenate(pphys), env.phys.cpu().numpy())
    env.reset()
    np.testing.assert_array_equal(env.phys.cpu().numpy(), A.reset_phys(seeds, np.ones(2 * N)))
    mask = torch.zeros(2 * N, dtype=torch.bool, device="cuda")
    mask[::3] = True
    before, before_obs = env.phys.cpu().numpy().copy(), env.state.cpu().numpy().copy()
    raw = env.partial_reset(mask).cpu().numpy()
    after = env.phys.cpu().numpy()
    m = mask.cpu().numpy()
    np.testing.assert_array_equal(after[~m], before[~m])
    np.testing.assert_array_equal(raw[~m], before_obs[~m])
    np.testing.assert_array_equal(after[m], A.reset_phys(seeds[m], np.full(m.sum(), 2)))
    cc.check_obs(raw[m], A.observe(after[m]))


def test_rollout_tracks_the_oracle_step_by_step():
    """1000 steps of the scripted controller on half the envs and random actions on the other half: every step against
    the oracle from the device's state, every terminal reset where the oracle ends the episode."""
    import torch
    from torchrl_b200.env import get_vec_env
    N, steps = 64, 1000
    env = get_vec_env("Acrobot-v1", {"reward_scale": 0.1}, N)
    env.seed(11)
    seeds = 11 * N + np.arange(N)
    env.reset()
    episode = np.ones(N, np.int64)
    phys = env.phys.cpu().numpy().copy()
    el = np.zeros(N, np.int64)
    rs = np.random.RandomState(0)
    n_term = n_limit = 0
    for t in range(steps):
        a = np.where(np.arange(N) < N // 2, A.pump(phys), rs.randint(0, 3, N)).astype(np.float32)
        obs, r, done, info = env.step(torch.as_tensor(a, device="cuda"))
        wph, wobs, wr, wd, wtl, wel = A.step(phys, a, el, reward_scale=0.1)
        got = env.phys.cpu().numpy().copy()
        cc.check_phys(got, wph, ULPS)
        cc.check_obs(obs.cpu().numpy(), wobs)
        d = done.cpu().numpy().reshape(-1)
        ok = ~_near_goal(wph)
        np.testing.assert_array_equal(r.cpu().numpy().reshape(-1)[ok], wr[ok])
        np.testing.assert_array_equal(d[ok], wd[ok])
        np.testing.assert_array_equal(info["time_limit"].cpu().numpy(), wtl)
        el = wel
        if d.any():
            n_term += int((d & ~wtl).sum())
            n_limit += int(wtl.sum())
            env.partial_reset(done.reshape(-1))
            got = env.phys.cpu().numpy().copy()
            np.testing.assert_array_equal(got[d], A.reset_phys(seeds[d], episode[d]))
            episode[d] += 1
            el[d] = 0
        phys = got
    assert n_term > 5 * (N // 2) and n_limit > 0                   # the controller's envs end many episodes early


def test_normobs_moments_match_the_chan_formula():
    import torch
    from torchrl_b200.env import get_vec_env
    N = 1000
    env = get_vec_env("Acrobot-v1", {"obs_norm": True}, N)
    env.seed(2)
    env.reset()
    nrm = env._obs_normalizer
    mean, var, count = (t.cpu().numpy().astype(np.float64).copy() for t in (nrm._mean, nrm._var, nrm._count))
    for k in range(3):
        act = (np.arange(N) % 3).astype(np.float32)
        obs, *_ = env.step(torch.as_tensor(act, device="cuda"))
        x = env.state.cpu().numpy().astype(np.float64)
        sums = env.batch_sums.cpu().numpy()
        np.testing.assert_allclose(sums[:6], x.sum(0), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sums[6:], (x * x).sum(0), rtol=1e-12)
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
    env = get_vec_env("Acrobot-v1", {}, 8)
    env.reset()
    before, before_obs = env.phys.clone(), env.state.clone()
    with pytest.raises(ValueError, match="actions 0, 1 and 2"):
        env.step(torch.tensor([0, 1, 0.5, 2, 0, 3, 1, float("nan")], device="cuda"))
    for i in (2, 5, 7):
        assert torch.equal(env.phys[i], before[i]) and torch.equal(env.state[i], before_obs[i])
    assert not torch.equal(env.phys[0], before[0])
    env.step(torch.ones(8, device="cuda"))                    # the flag was cleared: valid actions go through
    with pytest.raises(ValueError):
        env.step(torch.full((8,), -1.0, device="cuda"))


def test_spaces_and_routing():
    from torchrl_b200.env import AcrobotVecEnv, get_vec_env
    env = get_vec_env("Acrobot-v1", {}, 3)
    assert isinstance(env, AcrobotVecEnv) and env._max_episode_steps == 500 and not env.lockstep
    assert env.observation_space.shape == (6,) and env.action_space.n == 3
    np.testing.assert_array_equal(env.observation_space.high, [1, 1, 1, 1, 4 * math.pi, 9 * math.pi])


# ------------------------------------------------------------------------------------------ collector
@pytest.mark.parametrize("quirks", [True, False])
@pytest.mark.parametrize("obs_norm", [False, True])
def test_collector_graph_equals_eager(quirks, obs_norm):
    """The scripted controller ends episodes at different steps in different envs; the captured step and eager steps
    store bit-identical rows, and both leave the envs and the collector in the same state."""
    rows = cc.collector_graph_equals_eager(_case(), quirks, obs_norm, T=64)
    term = sum(int(r["terminals"].sum()) for r in rows)
    assert term > 24                                                 # terminal resets happened inside the epochs


def test_collector_rows_match_the_oracle():
    n_term = cc.collector_rows_match_the_oracle(_case(), 400, ULPS)
    assert n_term >= 24


def test_collector_step_graph_launch_count():
    cc.collector_launch_count(_case())


def test_eval_returns_the_episode_returns():
    """eval_one_epoch with the scripted controller returns the returns of the same episodes run step by step, and
    those episodes end where the oracle's step from the device's state ends them."""
    import torch
    col, buf, env = cc.collector(_case(), True, True, False, N=16)
    col.eval_env.seed(42)
    ev = col.eval_one_epoch()
    rets = np.array(ev["eval_rewards"])
    assert len(rets) == 16 and np.all(rets <= 0) and np.all(rets == np.round(rets))
    # the same episodes, step by step on a fresh env with the same seed
    from torchrl_b200.env import get_vec_env
    e = get_vec_env("Acrobot-v1", {}, 16)
    e.seed(42)
    ob = e.reset()
    ret, live = np.zeros(16), np.ones(16, bool)
    for _ in range(500):
        phys = e.phys.cpu().numpy().copy()
        a = _controller(ob)
        ob, r, d, info = e.step(a)
        _, term = A.dynamics(phys, a.cpu().numpy())
        dd = d.cpu().numpy().reshape(-1)
        ok = ~_near_goal(e.phys.cpu().numpy())
        np.testing.assert_array_equal(dd[ok], (term | info["time_limit"].cpu().numpy())[ok])
        ret += np.where(live, r.cpu().numpy().reshape(-1), 0.0)
        live &= ~dd
        if not live.any():
            break
        if dd.any():
            ob = e.partial_reset(torch.as_tensor(dd, device="cuda"))
    np.testing.assert_array_equal(rets, ret)
    assert (rets > -500).mean() >= 0.9                            # the controller lifts the tip in most episodes


# ------------------------------------------------------------------------------------------ agents
@pytest.mark.parametrize("kind", ["dqn", "qrdqn", "ppo", "a2c", "reinforce"])
def test_one_epoch_of_each_agent(kind):
    agent, col, buf, env = cc.discrete_agent("Acrobot-v1", kind, 6)
    out = cc.one_epoch(agent, col, kind, kind in ("dqn", "qrdqn"))
    assert all(-500 <= r <= 0 for r in out["train_rewards"])
    acts = buf._acts.cpu().numpy()
    assert set(np.unique(acts[:buf._size])) <= {0.0, 1.0, 2.0}
    ev = col.eval_one_epoch()
    assert len(ev["eval_rewards"]) == 16 and all(-500 <= r <= 0 for r in ev["eval_rewards"])


def test_dqn_resume_continues_identically(tmp_path):
    import torch
    path = str(tmp_path / "ck.pt")

    def epochs(agent, col, first, n):
        out = []
        for e in range(first, first + n):
            agent.current_epoch = e
            out.append(col.train_one_epoch()["train_epoch_reward"])
            agent.update_per_epoch()
        return out

    agent, col, buf, env = cc.discrete_agent("Acrobot-v1", "dqn", 6, seed=1, use_graph=False)
    agent.pretrain()
    epochs(agent, col, 0, 3)                                      # mid-episode at the checkpoint
    agent.save_checkpoint(path)
    want_r = epochs(agent, col, 3, 3)
    want, want_t, want_phys = agent.opt.data.clone(), agent._target_flat.data.clone(), env.phys.clone()
    agent2, col2, buf2, env2 = cc.discrete_agent("Acrobot-v1", "dqn", 6, seed=77, use_graph=False)
    assert agent2.load_checkpoint(path) == 3
    got_r = epochs(agent2, col2, 3, 3)
    np.testing.assert_allclose(got_r, want_r, rtol=1e-6)
    assert torch.equal(env2.phys, want_phys)
    torch.testing.assert_close(agent2.opt.data, want, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(agent2._target_flat.data, want_t, rtol=1e-5, atol=1e-7)
