"""Atari games through the host chain, GPU side: the WarpFrame + FrameStack kernel bit for bit against the NumPy
restatement (oracle/atari_frames.py) and OpenCV's outputs (tests/golden/atari_frames.npz), its argument checks, the
to_float map, DQN and PPO epochs over host envs (in process and in two worker processes) whose ring rows equal the
oracle chain replayed with the same actions, the launches of a host step, and DQN learning the fake game."""
import os

import numpy as np
import pytest

from oracle import atari_frames as af
from oracle import fake_ale

pytestmark = pytest.mark.gpu

ENV_ID = "FakeAleNoFrameskip-v4"
GAME = dict(fire=True, lives=3, hazard=41, max_episode_steps=150)


def make_fake(env_id):
    """Top-level (picklable) `make` hook: the fake game, short enough that lives, game overs and time limits occur."""
    return fake_ale.make(env_id, **GAME)


def make_learn(env_id):
    return fake_ale.make(env_id, fire=True, lives=3, hazard=97, max_episode_steps=2000)


def _frames(golden_dir, H, M, rs):
    z = np.load(os.path.join(golden_dir, "atari_frames.npz"))
    base = z["rgb_%d" % H]
    noise = rs.randint(0, 256, (max(M - len(base), 0),) + base.shape[1:]).astype(np.uint8)
    return np.concatenate([base, noise])[:M], z["warp_%d" % H]


def _tables(H, W):
    import torch
    from torchrl_b200.env.atari_host import area_tables
    ti, tw = area_tables(H, W)
    return torch.from_numpy(ti).cuda(), torch.from_numpy(tw).cuda()


@pytest.mark.parametrize("H", [210, 250])
@pytest.mark.parametrize("N", [1, 7, 512])
@pytest.mark.parametrize("fresh", ["all", "none", "mixed"])
def test_warp_stack_bit_exact(golden_dir, H, N, fresh):
    import torch
    from torchrl_b200 import ops
    rs = np.random.RandomState(N + H)
    frames, golden = _frames(golden_dir, H, N, rs)
    W, C = 160, 4
    want_warp = af.warp(frames)
    k = min(N, len(golden))
    np.testing.assert_array_equal(want_warp[:k], golden[:k])
    stack0 = rs.randint(0, 256, (N, C, 84, 84)).astype(np.uint8)
    mask = {"all": np.ones(N, bool), "none": np.zeros(N, bool), "mixed": rs.rand(N) < 0.5}[fresh]
    want = stack0.copy()
    for n in range(N):
        af.stack_update(want[n], want_warp[n], mask[n])
    stack = torch.from_numpy(stack0).cuda()
    ti, tw = _tables(H, W)
    before = ops._lib.launch_count()
    ops.atari_warp_stack(torch.from_numpy(frames).cuda(), stack, ti, tw,
                         fresh=torch.from_numpy(mask.astype(np.uint8)).cuda())
    assert ops._lib.launch_count() - before == 1
    np.testing.assert_array_equal(stack.cpu().numpy(), want)
    # packed frames of some envs (partial reset): only those stacks are refilled
    idx = np.flatnonzero(mask)
    if idx.size:
        want2 = want.copy()
        want2[idx] = want_warp[::-1][:idx.size][:, None]
        ops.atari_warp_stack(torch.from_numpy(frames[::-1][:idx.size].copy()).cuda(), stack, ti, tw,
                             env_idx=torch.from_numpy(idx.astype(np.int32)).cuda())
        np.testing.assert_array_equal(stack.cpu().numpy(), want2)
    # no mask: every env fresh
    ops.atari_warp_stack(torch.from_numpy(frames).cuda(), stack, ti, tw)
    np.testing.assert_array_equal(stack.cpu().numpy(), np.repeat(want_warp[:, None], C, axis=1))


def test_warp_stack_rejects_malformed_shapes():
    import torch
    from torchrl_b200 import _lib, ops
    ti, tw = _tables(210, 160)
    stack = torch.zeros(2, 4, 84, 84, dtype=torch.uint8, device="cuda")
    good = torch.zeros(2, 210, 160, 3, dtype=torch.uint8, device="cuda")
    for H, W in ((83, 160), (210, 83), (210, 100), (1500, 160)):           # too small, 3W % 16 != 0, smem too big
        f = torch.zeros(2, H, W, 3, dtype=torch.uint8, device="cuda")
        with pytest.raises(RuntimeError, match=r"rc=-1"):
            ops.atari_warp_stack(f, stack, ti, tw)
    with pytest.raises(RuntimeError, match=r"rc=-1.*M == N"):
        ops.atari_warp_stack(good[:1], stack, ti, tw)
    with pytest.raises(RuntimeError, match=r"rc=-1.*16-byte"):
        _lib.call("trl_atari_warp_stack", good.view(-1)[1:], None, None, stack, ti, tw, 2, 2, 210, 160, 4, 0)
    with pytest.raises(ValueError):
        ops.atari_warp_stack(good, torch.zeros(2, 4, 84, 80, dtype=torch.uint8, device="cuda"), ti, tw)
    with pytest.raises(RuntimeError, match=r"rc=-1.*multiple of 4"):
        _lib.call("trl_u8_lut_f32", good, torch.zeros(3, device="cuda"), 3, torch.zeros(256, device="cuda"), 0)


@pytest.mark.parametrize("scale", [True, False])
def test_to_float_is_the_lut(scale):
    import torch
    from torchrl_b200 import ops
    from torchrl_b200.env.atari_host import frame_lut
    x = torch.randint(0, 256, (3, 4, 84, 84), dtype=torch.uint8, device="cuda")
    x.view(-1)[:256] = torch.arange(256, device="cuda").to(torch.uint8)
    out = ops.u8_lut_f32(x, torch.from_numpy(frame_lut(scale)).cuda())
    np.testing.assert_array_equal(out.cpu().numpy(), af.lut(scale)[x.cpu().numpy()])


# ---------------------------------------------------------------------------------------------------- collectors
def _env(N, procs, param, make=make_fake):
    from torchrl_b200.env import get_subprocvec_env, get_vec_env
    if procs:
        return get_subprocvec_env(ENV_ID, param, N, procs, device="cuda", make=make)
    return get_vec_env(ENV_ID, param, N, device="cuda", make=make)


class OracleChain:
    """The product's host chain in this process, through the oracle's WarpFrame + FrameStack."""

    def __init__(self, N, param):
        from torchrl_b200.hostenv import VecEnv, get_atari_env
        self.venv = VecEnv(N, get_atari_env, [ENV_ID, param, make_fake])

    def reset(self, seed):
        self.venv.seed(seed)
        self.stack = np.repeat(af.warp(np.asarray(self.venv.reset()))[:, None], 4, axis=1)

    def step(self, acts):
        ob, r, d, info = self.venv.step(acts)
        self.stack = np.concatenate([self.stack[:, 1:], af.warp(np.asarray(ob))[:, None]], axis=1)
        return np.array(r)[:, 0], np.array(d)[:, 0], np.array(info["time_limit"])

    def partial_reset(self, mask):
        ob = np.asarray(self.venv.partial_reset(mask))
        self.stack[mask] = af.warp(ob[mask])[:, None]


def _check_rows(buf, T, N, param, max_frames, on_policy, seed=0):
    """Every stored row against the oracle chain replayed with the stored actions and the collector's resets."""
    ora = OracleChain(N, param)
    ora.reset(seed)
    obs, nxt = buf._obs.cpu().numpy(), buf._next_obs.cpu().numpy()
    acts = buf._acts.cpu().numpy().reshape(-1, N)
    rew, term, tl = (getattr(buf, k).cpu().numpy().reshape(-1, N) for k in ("_rewards", "_terminals", "_time_limits"))
    steps = np.zeros(N, np.int64)
    events = 0
    for t in range(T):
        np.testing.assert_array_equal(obs[t], ora.stack)
        r, d, l = ora.step(acts[t].astype(np.int64))
        np.testing.assert_array_equal(nxt[t], ora.stack)
        steps += 1
        cut = steps >= max_frames
        np.testing.assert_array_equal(term[t].astype(bool), d | (cut if on_policy else False))
        np.testing.assert_array_equal(tl[t].astype(bool), l)
        keep = ~cut if on_policy else np.ones(N, bool)          # on-policy cut rows hold r + discount * V(next)
        np.testing.assert_array_equal(rew[t][keep], r.astype(np.float32)[keep])
        mask = d | cut
        events += int(mask.sum())
        if mask.any():
            ora.partial_reset(mask)
        steps[mask] = 0
    ora.venv.close()
    return events


def _dqn(env, eval_env, N, T, max_frames, rows=None, lr=1e-3, decay=100, discount=0.99, opt_times=4):
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import DQN
    from torchrl_b200.collector import PixelVecCollector
    from torchrl_b200.replay_buffers import BaseReplayBuffer
    from torchrl_b200.utils import NullLogger
    A = env.action_space.n
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=(rows or T) * N)
    qf = networks.Net(input_shape=(4, 84, 84), output_shape=A,
                      hidden_shapes=[[16, [8, 8], [4, 4], [0, 0]], [32, [4, 4], [2, 2], [0, 0]]],
                      append_hidden_shapes=[64], base_type=networks.CNNBase, activation_func=nn.ReLU)
    pf = policies.EpsilonGreedyDQNDiscretePolicy(qf=qf, start_epsilon=1.0, end_epsilon=0.05, decay_frames=decay,
                                                 action_shape=A)
    col = PixelVecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=torch.device("cuda:0"),
                            epoch_frames=T * N, max_episode_frames=max_frames)
    agent = DQN(qf=qf, pf=pf, qlr=lr, optimizer_info={"eps": 1e-4}, env=env, replay_buffer=buf, collector=col,
                logger=NullLogger(), discount=discount, batch_size=64, device=torch.device("cuda:0"), save_dir=None,
                opt_times=opt_times, use_soft_update=False, target_hard_update_period=20, pretrain_epochs=1,
                num_epochs=2)
    return agent, col, buf


@pytest.mark.parametrize("procs", [0, 2])
def test_dqn_epoch_rows_equal_the_oracle_chain(procs):
    import torch
    N, T, max_frames = 4, 40, 9
    param = {"frame_stack": True, "scale": True, "clip_rewards": True}
    env, eval_env = _env(N, procs, param), _env(N, procs, param)
    try:
        env.seed(0)
        torch.manual_seed(0)
        agent, col, buf = _dqn(env, eval_env, N, T, max_frames)
        col.train_one_epoch()
        agent.update_per_epoch()
        assert all(np.isfinite(i["Training/qf_loss"]) for i in agent._last_infos)
        assert _check_rows(buf, T, N, param, max_frames, on_policy=False) > 0
        out = col.eval_one_epoch()
        assert len(out["eval_rewards"]) == N and np.all(np.isfinite(out["eval_rewards"]))
    finally:
        env.close()
        eval_env.close()


@pytest.mark.parametrize("procs", [0, 2])
def test_ppo_epoch_rows_equal_the_oracle_chain(procs):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import PPO
    from torchrl_b200.collector import VecOnPolicyCollector
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    from torchrl_b200.utils import NullLogger
    N, T, max_frames = 4, 32, 11
    param = {"frame_stack": True, "scale": False, "clip_rewards": False}
    env, eval_env = _env(N, procs, param), _env(N, procs, param)
    try:
        env.seed(0)
        torch.manual_seed(0)
        dev = torch.device("cuda:0")
        buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
        net = dict(input_shape=(4, 84, 84), hidden_shapes=[[16, [8, 8], [4, 4], [0, 0]], [32, [4, 4], [2, 2], [0, 0]]],
                   append_hidden_shapes=[16], base_type=networks.CNNBase, activation_func=torch.nn.Tanh)
        pf = policies.CategoricalDisPolicy(output_shape=env.action_space.n, **net)
        vf = networks.Net(output_shape=1, **net)
        col = VecOnPolicyCollector(vf, env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev,
                                   epoch_frames=T * N, max_episode_frames=max_frames)
        agent = PPO(pf=pf, vf=vf, env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99,
                    num_epochs=2, batch_size=2 * N, gae=True, device=dev, save_dir=None, shuffle=True, tau=0.95,
                    plr=3e-4, vlr=3e-4, entropy_coeff=0.01, clip_para=0.1, opt_epochs=1)
        col.train_one_epoch()
        agent.process_epoch_samples()
        assert _check_rows(buf, T, N, param, max_frames, on_policy=True) > 0
        agent.update_per_epoch()
        out = col.eval_one_epoch()
        assert len(out["eval_rewards"]) == N
    finally:
        env.close()
        eval_env.close()


def test_frame_deduplicated_ring_is_refused():
    import torch
    from torchrl_b200.replay_buffers import MemoryEfficientReplayBuffer
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.collector import PixelVecCollector
    param = {"frame_stack": True}
    env, eval_env = _env(2, 0, param), _env(2, 0, param)
    qf = networks.Net(input_shape=(4, 84, 84), output_shape=4, hidden_shapes=[[16, [8, 8], [4, 4], [0, 0]]],
                      append_hidden_shapes=[16], base_type=networks.CNNBase, activation_func=torch.nn.ReLU)
    pf = policies.EpsilonGreedyDQNDiscretePolicy(qf=qf, start_epsilon=1.0, end_epsilon=0.1, decay_frames=10,
                                                 action_shape=4)
    with pytest.raises(NotImplementedError, match="de-duplicated"):
        PixelVecCollector(env=env, eval_env=eval_env, pf=pf, device=torch.device("cuda:0"), epoch_frames=8,
                          replay_buffer=MemoryEfficientReplayBuffer(env_nums=2, max_replay_buffer_size=16))
    with pytest.raises(TypeError, match="eval_env"):
        PixelVecCollector(env=env, pf=pf, device=torch.device("cuda:0"), epoch_frames=8,
                          replay_buffer=MemoryEfficientReplayBuffer(env_nums=2, max_replay_buffer_size=16))
    env.close()
    eval_env.close()


def test_launches_per_host_step():
    """env.launch_step is one launch (the frame kernel) and partial_reset one more when an env is masked, none
    otherwise; a collector host step launches what the eager device-env step launches with the env's step and its
    in-graph reset replaced by those."""
    import torch
    from torchrl_b200 import _lib
    from torchrl_b200.env import get_vec_env
    N = 4
    env = _env(N, 0, {"frame_stack": True})
    env.seed(0)
    env.reset()
    acts = torch.zeros(N, device="cuda")
    for fn, n in ((lambda: env.launch_step(acts), 1), (lambda: env.partial_reset(np.zeros(N, bool)), 0),
                  (lambda: env.partial_reset(np.eye(N, dtype=bool)[1]), 1)):
        before = _lib.launch_count()
        fn()
        assert _lib.launch_count() - before == n
    # the same DQN step on SynthAtari (eager) and on the host env, with and without a reset on the host step
    host_agent = _dqn(env, _env(N, 0, {"frame_stack": True}), N, 4, 2)
    syn = get_vec_env("SynthAtari-v0", {}, N)
    syn_agent = _dqn(syn, get_vec_env("SynthAtari-v0", {}, N), N, 4, 2)
    syn_agent[1].use_cuda_graph = False
    counts, resets = [], []
    for col in (syn_agent[1], host_agent[1]):
        for k in range(2):
            before = _lib.launch_count()
            col._step()
            counts.append(_lib.launch_count() - before)
            resets.append(bool(env.host_done.any()) or k == 1)     # a life lost, or the cut at max frames 2
    # synth: env step + in-graph reset on every step; host: the frame launch, plus one on steps where an env resets
    assert counts[0] == counts[1] and counts[2] == counts[0] - 1 + resets[2] and counts[3] == counts[0] - 1 + 1, \
        (counts, resets)
    env.close()


def test_dqn_learns_the_fake_game():
    """Greedy evaluation over the first life passes the midpoint between a random policy's return (0) and the
    optimal one (fake_ale.optimal_first_life_return).  On an H100 the first evaluation, after 4 epochs, scored 19.1
    against a target of 9.4; the budget of 24 epochs leaves a wide margin."""
    import torch
    N, T, epochs = 16, 50, 24
    param = {"frame_stack": True, "scale": True, "clip_rewards": True}
    env, eval_env = _env(N, 0, param, make_learn), _env(8, 0, param, make_learn)
    env.seed(0)
    eval_env.seed(123)
    torch.manual_seed(0)
    np.random.seed(0)
    agent, col, buf = _dqn(env, eval_env, N, T, 10 ** 6, rows=200, lr=5e-4, decay=T * 6, discount=0.9,
                           opt_times=T)
    agent.pretrain()
    best, hist = -1e9, []
    target = 0.5 * (0.0 + fake_ale.optimal_first_life_return(97))
    for epoch in range(epochs):
        agent.current_epoch = epoch
        col.train_one_epoch()
        agent.update_per_epoch()
        if epoch % 4 == 3:
            ret = float(np.mean(col.eval_one_epoch()["eval_rewards"]))
            hist.append(ret)
            best = max(best, ret)
            if ret > target:
                break
    print("dqn eval returns", hist, "target", target)
    env.close()
    eval_env.close()
    assert best > target, (hist, target)
