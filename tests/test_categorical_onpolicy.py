"""Discrete on-policy path on the device: A2C / PPO with CategoricalDisPolicy against the reference's own updates
(tests/golden/categorical_reference.npz, oracle/make_golden_categorical.py; tolerances of test_onpolicy_algos.py), the
captured-graph epoch loop against the eager one, the uint8 on-policy pixel collector, evaluation on pixel envs,
checkpoint resume, and the reference's discrete Atari examples run unmodified."""
import os

import numpy as np
import pytest

from oracle import make_golden_categorical as gold
from oracle import synth_atari as oa

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "categorical_reference.npz")


class _Logger:
    def __init__(self):
        self.infos = []

    def add_update_info(self, info):
        self.infos.append(info)

    def add_epoch_info(self, *a, **k):
        pass

    def log(self, *a):
        pass

    def finish(self):
        pass


class _Col:
    epoch_frames = 64


def _state(rec, net):
    import torch
    return {k[len(net) + 1:]: torch.as_tensor(v) for k, v in rec.items() if k.startswith(net + ".")}


def _device_agent(kind, arch, init):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import A2C, PPO
    from torchrl_b200.spaces import Box, Discrete

    class Env:
        action_space = Discrete(gold.A)
        observation_space = Box(-np.ones(11), np.ones(11))
    kw = gold.net_kwargs(networks, torch, arch)
    pf = policies.CategoricalDisPolicy(output_shape=gold.A, **kw)
    vf = networks.Net(output_shape=1, **kw)
    pf.load_state_dict(_state(init, "pf"))
    vf.load_state_dict(_state(init, "vf"))
    cls = {"a2c": A2C, "ppo": PPO}[kind]
    return cls(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=_Col(), logger=_Logger(), discount=0.99,
               num_epochs=10, batch_size=64, gae=True, device="cuda:0", save_dir=None, shuffle=True, tau=0.95,
               use_cuda_graph=False, **gold.KW[kind])


@pytest.mark.parametrize("case", sorted(gold.CASES))
def test_update_matches_reference(case):
    import torch
    kind, arch, n, B, seed = gold.CASES[case]
    ref = gold.load(GOLDEN)
    r = ref[case]
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # cuDNN's TF32 convolutions would dominate the error
    try:
        mine = _device_agent(kind, arch, ref[arch]["init"])
        infos = [mine.update(b) for b in gold.batches(arch, n, B, seed)]
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    for u, m in enumerate(infos):
        want = r["info%d" % u]
        assert set(want) == set(m), (sorted(want), sorted(m))
        for k, v in want.items():
            assert abs(m[k] - v) <= 2e-3 * abs(v) + 2e-4, (u, k, m[k], v)
    if kind == "ppo":
        assert not any(k.startswith("log_std/") for k in infos[0])
    else:
        assert not any(k.startswith("std/") for k in infos[0])
    for net in ("pf", "vf"):
        for k, v in getattr(mine, net).state_dict().items():
            np.testing.assert_allclose(v.detach().cpu().numpy(), r["final"]["%s.%s" % (net, k)], atol=2e-4,
                                       err_msg=k)


def _pixel_agent(kind, N=16, T=8, use_graph=True, seed=0, max_frames=5, batch_rows=4, hidden=None):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import A2C, PPO
    from torchrl_b200.collector import VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    dev = torch.device("cuda:0")
    env = get_vec_env("SynthAtari-v0", {}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    net = dict(input_shape=(4, 84, 84), hidden_shapes=hidden or gold.CNN["hidden"], append_hidden_shapes=[16],
               base_type=networks.CNNBase, activation_func=torch.nn.Tanh)
    pf = policies.CategoricalDisPolicy(output_shape=6, **net)
    vf = networks.Net(output_shape=1, **net)
    col = VecOnPolicyCollector(vf, env=env, pf=pf, replay_buffer=buf, device=dev, train_render=False,
                               epoch_frames=T * N, max_episode_frames=max_frames, eval_episodes=1,
                               use_cuda_graph=use_graph)
    common = dict(pf=pf, vf=vf, env=env, replay_buffer=buf, collector=col, logger=_Logger(), discount=0.99,
                  num_epochs=10, batch_size=batch_rows * N, gae=True, device=dev, save_dir=None, shuffle=True,
                  tau=0.95, use_cuda_graph=use_graph, plr=3e-4, vlr=3e-4, entropy_coeff=0.01)
    agent = PPO(clip_para=0.1, opt_epochs=2, **common) if kind == "ppo" else A2C(**common)
    return agent, col, buf, env


def _pixel_nets():
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    net = dict(input_shape=(4, 84, 84), hidden_shapes=gold.CNN["hidden"], append_hidden_shapes=[16],
               base_type=networks.CNNBase, activation_func=torch.nn.Tanh)
    return policies.CategoricalDisPolicy(output_shape=6, **net), networks.Net(output_shape=1, **net)


@pytest.mark.parametrize("kind", ["a2c", "ppo"])
def test_fused_epoch_equals_eager_updates_of_a_twin_agent(kind):
    """The fused, graph-captured epoch (old log-probs in memory-bounded chunks, row gather of uint8 frames scaled in the
    graph, per-epoch advantage table read through the device counter, categorical loss kernel) against `update(batch)`
    of a twin agent with the same starting weights, fed the same minibatches in the same np.random order.  The twin
    computes its old log-probs from its target policy and its advantage statistics per minibatch, independently of
    the epoch machinery."""
    import torch
    from torchrl_b200.algo import A2C, PPO
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        N, T, rows = 16, 32, 4
        agent, col, buf, env = _pixel_agent(kind, N=N, T=T, seed=7, max_frames=9, batch_rows=rows, use_graph=True)
        agent.current_epoch = 0
        col.train_one_epoch()
        init = {n: {k: v.detach().clone() for k, v in getattr(agent, n).state_dict().items()} for n in ("pf", "vf")}
        rng = np.random.get_state()
        agent.update_per_epoch()
        assert agent._mb_graph is not None                       # the later minibatches were graph replays
        fused_infos = [dict(i) for i in agent._last_infos]
        # the twin: same weights, eager update(batch) on the minibatches update_per_epoch visited
        pf, vf = _pixel_nets()
        pf.load_state_dict(init["pf"])
        vf.load_state_dict(init["vf"])
        common = dict(pf=pf, vf=vf, env=env, replay_buffer=None, collector=_Col(), logger=_Logger(), discount=0.99,
                      num_epochs=10, batch_size=rows * N, gae=True, device="cuda:0", save_dir=None, shuffle=True,
                      tau=0.95, use_cuda_graph=False, plr=3e-4, vlr=3e-4, entropy_coeff=0.01)
        twin = PPO(clip_para=0.1, opt_epochs=2, **common) if kind == "ppo" else A2C(**common)
        np.random.set_state(rng)
        passes = 2 if kind == "ppo" else 1
        eager_infos = []
        keys = ["obs", "acts", "advs", "estimate_returns", "values"]
        for _ in range(passes):
            order = np.random.permutation(T)
            for u in range(T // rows):
                idx = torch.as_tensor(order[u * rows:(u + 1) * rows], dtype=torch.int64, device="cuda")
                b = {k: v.clone() for k, v in buf.gather_rows(idx, keys).items()}
                b["obs"] = env.to_float(b["obs"].contiguous())
                eager_infos.append(twin.update(b))
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert len(eager_infos) == len(fused_infos) == passes * T // rows
    for u, (m, want) in enumerate(zip(fused_infos, eager_infos)):
        assert set(m) == set(want), (sorted(m), sorted(want))
        for k, v in want.items():
            assert abs(m[k] - v) <= 2e-3 * abs(v) + 2e-4, (u, k, m[k], v)
    if kind == "ppo":
        # the first minibatch of the epoch sees the policy its old log-probs came from
        assert abs(fused_infos[0]["ratio/max"] - 1.0) < 1e-5 and abs(fused_infos[0]["ratio/min"] - 1.0) < 1e-5
        moved = max(max(i["ratio/max"] - 1.0, 1.0 - i["ratio/min"]) for i in fused_infos)
        assert moved > 1e-4                                               # later ones have moved away from it
    for n in ("pf", "vf"):
        mine, ref = getattr(agent, n).state_dict(), getattr(twin, n).state_dict()
        assert max(float((mine[k] - init[n][k]).abs().max()) for k in mine) > 1e-4, "no step was taken"
        for k in ref:
            np.testing.assert_allclose(mine[k].cpu().numpy(), ref[k].cpu().numpy(), atol=2e-4, err_msg=n + "." + k)


def test_pixel_on_policy_collector_rows():
    import torch
    from torchrl_b200.collector.on_policy import PixelVecOnPolicyCollector
    N, T = 16, 24
    agent, col, buf, env = _pixel_agent("ppo", N=N, T=T, max_frames=5)
    assert isinstance(col, PixelVecOnPolicyCollector)
    seeds0 = env.seeds.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    lat0 = env.latent.cpu().numpy()
    col.train_one_epoch()
    assert buf._obs.dtype == torch.uint8 and buf._obs.shape == (T, N, 4, 84, 84)
    assert buf._next_obs.shape == (T, N, 4, 84, 84) and buf._acts.shape == (T, N)
    obs, nxt = buf._obs.cpu().numpy(), buf._next_obs.cpu().numpy()
    acts = buf._acts.cpu().numpy()
    term = buf._terminals.cpu().numpy()[..., 0].astype(bool)
    rew = buf._rewards.cpu().numpy()[..., 0]
    assert acts.min() >= 0 and acts.max() <= 5 and np.all(acts == np.round(acts))
    assert len(np.unique(acts)) > 1
    for t in range(T - 1):
        np.testing.assert_array_equal(nxt[t][:, :3], obs[t][:, 1:])
        cont = ~term[t]
        np.testing.assert_array_equal(obs[t + 1][cont], nxt[t][cont])
    with torch.no_grad():
        v = agent.vf(env.to_float(buf._obs.reshape(T * N, 4, 84, 84).contiguous())).reshape(T, N)
        vn = agent.vf(env.to_float(buf._next_obs.reshape(T * N, 4, 84, 84).contiguous())).reshape(T, N)
    np.testing.assert_allclose(buf._values.cpu().numpy()[..., 0], v.cpu().numpy(), atol=1e-5, rtol=1e-4)
    # replay the recorded actions through the NumPy game: rewards, misses and frames are bit-exact; rows cut by the
    # 5-frame collector timeout store r + discount * V(next_obs)
    lat = {k: lat0[:, i].astype(np.int64) for i, k in enumerate(("bx", "by", "vx", "vy", "px"))}
    episodes = np.zeros(N, dtype=np.int64)
    steps = np.zeros(N, dtype=np.int64)
    cut_rows = 0
    for t in range(T):
        lat, r, miss = oa.step_latent(lat, acts[t].astype(np.int64))
        steps += 1
        np.testing.assert_array_equal(nxt[t][:, 3], oa.render(lat))
        surpass = steps >= 5
        want_r = r.astype(np.float32)
        want_r = np.where(surpass, want_r + np.float32(0.99) * vn[t].cpu().numpy(), want_r)
        np.testing.assert_allclose(rew[t], want_r, atol=1e-5, rtol=1e-5)
        np.testing.assert_array_equal(term[t], miss | surpass)
        cut_rows += int(surpass.sum())
        done = miss | surpass
        if done.any():
            episodes[done] += 1
            fresh = oa.reset_latent(seeds0[done].astype(np.uint64), episodes[done].astype(np.uint64))
            for k in lat:
                lat[k][done] = fresh[k]
            steps[done] = 0
    assert cut_rows > 0


def test_pixel_collector_graph_equals_eager():
    import torch
    runs = []
    for g in (False, True):
        agent, col, buf, env = _pixel_agent("a2c", use_graph=g, seed=4)
        for _ in range(2):
            col.train_one_epoch()
        runs.append({k: getattr(buf, "_" + k).clone() for k in ("obs", "next_obs", "acts", "rewards", "values",
                                                                 "terminals", "time_limits")})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


@pytest.mark.parametrize("kind", ["a2c", "ppo"])
def test_epoch_loop_graph_path_equals_eager_path(kind):
    import torch
    runs = []
    for g in (False, True):
        agent, col, buf, env = _pixel_agent(kind, use_graph=g, seed=2)
        for epoch in range(3):
            agent.current_epoch = epoch
            col.train_one_epoch()
            agent.update_per_epoch()
        runs.append((agent.opt.data.clone(), [dict(i) for i in agent._last_infos]))
        keys = set(agent._last_infos[0])
        assert ("log_std/mean" not in keys) and ("std/mean" not in keys)
        assert all(np.isfinite(v) for i in agent._last_infos for v in i.values())
    (p0, i0), (p1, i1) = runs
    torch.testing.assert_close(p0, p1, rtol=1e-3, atol=2e-5)
    for d0, d1 in zip(i0, i1):
        for k in d0:
            assert abs(d0[k] - d1[k]) <= 2e-3 * max(1.0, abs(d0[k])), (k, d0[k], d1[k])


def test_eval_on_pixel_envs_scales_frames():
    """eval_one_epoch feeds float frames to eval_act: the on-policy categorical collector and the off-policy
    PixelVecCollector (DQN) both evaluate on the uint8 env."""
    from tests.test_atari import _build_pixel
    agent, col, buf, env = _pixel_agent("ppo", N=8)
    out = col.eval_one_epoch()
    assert len(out["eval_rewards"]) == 8 and out["eval_traj_length"] > 0
    agent, col, buf, env = _build_pixel("dqn", N=8)
    out = col.eval_one_epoch()
    assert len(out["eval_rewards"]) == 8 and out["eval_traj_length"] > 0


def test_categorical_ppo_resume_continues_identically(tmp_path):
    import torch
    path = str(tmp_path / "ck.pt")

    def epochs(agent, col, first, n):
        out = []
        for e in range(first, first + n):
            agent.current_epoch = e
            out.append(col.train_one_epoch()["train_epoch_reward"])
            agent.update_per_epoch()
        return out
    agent, col, buf, env = _pixel_agent("ppo", use_graph=False, seed=3)
    epochs(agent, col, 0, 2)
    agent.save_checkpoint(path)
    want_r = epochs(agent, col, 2, 2)
    want = agent.opt.data.clone()
    want_acts = buf._acts.clone()
    agent2, col2, buf2, env2 = _pixel_agent("ppo", use_graph=False, seed=99)
    assert agent2.load_checkpoint(path) == 2
    got_r = epochs(agent2, col2, 2, 2)
    np.testing.assert_allclose(got_r, want_r, rtol=1e-5)
    assert torch.equal(buf2._acts, want_acts)
    torch.testing.assert_close(agent2.opt.data, want, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("script,cfg,key", [("ppo_discrete_atari_vec.py", "ppo_synth_atari.json", "ppo"),
                                            ("a2c_discrete_atari_vec.py", "a2c_synth_atari.json", "a2c")])
def test_reference_discrete_example_runs_unmodified(tmp_path, script, cfg, key):
    from tests.test_reference_examples import REF_EXAMPLES, _run_reference_example
    if not os.path.isdir(REF_EXAMPLES):
        pytest.skip("oracle/_ref not built")

    def patch(c):
        n = 16
        c["replay_buffer"]["size"] = n * 16
        c["collector"].update(epoch_frames=n * 16, max_episode_frames=40)
        c["general_setting"].update(num_epochs=3, batch_size=n * 4, eval_interval=2, save_interval=2)
        if key == "ppo":
            c["ppo"]["opt_epochs"] = 2
    work, header = _run_reference_example(script, cfg, patch, 16, tmp_path)
    files = set(os.listdir(work / "model"))
    for f in ("model_pf_best.pth", "model_vf_0.pth", "model_pf_finish.pth"):
        assert f in files, files
    for k in ("Train_Epoch_Reward", "Training/policy_loss_Mean", "Training/vf_loss_Mean", "eval_traj_length"):
        assert k in header, header
    if key == "ppo":
        assert "ratio/max_Mean" in header and "log_std/mean_Mean" not in header
    else:
        assert "ent_Mean" in header and "std/mean_Mean" not in header
