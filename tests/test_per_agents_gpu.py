"""Prioritised replay in the continuous-control agents and in the captured prioritised epoch: importance-weighted critic
losses (weights of 1 reproduce the uniform update bit for bit), the priorities the update writes, eager and captured
epochs that agree bit for bit, rings past 4096 rows, resume, and TD3 learning Pendulum-v1 with prioritised replay."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import ref_numpy as rn
from tests.test_layer_kernels import U, same_bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["ddpg", "td3", "twin_sac_q", "sac", "twin_sac"]


def _agent(kind, per=True, N=16, ring_rows=160, seed=0, use_graph=True, opt_times=8, hidden=64, cfg=None):
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import DDPG, SAC, TD3, TwinSAC, TwinSACQ
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer, PrioritizedReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device("cuda:0")
    env = get_vec_env("Pendulum-v1", {"reward_scale": 1, "obs_norm": False}, N)
    eval_env = get_vec_env("Pendulum-v1", {"reward_scale": 1, "obs_norm": False}, N)
    env.seed(seed); eval_env.seed(seed + 1000); torch.manual_seed(seed); np.random.seed(seed)
    o, a = 3, 1
    net = dict(hidden_shapes=[hidden, hidden], append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=nn.ReLU)
    if per:
        buf = PrioritizedReplayBuffer(env_nums=N, max_replay_buffer_size=ring_rows * N, alpha=0.6, beta=0.4)
    else:
        buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=ring_rows * N)
    if kind in ("sac", "twin_sac", "twin_sac_q"):
        pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, tanh_action=True, **net)
    elif kind == "ddpg":
        pf = policies.DetContPolicy(input_shape=o, output_shape=a, tanh_action=True, **net)
    else:
        pf = policies.FixGuassianContPolicy(input_shape=o, output_shape=a, tanh_action=True, norm_std_explore=0.1,
                                            **net)
    qf1 = networks.QNet(input_shape=o + a, output_shape=1, **net)
    qf2 = networks.QNet(input_shape=o + a, output_shape=1, **net)
    vf = networks.Net(input_shape=o, output_shape=1, **net)
    col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=40 * N,
                       max_episode_frames=200, use_cuda_graph=use_graph)
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99, batch_size=8 * N,
                  device=dev, save_dir=None, tau=0.005, use_soft_update=True, opt_times=opt_times, pretrain_epochs=1,
                  num_epochs=3, use_cuda_graph=use_graph)
    if kind == "td3":
        agent = TD3(pf=pf, qf1=qf1, qf2=qf2, plr=1e-3, qlr=1e-3, **common)
    elif kind == "ddpg":
        agent = DDPG(pf=pf, qf=qf1, plr=1e-3, qlr=1e-3, **common)
    elif kind == "twin_sac_q":
        agent = TwinSACQ(pf=pf, qf1=qf1, qf2=qf2, plr=3e-4, qlr=3e-4, policy_std_reg_weight=0,
                         policy_mean_reg_weight=0, **common)
    elif kind == "sac":
        agent = SAC(pf=pf, vf=vf, qf=qf1, plr=3e-4, vlr=3e-4, qlr=3e-4, **common)
    else:
        agent = TwinSAC(pf=pf, vf=vf, qf1=qf1, qf2=qf2, plr=3e-4, vlr=3e-4, qlr=3e-4, **common)
    return agent, col, buf, env


def _batch(seed, B, o=3, a=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"obs": torch.randn(B, o, device="cuda", generator=g),
            "next_obs": torch.randn(B, o, device="cuda", generator=g),
            "acts": torch.rand(B, a, device="cuda", generator=g) * 2 - 1,
            "rewards": torch.randn(B, 1, device="cuda", generator=g),
            "terminals": (torch.rand(B, 1, device="cuda", generator=g) < 0.1).to(torch.uint8)}


@pytest.mark.parametrize("kind", KINDS)
def test_unit_weights_reproduce_the_uniform_update(kind):
    """two identical agents update on the same rows, one with weights of 1: the same parameters and targets, bit for
    bit, over three updates (TD3: both graph variants)"""
    a1 = _agent(kind, per=False)[0]
    a2 = _agent(kind, per=True)[0]
    assert same_bits(a1.opt.data, a2.opt.data)
    for k in range(3):
        batch = _batch(k, a1.batch_size)
        a1.update(batch)
        a2.update(dict(batch, weights=torch.ones(a1.batch_size, 1, device="cuda")))
        assert same_bits(a1.opt.data, a2.opt.data), "parameters differ after update %d" % k
        assert same_bits(a1._target_flat.data, a2._target_flat.data)


@pytest.mark.parametrize("kind", KINDS)
def test_critic_loss_is_importance_weighted(kind):
    """the agent's critic loss with non-unit weights: the gradient of mean(w (q - y)^2) against fp64 and the
    unweighted |q - y| in its TD buffer, one column per critic"""
    agent = _agent(kind, per=True)[0]
    agent._ub_setup()
    B = agent.batch_size
    torch.manual_seed(5)
    q1, q2, y = (torch.randn(B, device="cuda") for _ in range(3))
    w = torch.rand(B, 1, device="cuda") + 0.1
    twin = agent.TD_COLUMNS == 2
    info = torch.zeros(2, device="cuda")
    g1, g2, _ = agent._critic_loss({"weights": w}, q1, q2 if twin else None, y, info)
    td = agent._td.reshape(B, -1)
    assert td.shape[1] == agent.TD_COLUMNS
    for k, (q, g) in enumerate(zip((q1, q2), (g1, g2))):
        if k == 1 and not twin:
            break
        d = (q - y).double()
        want = 2 * d * w.reshape(-1).double() / B
        assert torch.all((g.double() - want).abs() <= 4 * U * want.abs())
        assert same_bits(td[:, k], (q - y).abs())
        loss = (w.reshape(-1).double() * d * d).mean().item()
        assert abs(info[k].item() - loss) <= 8 * U * loss


@pytest.mark.parametrize("kind", KINDS)
def test_prioritised_update_writes_the_oracle_priorities(kind):
    """one captured prioritised update per epoch: the drawn rows' new priorities are per_update of the update's |TD|
    (mean over the row's N transitions and the critics), and the running max follows"""
    agent, col, buf, env = _agent(kind, per=True, opt_times=1)
    agent.pretrain()
    col.train_one_epoch()
    for _ in range(2):
        before = buf._priorities.clone()
        mx0 = float(buf._max_prio.item())
        agent.update_per_epoch()
        ub = agent._ub
        rows = ub["rows"].cpu().numpy()
        td = agent._td.reshape(ub["b"], -1).cpu().numpy()
        ref = before.cpu().numpy()
        rmax = rn.per_update(ref, rows, td, buf.alpha, buf.eps, mx0)
        got = buf._priorities.cpu().numpy()
        assert np.all(np.abs(got.astype(np.float64) - ref) <= (14 * 2.0 ** -53 + 12 * U) * ref)
        assert abs(float(buf._max_prio.item()) - rmax) <= 12 * U * rmax
        w = ub["w_samples"].reshape(ub["b"], -1)
        assert torch.all(w == w[:, :1]) and torch.all(w > 0) and torch.all(w <= 1)


def _qr_agent(use_graph, opt_times, N=32, seed=0):
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import QRDQN
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import PrioritizedReplayBuffer
    from torchrl_b200.utils import NullLogger
    env = get_vec_env("CartPole-v1", {}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    Q = 8
    buf = PrioritizedReplayBuffer(env_nums=N, max_replay_buffer_size=200 * N)
    qf = networks.Net(input_shape=(4,), output_shape=2 * Q, hidden_shapes=[64, 64], append_hidden_shapes=[],
                      base_type=networks.MLPBase, activation_func=nn.ReLU)
    pf = policies.EpsilonGreedyQRDQNDiscretePolicy(quantile_num=Q, qf=qf, start_epsilon=1.0, end_epsilon=0.1,
                                                   decay_frames=40, action_shape=2)
    col = VecCollector(env=env, pf=pf, replay_buffer=buf, device="cuda", epoch_frames=40 * N, max_episode_frames=1000,
                       use_cuda_graph=use_graph)
    agent = QRDQN(quantile_num=Q, qf=qf, pf=pf, qlr=1e-3, env=env, replay_buffer=buf, collector=col,
                  logger=NullLogger(), discount=0.99, batch_size=4 * N, device="cuda", save_dir=None,
                  opt_times=opt_times, use_soft_update=True, tau=0.005, pretrain_epochs=1, num_epochs=3,
                  use_cuda_graph=use_graph)
    return agent, col, buf


def _collected(kind, opt_times):
    if kind == "qr_dqn":
        agent, col, buf = _qr_agent(True, opt_times)
    else:
        agent, col, buf, _ = _agent(kind, per=True, use_graph=True, opt_times=opt_times)
    agent.pretrain()
    col.train_one_epoch()
    return agent, buf


def _epochs(agent, buf, epochs):
    """`epochs` prioritised epochs; after each: the last update's drawn rows, the priorities, the parameters and the
    epoch's log rows"""
    out = []
    for _ in range(epochs):
        agent.update_per_epoch(flush_infos=False)
        ub = agent._ub
        out.append([ub["rows"].clone(), buf._priorities.clone(), agent.opt.data.clone(), ub["log32"].clone()])
    return out


@pytest.mark.parametrize("opt_times,epochs", [(1, 12), (8, 2)])
@pytest.mark.parametrize("kind", ["td3", "qr_dqn"])
def test_eager_and_captured_prioritised_epochs_agree(kind, opt_times, epochs):
    """from identical state (the second agent's ring is overwritten with the first's: the epsilon-greedy CartPole
    collector does not repeat its rows from run to run), eager and captured updates: with one update per epoch the
    rows of every update, with 8 the whole epoch (the first epoch runs each variant eagerly three times, then captures
    it; the second only replays)"""
    eager, eb = _collected(kind, opt_times)
    graph, gb = _collected(kind, opt_times)
    assert same_bits(eager.opt.data, graph.opt.data)
    for k in list(eb._keys) + ["priorities", "max_prio", "top_dev", "size_dev"]:
        getattr(gb, "_" + k).copy_(getattr(eb, "_" + k))
    np.random.seed(123)
    torch.manual_seed(123)
    eager.use_cuda_graph = False
    want = _epochs(eager, eb, epochs)
    np.random.seed(123)
    torch.manual_seed(123)
    got = _epochs(graph, gb, epochs)
    assert graph._graphs and not eager._graphs
    names = ("drawn rows", "priorities", "parameters", "log rows")
    for k, (e_all, g_all) in enumerate(zip(want, got)):
        for name, e, g in zip(names, e_all, g_all):
            same = torch.equal(e, g) if e.dtype == torch.int64 else same_bits(e, g)
            assert same, "%s differ between the eager and the captured run after epoch %d" % (name, k)


def test_td3_on_a_ring_past_4096_rows_moves_its_priorities():
    """config/td3_pendulum.json's 100,000-transition ring at 16 envs: 6,250 rows"""
    agent, col, buf, _ = _agent("td3", per=True, ring_rows=100000 // 16, opt_times=50)
    assert buf._max_replay_buffer_size == 6250
    agent.pretrain()
    for _ in range(2):
        col.train_one_epoch()
        p0 = buf._priorities.clone()
        agent.update_per_epoch()
        assert not torch.equal(p0, buf._priorities)
        assert all(np.isfinite(v) for info in agent._last_infos for v in info.values())
    assert len(agent._graphs) == 2, "TD3's two variants replay captured graphs"
    live = buf._priorities[:buf.num_steps_can_sample()]
    assert torch.all(live > 0) and torch.all(buf._priorities[buf.num_steps_can_sample():] == 0)


def test_td3_resume_under_prioritised_replay(tmp_path):
    path = str(tmp_path / "ck.pt")

    def epochs(agent, col, first, n):
        for e in range(first, first + n):
            agent.current_epoch = e
            col.train_one_epoch()
            agent.update_per_epoch()

    agent, col, buf, env = _agent("td3", per=True, seed=1)
    agent.pretrain()
    epochs(agent, col, 0, 2)
    agent.save_checkpoint(path)
    state = torch.load(path, map_location="cpu", weights_only=False)
    assert not any(k.startswith("_sampler") for k in state["buffer_tensors"]), "sampler scratch is not state"
    epochs(agent, col, 2, 2)
    want = (agent.opt.data.clone(), agent._target_flat.data.clone(), buf._priorities.clone())
    agent2, col2, buf2, env2 = _agent("td3", per=True, seed=77)
    assert agent2.load_checkpoint(path) == 2
    epochs(agent2, col2, 2, 2)
    got = (agent2.opt.data, agent2._target_flat.data, buf2._priorities)
    for w, g in zip(want, got):
        assert same_bits(w, g)


def test_td3_learns_pendulum_with_prioritised_replay():
    """TD3 with config/td3_pendulum.json and a PrioritizedReplayBuffer (alpha 0.6, beta 0.4) on the config's ring at
    16 envs (6,250 rows), seed 0, reaches the uniform test's -500 within its 25-epoch budget
    (tests/test_pendulum_learning_gpu.py), evaluating greedily every 5 epochs on 16 envs.
    Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), `python -m tests.test_per_agents_gpu`:
        epochs 5-25: -1144, -850, -445, -398, -491 (the uniform run: -793, -500, -148, -241, -157)"""
    returns = train_per(25)
    assert max(returns) >= -500.0, returns


def train_per(epochs, seed=0, report=None):
    """Train TD3 with prioritised replay on Pendulum-v1; the mean greedy returns after every 5 epochs."""
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import TD3
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import PrioritizedReplayBuffer
    from torchrl_b200.utils import NullLogger
    N = 16
    cfg = json.load(open(os.path.join(ROOT, "config", "td3_pendulum.json")))
    g = cfg["general_setting"]
    dev = torch.device("cuda:0")
    env, eval_env = get_vec_env("Pendulum-v1", cfg["env"], N), get_vec_env("Pendulum-v1", cfg["env"], N)
    env.seed(seed); eval_env.seed(seed + 1000); torch.manual_seed(seed); np.random.seed(seed)
    buf = PrioritizedReplayBuffer(env_nums=N, max_replay_buffer_size=int(cfg["replay_buffer"]["size"]),
                                  time_limit_filter=cfg["replay_buffer"]["time_limit_filter"], alpha=0.6, beta=0.4)
    net = dict(cfg["net"], base_type=networks.MLPBase, activation_func=torch.nn.ReLU)
    pf = policies.FixGuassianContPolicy(input_shape=3, output_shape=1, **net, **cfg["policy"])
    qf1 = networks.QNet(input_shape=4, output_shape=1, **net)
    qf2 = networks.QNet(input_shape=4, output_shape=1, **net)
    col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, **cfg["collector"])
    common = dict(g, num_epochs=epochs, env=env, replay_buffer=buf, collector=col, logger=NullLogger(), device=dev,
                  save_dir=None)
    for k in ("eval_interval", "save_interval"):
        common.pop(k)
    agent = TD3(pf=pf, qf1=qf1, qf2=qf2, **cfg["td3"], **common)
    agent.pretrain()
    returns = []
    for epoch in range(epochs):
        agent.current_epoch = epoch
        col.train_one_epoch()
        agent.update_per_epoch()
        if (epoch + 1) % 5 == 0:
            returns.append(float(np.mean(col.eval_one_epoch()["eval_rewards"])))
            if report is not None:
                report(epoch + 1, returns[-1])
    return returns


if __name__ == "__main__":
    train_per(25, report=lambda e, r: print("epoch %d return %.1f" % (e, r), flush=True))
