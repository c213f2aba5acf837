"""Bootstrapped DQN on the device: the masked multi-head loss kernel and the collector's head / action / mask kernel
(csrc/bootstrapped.cu) against fp64 NumPy and torch autograd, the agent against the executed reference
(tests/golden/bootstrapped_dqn_reference.npz), the pixel collector on both ring types, resume and the launcher."""
import csv
import math
import os
import types

import numpy as np
import pytest

from oracle import make_golden_bootstrapped as G
from oracle import ref_bootstrapped as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _loss_inputs(H, B, A, seed, masks="random"):
    """fp32 network outputs, float actions, rewards, a third terminal rows, tied next-state maxima on every other
    sample, and masks: Bernoulli(0.5) (one all-zero and one all-one row), all zero or all one."""
    rs = np.random.RandomState(seed)
    pred = rs.randn(H, B, A).astype(np.float32)
    nxt = rs.randn(H, B, A).astype(np.float32)
    nxt[:, ::2, A - 1] = nxt[:, ::2, 0] = np.abs(nxt[:, ::2]).max(axis=-1) + 0.5
    acts = rs.randint(0, A, B).astype(np.float32)
    rew = rs.randn(B).astype(np.float32)
    term = (rs.rand(B) < 0.33).astype(np.uint8)
    if masks == "zero":
        m = np.zeros((B, H), np.uint8)
    elif masks == "one":
        m = np.ones((B, H), np.uint8)
    else:
        m = (rs.rand(B, H) < 0.5).astype(np.uint8)
        m[0] = 0
        if B > 1:
            m[1] = 1
    return pred, nxt, acts, rew, term, m


def _device_loss(pred, nxt, acts, rew, term, m, gamma=0.99):
    import torch
    from torchrl_b200 import ops
    B = rew.size
    grad = torch.full(pred.shape, float("nan"), dtype=torch.float32, device=DEV)     # every element must be written
    info = torch.full((3,), float("nan"), dtype=torch.float32, device=DEV)
    ops.bootstrapped_dqn_loss(_t(pred), _t(nxt), _t(acts), _t(rew), _t(term), _t(m), gamma,
                              ops.OffPolicyScratch(B, DEV), info=info, grad=grad)
    return grad.cpu().numpy(), info.cpu().numpy()


def _autograd_loss(pred, nxt, acts, rew, term, m, gamma=0.99):
    """The reference's expression (bootstrapped_dqn.py:89-105) in fp64 torch on the CPU."""
    import torch
    H = pred.shape[0]
    p = torch.tensor(pred, dtype=torch.float64, requires_grad=True)
    q_next = torch.tensor(nxt, dtype=torch.float64)
    a = torch.tensor(acts).long().unsqueeze(1)
    r = torch.tensor(rew, dtype=torch.float64).unsqueeze(1)
    d = torch.tensor(term, dtype=torch.float64).unsqueeze(1)
    losses = []
    for h in range(H):
        q_s_a = p[h].gather(1, a)
        target = r + gamma * (1 - d) * q_next[h].max(1, keepdim=True)[0]
        losses.append((q_s_a - target) ** 2)
    loss = (torch.cat(losses, dim=1) * torch.tensor(m, dtype=torch.float64) / H).sum(1).mean()
    loss.backward()
    return float(loss.detach()), p.grad.numpy()


@pytest.mark.parametrize("A", [2, 6, 18])
@pytest.mark.parametrize("H", [1, 10])
@pytest.mark.parametrize("B", [1, 7, 4096, 65537])
def test_loss_kernel_against_fp64(B, H, A):
    args = _loss_inputs(H, B, A, seed=B + 7 * H + A)
    g, info = _device_loss(*args)
    loss64, g64, info64 = R.bootstrapped_dqn_loss(*args, 0.99)
    loss_t, g_t = _autograd_loss(*args)
    np.testing.assert_allclose(loss64, loss_t, rtol=1e-12)
    np.testing.assert_allclose(g64, g_t, rtol=1e-12, atol=1e-18)
    # fp32 per element: |Q - y| carries a few ulp of |y| ~ 5; the sums are fp64
    np.testing.assert_allclose(info[0], loss64, rtol=1e-5)
    np.testing.assert_allclose(info[1:], info64[1:], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(g, g64, rtol=1e-5, atol=1e-5 * 2.0 / (H * B))
    pred, _, acts, _, _, m = args
    taken = np.zeros(pred.shape, bool)
    taken[:, np.arange(B), acts.astype(np.int64)] = True
    assert np.all(g[~taken] == 0)                                     # zero off the taken action
    assert np.all(g[m.T == 0] == 0)                                   # masked-out heads get no gradient
    assert np.all(g[:, 0, :] == 0)                                    # sample 0 has an all-zero mask row


@pytest.mark.parametrize("B,H,A", [(1, 1, 2), (7, 10, 6), (4096, 10, 18)])
def test_loss_kernel_all_zero_and_all_one_masks(B, H, A):
    args = _loss_inputs(H, B, A, seed=3, masks="zero")
    g, info = _device_loss(*args)
    assert info[0] == 0.0 and np.all(g == 0.0)
    _, _, info64 = R.bootstrapped_dqn_loss(*args, 0.99)
    np.testing.assert_allclose(info[1:], info64[1:], rtol=1e-5, atol=1e-6)
    args = _loss_inputs(H, B, A, seed=4, masks="one")
    g, info = _device_loss(*args)
    loss64, g64, _ = R.bootstrapped_dqn_loss(*args, 0.99)
    np.testing.assert_allclose(info[0], loss64, rtol=1e-5)
    np.testing.assert_allclose(g, g64, rtol=1e-5, atol=1e-5 * 2.0 / (H * B))
    # all terminal: the targets are the rewards alone
    pred, nxt, acts, rew, term, m = args
    _, info_t = _device_loss(pred, nxt, acts, rew, np.ones_like(term), m)
    q = pred[:, np.arange(B), acts.astype(np.int64)].astype(np.float64)
    np.testing.assert_allclose(info_t[0], ((q - rew.astype(np.float64)) ** 2).mean(), rtol=1e-5)


@pytest.mark.parametrize("B,H,A", [(7, 1, 2), (4096, 10, 6)])
def test_loss_kernel_equals_the_sum_of_weighted_dqn_losses(B, H, A):
    """Sum over heads of the existing DQN-form kernel with importance weights m_h / H."""
    import torch
    from torchrl_b200 import ops
    pred, nxt, acts, rew, term, m = _loss_inputs(H, B, A, seed=11)
    g, info = _device_loss(pred, nxt, acts, rew, term, m)
    scratch = ops.OffPolicyScratch(B, DEV)
    total = 0.0
    for h in range(H):
        w = _t((m[:, h] / np.float32(H)).astype(np.float32))
        gh, ih = ops.qr_dqn_loss(_t(pred[h]), _t(nxt[h]), _t(acts), _t(rew), _t(term), 0.99, scratch, A, 1, mse=True,
                                 weights=w)
        total += float(ih[0])
        np.testing.assert_allclose(g[h], gh.cpu().numpy(), rtol=1e-5, atol=1e-6 / B)
        torch.cuda.synchronize()
    np.testing.assert_allclose(info[0], total, rtol=1e-5)


def _act_inputs(N, H, A, seed):
    rs = np.random.RandomState(seed)
    q = rs.randn(H, N, A).astype(np.float32)
    q[:, ::5, :] = 0.25                                               # all tied: action 0
    q[:, 1::5, 2 % A] = q[:, 1::5, A - 1] = 9.0                       # two tied maxima
    step = np.where(rs.rand(N) < 0.4, 0, rs.randint(1, 50, N)).astype(np.int32)
    step[:2] = 0
    head = rs.randint(0, H, N).astype(np.int32)
    u = rs.rand(N).astype(np.float32)
    u[0] = 0.0
    u[1:2] = np.float32(1 - 2 ** -24)                                 # floor(u * H) reaches H: clamped to H - 1
    um = rs.rand(N, H).astype(np.float32)
    return q, step, head, u, um


@pytest.mark.parametrize("N,H,A", [(37, 10, 6), (1000, 3, 18), (1, 1, 2)])
def test_act_kernel_with_supplied_uniforms(N, H, A):
    import torch
    from torchrl_b200 import ops
    q, step, head, u, um = _act_inputs(N, H, A, seed=N)
    T, top = 5, 3
    ring = torch.full((T, N, H), 0xA5, dtype=torch.uint8, device=DEV)
    d_head, act = _t(head), torch.full((N,), float("nan"), device=DEV)
    ops.bootstrapped_act(_t(q), _t(step), d_head, act, ring, torch.tensor([top], dtype=torch.int32, device=DEV), 0.3,
                         u_head=_t(u), u_mask=_t(um))
    want_head, want_act, want_mask = R.bootstrapped_act(q, step, head, u, um, 0.3)
    np.testing.assert_array_equal(d_head.cpu().numpy(), want_head)
    np.testing.assert_array_equal(act.cpu().numpy(), want_act.astype(np.float32))
    r = ring.cpu().numpy()
    np.testing.assert_array_equal(r[top], want_mask)
    assert np.all(np.delete(r, top, axis=0) == 0xA5)                 # no other ring row touched
    if N > 1:
        assert want_head[1] == H - 1 and want_act[0] == 0 and want_act[1] == 2 % A


def test_act_kernel_with_philox():
    import torch
    from torchrl_b200 import ops
    N, H, A, p = 4096, 10, 6, 0.3
    q, _, head, _, _ = _act_inputs(N, H, A, seed=5)
    zero = torch.zeros(N, dtype=torch.int32, device=DEV)              # every env starts an episode
    top = torch.zeros(1, dtype=torch.int32, device=DEV)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    rng = types.SimpleNamespace(seed=12345, counter=torch.tensor([7], dtype=torch.int64, device=DEV))

    def draw():
        ring = torch.zeros(1, N, H, dtype=torch.uint8, device=DEV)
        hd, act = _t(head), torch.empty(N, device=DEV)
        ops.bootstrapped_act(_t(q), zero, hd, act, ring, top, p, rng=rng, ticket=ticket)
        return hd.cpu().numpy(), act.cpu().numpy(), ring[0].cpu().numpy()

    h1, a1, m1 = draw()
    assert int(rng.counter) == 8 and int(ticket) == 0                 # the launch advanced its counter
    h2, _, m2 = draw()
    assert int(rng.counter) == 9
    rng.counter.fill_(7)
    h3, a3, m3 = draw()
    assert np.array_equal(h1, h3) and np.array_equal(m1, m3) and np.array_equal(a1, a3)
    assert not np.array_equal(m1, m2) and not np.array_equal(h1, h2)
    np.testing.assert_array_equal(a1, q[h1.astype(np.int64), np.arange(N)].argmax(-1))
    for m in (m1, m2):                                                # Bernoulli(p): 5 standard deviations
        assert abs(m.mean() - p) < 5 * math.sqrt(p * (1 - p) / m.size)
    for h in (h1, h2):                                                # uniform heads: 5 standard deviations per bin
        counts = np.bincount(h, minlength=H)
        assert counts.size == H and np.all(np.abs(counts - N / H) < 5 * math.sqrt(N / H * (1 - 1 / H)))
    # captured once, replayed: each replay reads and advances the counter
    ring = torch.zeros(1, N, H, dtype=torch.uint8, device=DEV)
    hd, act = _t(head), torch.empty(N, device=DEV)
    rng.counter.fill_(7)
    qd = _t(q)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.bootstrapped_act(qd, zero, hd, act, ring, top, p, rng=rng, ticket=ticket)
    g.replay()
    assert np.array_equal(ring[0].cpu().numpy(), m1) and int(rng.counter) == 8
    g.replay()
    assert np.array_equal(ring[0].cpu().numpy(), m2) and int(rng.counter) == 9


# ------------------------------------------------------------------------------------------------ agent
def _build(N=37, rows=40, dedup=False, graph_col=False, graph_agent=False, H=4, seed=0, max_frames=13, batch_rows=2,
           opt_times=3, p=0.5, frame=None, head_hidden=64, agent_kw=None):
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import BootstrappedDQN
    from torchrl_b200.collector import PixelVecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer, MemoryEfficientReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device(DEV)
    env = get_vec_env("SynthAtari-v0", {}, N)
    eval_env = get_vec_env("SynthAtari-v0", {}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    buf = (MemoryEfficientReplayBuffer if dedup else BaseReplayBuffer)(env_nums=N, max_replay_buffer_size=rows * N)
    if frame is None:
        net = dict(input_shape=(4, 84, 84), hidden_shapes=[[16, [8, 8], [4, 4], [0, 0]], [32, [4, 4], [2, 2], [0, 0]]],
                   append_hidden_shapes=[head_hidden])
    else:
        net = frame
    qf = networks.BootstrappedNet(output_shape=6, base_type=networks.CNNBase, head_num=H, activation_func=nn.ReLU,
                                  **net)
    pf = policies.BootstrappedDQNDiscretePolicy(qf=qf, head_num=H, action_shape=6)
    col = PixelVecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=8 * N,
                            max_episode_frames=max_frames, use_cuda_graph=graph_col)
    kw = dict(use_soft_update=False, target_hard_update_period=3)
    kw.update(agent_kw or {})
    agent = BootstrappedDQN(head_num=H, bernoulli_p=p, qf=qf, pf=pf, qlr=1e-3, optimizer_info={"eps": 1e-4}, env=env,
                            replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99,
                            batch_size=batch_rows * N, device=dev, save_dir=None, opt_times=opt_times,
                            pretrain_epochs=1, num_epochs=2, use_cuda_graph=graph_agent, **kw)
    return agent, col, buf, env


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "bootstrapped_dqn_reference.npz")))


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_agent_matches_the_executed_reference(golden, case):
    """Eager `update(batch)` on the recorded batches from the recorded initial weights: every update's logged loss and
    mean reward, and the parameters after the last update (hard target copies and Polyak averaging included)."""
    import torch
    H, n, kw, _ = G.CASES[case]
    frame = dict(input_shape=G.OBS, hidden_shapes=G.HIDDEN, append_hidden_shapes=G.APPEND)
    agent, col, buf, env = _build(N=G.B, rows=2, H=H, batch_rows=1, frame=frame, agent_kw=kw)
    init = {k.split("|", 2)[2]: torch.from_numpy(v) for k, v in golden.items() if k.startswith(case + "|init|")}
    with torch.no_grad():
        agent.qf.load_state_dict(init)                               # in place: the flat-buffer views stay intact
        agent.target_qf.load_state_dict(init)
    for f in (agent.opt, agent._target_flat):
        if hasattr(f, "refresh_split"):
            f.refresh_split()
    for u, b in enumerate(G.batches(H, n, G.CASES[case][3])):
        feed = dict(b, obs=G.frames_to_float(b["obs"]), next_obs=G.frames_to_float(b["next_obs"]))
        info = agent.update(feed)
        want = golden["%s|update%d|info" % (case, u)]
        np.testing.assert_allclose(info["Training/qf_loss"], want[0], rtol=2e-3, atol=2e-4)
        np.testing.assert_allclose(info["Reward_Mean"], want[1], rtol=2e-3, atol=2e-4)
        assert np.isfinite(info["q_s_a"])
    final = agent.qf.state_dict()
    for k, v in golden.items():
        if k.startswith(case + "|final|"):
            name = k.split("|", 2)[2]
            np.testing.assert_allclose(final[name].cpu().numpy(), v, rtol=0, atol=2e-4, err_msg=name)


def test_captured_update_equals_eager_over_one_epoch():
    import torch
    runs = []
    for graph in (False, True):
        agent, col, buf, env = _build(N=16, rows=24, graph_agent=graph, seed=5, opt_times=6)
        agent.pretrain()
        agent.current_epoch = 0
        col.train_one_epoch()
        agent.update_per_epoch()
        runs.append((agent.opt.data.clone(), agent._last_infos, buf._masks.clone()))
    (p0, i0, m0), (p1, i1, m1) = runs
    assert torch.equal(m0, m1) and len(i0) == len(i1) == 6
    torch.testing.assert_close(p0, p1, rtol=1e-5, atol=1e-6)
    for d0, d1 in zip(i0, i1):
        for k in d0:
            assert abs(d0[k] - d1[k]) <= 1e-5 * max(1.0, abs(d0[k])), (k, d0[k], d1[k])


@pytest.mark.parametrize("dedup", [False, True])
def test_collector_heads_actions_and_masks(dedup):
    """300 eager steps of 37 envs with 13-frame episodes: each step's heads and mask row are exactly the kernel's
    draw for the step's Philox counter, heads change only where an episode starts, each action is the greedy action
    of the env's head, and the masks are Bernoulli(p)."""
    import torch
    from torchrl_b200 import ops
    N, H, p = 37, 4, 0.3
    agent, col, buf, env = _build(N=N, rows=400, dedup=dedup, H=H, p=p)
    pf, qf = col.pf, col.pf.qf
    assert buf._masks.dtype == torch.uint8 and buf._masks.shape == (400, N, H)
    changes = starts = ones = 0
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    row0 = torch.zeros(1, dtype=torch.int32, device=DEV)
    for t in range(300):
        top = buf._top
        cs, head0 = col.current_step.clone(), pf.head.clone()
        ctr = 0 if pf._rng.counter is None else int(pf._rng.counter)
        with torch.no_grad():
            q = qf.all_heads(env.to_float(env.obs)).contiguous()
        col._step()
        head1 = pf.head.clone()
        assert int(pf._rng.counter) == ctr + 1
        rng = types.SimpleNamespace(seed=pf._rng.seed, counter=torch.tensor([ctr], dtype=torch.int64, device=DEV))
        ring = torch.zeros(1, N, H, dtype=torch.uint8, device=DEV)
        hd, act = head0.clone(), torch.empty(N, device=DEV)
        ops.bootstrapped_act(q, cs, hd, act, ring, row0, p, rng=rng, ticket=ticket)
        assert torch.equal(hd, head1), t
        assert torch.equal(ring[0], buf._masks[top]), t
        a = buf._acts[top].long()
        qh = q[head1.long(), torch.arange(N, device=DEV)]
        best = qh.max(1)[0]
        assert torch.all(qh.gather(1, a[:, None])[:, 0] >= best - 1e-5 * (1 + best.abs())), t
        changed = head1 != head0
        assert not bool((changed & (cs != 0)).any()), t
        changes += int(changed.sum())
        starts += int((cs == 0).sum())
        ones += int(buf._masks[top].sum())
    assert starts > 300 * N / 13 * 0.5 and changes > starts * 0.5   # a new head is drawn at every episode start
    assert abs(ones / (300 * N * H) - p) < 5 * math.sqrt(p * (1 - p) / (300 * N * H))


def test_captured_collector_step_writes_the_same_masks_as_eager():
    import torch
    masks, acts = [], []
    for graph in (False, True):
        agent, col, buf, env = _build(N=37, rows=40, graph_col=graph, seed=2)
        for _ in range(30):
            col._step()
        masks.append(buf._masks.clone())
        acts.append(buf._acts.clone())
    assert torch.equal(masks[0], masks[1])
    assert float((acts[0] == acts[1]).float().mean()) > 0.99


def test_prioritised_replay_is_refused():
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import BootstrappedDQN
    from torchrl_b200.collector import PixelVecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import PrioritizedReplayBuffer
    from torchrl_b200.utils import NullLogger
    env, eval_env = get_vec_env("SynthAtari-v0", {}, 8), get_vec_env("SynthAtari-v0", {}, 8)
    buf = PrioritizedReplayBuffer(env_nums=8, max_replay_buffer_size=8 * 4)
    qf = networks.BootstrappedNet(output_shape=6, base_type=networks.CNNBase, head_num=2, activation_func=nn.ReLU,
                                  input_shape=(4, 84, 84), hidden_shapes=[[8, [8, 8], [4, 4], [0, 0]]],
                                  append_hidden_shapes=[])
    pf = policies.BootstrappedDQNDiscretePolicy(qf=qf, head_num=2, action_shape=6)
    col = PixelVecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=DEV, epoch_frames=8)
    with pytest.raises(NotImplementedError, match="prioritised"):
        BootstrappedDQN(head_num=2, qf=qf, pf=pf, qlr=1e-3, env=env, replay_buffer=buf, collector=col,
                        logger=NullLogger(), batch_size=8, device=DEV, save_dir=None)


def test_resume_continues_identically(tmp_path):
    import torch
    path = str(tmp_path / "ck.pt")

    def epochs(agent, col, first, n):
        for e in range(first, first + n):
            agent.current_epoch = e
            col.train_one_epoch()
            agent.update_per_epoch()

    agent, col, buf, env = _build(N=16, rows=30, H=3, seed=3)
    agent.pretrain()
    epochs(agent, col, 0, 2)
    agent.save_checkpoint(path)
    epochs(agent, col, 2, 1)
    want = (agent.opt.data.clone(), agent._target_flat.data.clone(), buf._masks.clone(), buf._acts.clone(),
            col.pf.head.clone(), int(col.pf._rng.counter), buf._top)
    agent2, col2, buf2, env2 = _build(N=16, rows=30, H=3, seed=77)
    agent2.load_checkpoint(path)
    epochs(agent2, col2, 2, 1)
    got = (agent2.opt.data, agent2._target_flat.data, buf2._masks, buf2._acts, col2.pf.head,
           int(col2.pf._rng.counter), buf2._top)
    assert torch.equal(got[2], want[2]) and torch.equal(got[3], want[3]) and torch.equal(got[4], want[4])
    assert got[5] == want[5] and got[6] == want[6]
    torch.testing.assert_close(got[0], want[0], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(got[1], want[1], rtol=1e-5, atol=1e-7)


def test_launcher_trains_on_a_shrunken_config(tmp_path):
    from tests.test_examples import _run

    def patch(c):
        c["replay_buffer"]["size"] = 32 * 40
        c["collector"].update(epoch_frames=32 * 8, max_episode_frames=30)
        c["general_setting"].update(pretrain_epochs=1, num_epochs=3, batch_size=64, opt_times=4, min_pool=0,
                                    target_hard_update_period=5, eval_interval=1, save_interval=1)
        c["net"].update(hidden_shapes=[[8, [8, 8], [4, 4], [0, 0]], [8, [4, 4], [2, 2], [0, 0]]],
                        append_hidden_shapes=[32])
        c["bootstrapped_dqn"]["head_num"] = 3
    work = _run("bootstrapped_dqn_atari_vec.py", "bootstrapped_dqn_synth_atari.json", patch, 32, tmp_path)
    assert "model_pf_finish.pth" in set(os.listdir(work / "model"))
    rows = list(csv.DictReader(open(work / "log.csv")))
    assert len(rows) == 3
    for key in ("Training/qf_loss", "Reward_Mean"):
        cols = [c for c in rows[0] if c.startswith(key)]
        assert cols, (key, list(rows[0]))
        assert all(math.isfinite(float(r[c])) for r in rows for c in cols), key
