"""SAC and TwinSAC with a state-value network (algo/off_policy/sac.py, twin_sac.py) and their value/policy loss
kernel trl_sac_v_loss.

CPU (reference present): `SACVPort` below -- a restatement of the reference's SAC.update (sac.py:74-208) and
TwinSAC.update (twin_sac.py:82-229) without the `assert v_target == v_pred` that raises for every batch of more than
one row -- reproduces, bit for bit, the unmodified reference run under `python -O` (which strips that assert).
GPU: the kernel against an fp64 NumPy restatement at the edges of its ABI; agent.update against SACVPort on
the same batches, weights and CPU noise (tolerances of test_offpolicy.py: logged scalars rtol 2e-3 + atol 2e-4,
parameters after 4 updates atol 2e-4); CUDA graph vs eager; checkpoint resume; one update at the benchmark's
sizes (logged scalars rtol 5e-3 + atol 5e-4, parameters 99.9 % within atol 5e-4 and all within 2*lr + 5e-4); both
configs end to end through compat/.
"""
import copy
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
O, A, HIDDEN, B, SEED = 11, 3, (24, 24), 48, 4
MODES = [(twin, rep, auto) for twin in (False, True) for rep in (True, False) for auto in (True, False)]
_MODE_IDS = ["%s-%s-%s" % ("twin" if t else "single", "reparam" if r else "score", "autoalpha" if a else "alpha1")
             for t, r, a in MODES]


# ----------------------------------------------------------------------------------------------- oracle port
class SACVPort:
    """SAC.update / TwinSAC.update (sac.py:74-208, twin_sac.py:82-229) op for op on the CPU, without the assert."""

    def __init__(self, pf, vf, qf1, qf2, act_dim, plr=3e-4, vlr=3e-4, qlr=3e-4, discount=0.99, tau=0.005,
                 std_reg=1e-3, mean_reg=1e-3, reparameterization=True, automatic_entropy_tuning=True, grad_clip=None):
        import torch
        self.pf, self.vf, self.qf1, self.qf2 = pf, vf, qf1, qf2
        self.tvf = copy.deepcopy(vf)
        self.qfs = [q for q in (qf1, qf2) if q is not None]
        self.q_opts = [torch.optim.Adam(q.parameters(), lr=qlr) for q in self.qfs]
        self.vf_opt = torch.optim.Adam(vf.parameters(), lr=vlr)
        self.pf_opt = torch.optim.Adam(pf.parameters(), lr=plr)
        self.auto = automatic_entropy_tuning
        if self.auto:
            self.target_entropy = -float(act_dim)
            self.log_alpha = torch.zeros(1, requires_grad=True)
            self.alpha_opt = torch.optim.Adam([self.log_alpha], lr=plr)
        self.discount, self.tau, self.std_reg, self.mean_reg = discount, tau, std_reg, mean_reg
        self.reparameterization, self.grad_clip = reparameterization, grad_clip

    def update(self, batch):
        import torch
        from oracle.ref_port import _polyak
        mse = torch.nn.functional.mse_loss
        rewards = torch.Tensor(batch["rewards"])
        terminals = torch.Tensor(batch["terminals"])
        obs = torch.Tensor(batch["obs"])
        actions = torch.Tensor(batch["acts"])
        next_obs = torch.Tensor(batch["next_obs"])
        s = self.pf.explore(obs, return_log_probs=True)
        mean, log_std, new_actions, log_probs = s["mean"], s["log_std"], s["action"], s["log_prob"]
        q_preds = [q([obs, actions]) for q in self.qfs]
        v_pred = self.vf(obs)
        if self.auto:
            alpha_loss = -(self.log_alpha * (log_probs + self.target_entropy).detach()).mean()
            self.alpha_opt.zero_grad()
            alpha_loss.backward()
            self.alpha_opt.step()
            alpha = self.log_alpha.exp()
        else:
            alpha = 1
        target_v = self.tvf(next_obs)
        q_target = rewards + (1. - terminals) * self.discount * target_v
        q_losses = [mse(q, q_target.detach()) for q in q_preds]
        q_new = self.qfs[0]([obs, new_actions])
        if len(self.qfs) > 1:
            q_new = torch.min(q_new, self.qfs[1]([obs, new_actions]))
        v_target = q_new - alpha * log_probs
        vf_loss = mse(v_pred, v_target.detach())
        if not self.reparameterization:
            policy_loss = (log_probs * (alpha * log_probs - (q_new - v_pred)).detach()).mean()
        else:
            policy_loss = (alpha * log_probs - q_new).mean()
        policy_loss = policy_loss + (self.std_reg * (log_std ** 2).mean() + self.mean_reg * (mean ** 2).mean())
        norms = []
        for opt, loss, net in ([(self.pf_opt, policy_loss, self.pf)] + list(zip(self.q_opts, q_losses, self.qfs))
                               + [(self.vf_opt, vf_loss, self.vf)]):
            opt.zero_grad()
            loss.backward()
            if self.grad_clip:
                norms.append(torch.nn.utils.clip_grad_norm_(net.parameters(), self.grad_clip))
            opt.step()
        _polyak(self.vf, self.tvf, self.tau)
        info = {"Reward_Mean": rewards.mean().item()}
        if self.auto:
            info["Alpha"] = alpha.item()
            info["Alpha_loss"] = alpha_loss.item()
        names = ["qf"] if len(self.qfs) == 1 else ["qf1", "qf2"]
        info["Training/policy_loss"] = policy_loss.item()
        info["Training/vf_loss"] = vf_loss.item()
        for n, l in zip(names, q_losses):
            info["Training/%s_loss" % n] = l.item()
        if self.grad_clip:
            for n, g in zip(["pf"] + names + ["vf"], norms):
                info["Training/%s_grad_norm" % n] = g.item()
        for name, t_ in (("log_std", log_std), ("log_probs", log_probs), ("mean", mean)):
            info[name + "/mean"] = t_.mean().item()
            info[name + "/std"] = t_.std().item()
            info[name + "/max"] = t_.max().item()
            info[name + "/min"] = t_.min().item()
        return info

    @property
    def nets(self):
        return [self.pf] + self.qfs + [self.vf, self.tvf]


def _batches(o=O, a=A, n=4, rows=B, seed=SEED):
    rs = np.random.RandomState(seed)
    return [{"obs": rs.randn(rows, o), "next_obs": rs.randn(rows, o), "acts": np.tanh(rs.randn(rows, a)),
             "rewards": rs.randn(rows, 1), "terminals": (rs.rand(rows, 1) < 0.1).astype(np.float64)} for _ in range(n)]


def _port(twin, rep, auto, grad_clip=None, o=O, a=A, hidden=HIDDEN, seed=SEED, lr=3e-4):
    import torch
    import torch.nn as nn
    from oracle import ref_port
    torch.manual_seed(seed)
    pf = ref_port.TanhGaussianPolicy(o, a, list(hidden), nn.ReLU, state_dependent_std=True)
    q1 = ref_port.QNet(o + a, 1, list(hidden), nn.ReLU)
    q2 = ref_port.QNet(o + a, 1, list(hidden), nn.ReLU) if twin else None
    vf = ref_port.MLPNet(o, 1, list(hidden), nn.ReLU)
    return SACVPort(pf, vf, q1, q2, a, plr=lr, vlr=lr, qlr=lr, reparameterization=rep, automatic_entropy_tuning=auto,
                    grad_clip=grad_clip)


# ----------------------------------------------------------------------------------------------- reference, CPU
_REF_SCRIPT = r"""
import pickle, sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
from oracle import reference_loader
reference_loader.load()
import gym
import torchrl.networks as networks, torchrl.policies as policies
from torchrl.algo.off_policy.sac import SAC
from torchrl.algo.off_policy.twin_sac import TwinSAC
twin, rep, auto = %(twin)r, %(rep)r, %(auto)r
o, a, hidden, seed = %(o)d, %(a)d, %(hidden)r, %(seed)d
batches = pickle.load(open(%(batches)r, "rb"))
torch.manual_seed(seed)
net = dict(hidden_shapes=list(hidden), append_hidden_shapes=[], base_type=networks.MLPBase,
           activation_func=torch.nn.ReLU)
pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, tanh_action=True, **net)
qf1 = networks.QNet(input_shape=o + a, output_shape=1, **net)
qf2 = networks.QNet(input_shape=o + a, output_shape=1, **net) if twin else None
vf = networks.Net(input_shape=o, output_shape=1, **net)
class Env:
    action_space = gym.spaces.Box(-np.ones(a), np.ones(a))
    observation_space = gym.spaces.Box(-np.ones(o), np.ones(o))
class Col:
    epoch_frames = 1
common = dict(env=Env(), replay_buffer=None, collector=Col(), logger=None, discount=0.99, batch_size=len(batches[0]["obs"]),
              device="cpu", save_dir=%(tmp)r, tau=0.005, use_soft_update=True, plr=3e-4, vlr=3e-4, qlr=3e-4,
              policy_std_reg_weight=1e-3, policy_mean_reg_weight=1e-3, reparameterization=rep,
              automatic_entropy_tuning=auto)
agent = TwinSAC(pf=pf, vf=vf, qf1=qf1, qf2=qf2, **common) if twin else SAC(pf=pf, vf=vf, qf=qf1, **common)
torch.manual_seed(100)
infos = [agent.update(b) for b in batches]
params = [p.detach().numpy().copy() for n_ in agent.networks for p in n_.parameters()]
pickle.dump((infos, params), open(%(out)r, "wb"))
"""


def _run_reference(tmp_path, twin, rep, auto, optimize=True, rows=B):
    import pickle
    bpath, out = tmp_path / "batches.pkl", tmp_path / "ref.pkl"
    pickle.dump(_batches(rows=rows), open(bpath, "wb"))
    script = tmp_path / "ref_sac_v.py"
    script.write_text(_REF_SCRIPT % dict(root=ROOT, twin=twin, rep=rep, auto=auto, o=O, a=A, hidden=HIDDEN,
                                         seed=SEED, batches=str(bpath), tmp=str(tmp_path), out=str(out)))
    r = subprocess.run([sys.executable] + (["-O"] if optimize else []) + [str(script)], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    return r, (pickle.load(open(out, "rb")) if r.returncode == 0 else None)


@pytest.mark.reference
@pytest.mark.parametrize("twin,rep,auto", MODES, ids=_MODE_IDS)
def test_port_reproduces_reference_under_O(tmp_path, twin, rep, auto):
    import torch
    r, got = _run_reference(tmp_path, twin, rep, auto)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ref_infos, ref_params = got
    torch.set_num_threads(torch.get_num_threads())
    port = _port(twin, rep, auto)
    torch.manual_seed(100)
    port_infos = [port.update(b) for b in _batches()]
    for x, y in zip(ref_infos, port_infos):
        assert x.keys() == y.keys()
        for k in x:
            assert x[k] == y[k] or (np.isnan(x[k]) and np.isnan(y[k])), k
    port_params = [p.detach().numpy() for n_ in port.nets for p in n_.parameters()]
    assert len(ref_params) == len(port_params)
    for x, y in zip(ref_params, port_params):
        np.testing.assert_array_equal(x, y)


@pytest.mark.reference
@pytest.mark.parametrize("twin", [False, True])
def test_reference_update_raises_at_its_assert(tmp_path, twin):
    """Without -O the reference's own update stops at `assert v_target == v_pred` for a batch of more than one
    row (the truth value of a (B, 1) tensor is ambiguous): why the oracle is the reference under -O."""
    r, _ = _run_reference(tmp_path, twin, True, True, optimize=False)
    assert r.returncode != 0
    assert "assert v_target == v_pred" in r.stderr, r.stderr[-3000:]


# ----------------------------------------------------------------------------------------------- kernel, GPU
def _np_sac_v(lp, q1, q2, v, alpha, rep):
    lp, q1, v = (np.asarray(x, np.float64) for x in (lp, q1, v))
    n = lp.size
    m = q1 if q2 is None else np.minimum(q1, np.asarray(q2, np.float64))
    t = m - alpha * lp
    vf_loss = np.mean((v - t) ** 2)
    g_v = 2 * (v - t) / n
    if rep:
        loss = np.mean(alpha * lp - m)
        g_lp = np.full(n, alpha / n)
        if q2 is None:
            g1, g2 = np.full(n, -1.0 / n), None
        else:
            q2d = np.asarray(q2, np.float64)
            g1 = np.where(q1 < q2d, -1.0 / n, np.where(q1 > q2d, 0.0, -0.5 / n))
            g2 = np.where(q2d < q1, -1.0 / n, np.where(q2d > q1, 0.0, -0.5 / n))
    else:
        c = alpha * lp - (m - v)
        loss = np.mean(lp * c)
        g_lp = c / n
        g1, g2 = np.zeros(n), (None if q2 is None else np.zeros(n))
    std = np.std(lp, ddof=1) if n > 1 else np.nan
    return loss, vf_loss, g_lp, g1, g2, g_v, [lp.mean(), std, lp.max(), lp.min()]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 4096, 65537])
@pytest.mark.parametrize("twin,rep,dev_alpha", [(True, True, True), (True, False, True), (False, True, False),
                                                (False, False, True), (True, True, False)])
def test_sac_v_loss_kernel_matches_fp64(n, twin, rep, dev_alpha):
    import torch
    from torchrl_b200 import ops
    rs = np.random.RandomState(n + 7 * twin + 3 * rep)
    lp, q1, q2, v = (rs.randn(n).astype(np.float32) for _ in range(4))
    q2[::3] = q1[::3]                                                  # exact ties on some rows
    T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()    # noqa: E731
    la = T(np.array([-0.4], np.float32)) if dev_alpha else None
    alpha = float(np.exp(np.float32(-0.4))) if dev_alpha else 1.0
    if dev_alpha:
        alpha = float(torch.exp(la).item())
    sc = ops.OffPolicyScratch(n, "cuda")
    g_lp, g1, g2, g_v, info = ops.sac_v_loss(T(lp), T(q1), T(q2) if twin else None, T(v), la, sc,
                                             reparameterization=rep)
    loss, vl, e_lp, e1, e2, e_v, st = _np_sac_v(lp, q1, q2 if twin else None, v, alpha, rep)
    info = info.cpu().numpy()
    assert abs(info[0] - loss) <= 1e-5 * max(1.0, abs(loss)), (info[0], loss)
    assert abs(info[1] - vl) <= 1e-5 * max(1.0, abs(vl)), (info[1], vl)
    np.testing.assert_allclose(info[[2, 4, 5]], [st[0], st[2], st[3]], rtol=1e-5, atol=1e-6)
    if n == 1:
        assert np.isnan(info[3])                                       # torch's std of one element
    else:
        np.testing.assert_allclose(info[3], st[1], rtol=1e-5)
    np.testing.assert_allclose(g_lp.cpu().numpy(), e_lp, rtol=1e-5, atol=5e-6 / n)    # fp32 cancellation in c
    np.testing.assert_allclose(g1.cpu().numpy(), e1, rtol=1e-6, atol=0)
    np.testing.assert_allclose(g_v.cpu().numpy(), e_v, rtol=1e-5, atol=5e-6 / n)      # fp32 cancellation in v - t
    if twin:
        np.testing.assert_allclose(g2.cpu().numpy(), e2, rtol=1e-6, atol=0)
    else:
        assert g2 is None


@pytest.mark.gpu
def test_sac_v_loss_kernel_all_rows_tied_and_terminal_targets():
    """Every row tied (torch.min splits the gradient), and the single-critic no-entropy TD target with terminal
    rows that feeds the critic MSE."""
    import torch
    from torchrl_b200 import ops
    n = 300
    rs = np.random.RandomState(5)
    lp, q, v = (rs.randn(n).astype(np.float32) for _ in range(3))
    T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()    # noqa: E731
    sc = ops.OffPolicyScratch(n, "cuda")
    _, g1, g2, _, info = ops.sac_v_loss(T(lp), T(q), T(q.copy()), T(v), None, sc)
    np.testing.assert_allclose(g1.cpu().numpy(), np.full(n, -0.5 / n), rtol=1e-6)
    np.testing.assert_allclose(g2.cpu().numpy(), np.full(n, -0.5 / n), rtol=1e-6)
    assert abs(info[0].item() - np.mean(lp.astype(np.float64) - q)) < 1e-5
    r, tv = rs.randn(n).astype(np.float32), rs.randn(n).astype(np.float32)
    d = (rs.rand(n) < 0.3).astype(np.uint8)
    d[:5] = 1
    y, _ = ops.td_target(T(r), T(d), T(tv), None, None, None, 0.99, sc)
    np.testing.assert_allclose(y.cpu().numpy(), r + (1.0 - d) * 0.99 * tv.astype(np.float64), rtol=1e-6, atol=1e-6)
    assert np.array_equal(y.cpu().numpy()[:5], r[:5])


def test_sac_v_loss_rejects_bad_arguments(native_lib):
    """Empty batch and NULL required pointers are refused before any launch, like the neighbouring entry points;
    the message is left in trl_last_error()."""
    import ctypes
    from torchrl_b200 import _lib
    L = native_lib
    p = ctypes.c_void_p(16)
    args = lambda B, **k: [k.get(n, p) for n in ("lp", "q1", "q2", "v", "la")] + [1.0, 1, B] + \
        [k.get(n, p) for n in ("g_lp", "g1", "g2", "g_v", "info", "sc", "tk")] + [None]   # noqa: E731
    for kw, msg in [(dict(B=0), "empty batch"), (dict(B=-3), "empty batch"), (dict(B=8, lp=None), "null pointer"),
                    (dict(B=8, v=None), "null pointer"), (dict(B=8, g_v=None), "null pointer"),
                    (dict(B=8, info=None), "null pointer"), (dict(B=8, sc=None), "null pointer"),
                    (dict(B=8, g2=None), "without g_qn2")]:
        B_ = kw.pop("B")
        rc = L.trl_sac_v_loss(*args(B_, **kw))
        assert rc != 0
        assert msg in L.trl_last_error().decode(), L.trl_last_error()
    assert _lib.load() is L


# ----------------------------------------------------------------------------------------------- agent, GPU
class _Env:
    def __init__(self, o, a):
        from torchrl_b200.spaces import Box
        self.action_space = Box(-np.ones(a), np.ones(a))
        self.observation_space = Box(-np.ones(o), np.ones(o))


class _Col:
    epoch_frames = 1


class _RB:
    env_nums = 1


def _device_agent(twin, rep, auto, grad_clip=None, o=O, a=A, hidden=HIDDEN, seed=SEED, rows=B, lr=3e-4,
                  use_cuda_graph=False):
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import SAC, TwinSAC
    torch.manual_seed(seed)
    net = dict(hidden_shapes=list(hidden), append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=nn.ReLU)
    pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, tanh_action=True, **net)
    qf1 = networks.QNet(input_shape=o + a, output_shape=1, **net)
    qf2 = networks.QNet(input_shape=o + a, output_shape=1, **net) if twin else None
    vf = networks.Net(input_shape=o, output_shape=1, **net)
    common = dict(env=_Env(o, a), replay_buffer=_RB(), collector=_Col(), logger=None, discount=0.99, batch_size=rows,
                  device="cuda:0", save_dir=None, tau=0.005, use_soft_update=True, use_cuda_graph=use_cuda_graph,
                  plr=lr, vlr=lr, qlr=lr, policy_std_reg_weight=1e-3, policy_mean_reg_weight=1e-3,
                  reparameterization=rep, automatic_entropy_tuning=auto, grad_clip=grad_clip)
    if twin:
        return TwinSAC(pf=pf, vf=vf, qf1=qf1, qf2=qf2, **common)
    return SAC(pf=pf, vf=vf, qf=qf1, **common)


def _compare_agent_and_port(twin, rep, auto, grad_clip=None, batches=None, o=O, a=A, hidden=HIDDEN, rows=B,
                            s_rtol=2e-3, s_atol=2e-4, p_atol=2e-4, p_bound=None):
    import torch
    from torchrl_b200.policies import set_noise_mode
    batches = batches if batches is not None else _batches()
    port = _port(twin, rep, auto, grad_clip, o=o, a=a, hidden=hidden)
    torch.manual_seed(100)
    port_infos = [port.update(b) for b in batches]
    set_noise_mode("reference_cpu")
    try:
        agent = _device_agent(twin, rep, auto, grad_clip, o=o, a=a, hidden=hidden, rows=rows)
        torch.manual_seed(100)
        infos = [agent.update(b) for b in batches]
    finally:
        set_noise_mode("philox")
    for u, (mine, ref) in enumerate(zip(infos, port_infos)):
        assert mine.keys() == ref.keys(), (mine.keys(), ref.keys())
        for k, v in ref.items():
            assert abs(mine[k] - v) <= s_rtol * abs(v) + s_atol, (u, k, mine[k], v)
    mine = torch.cat([p.detach().reshape(-1) for n in agent.networks for p in n.parameters()]).cpu().numpy()
    ref = torch.cat([p.detach().reshape(-1) for n in port.nets for p in n.parameters()]).numpy()
    if p_bound is None:
        np.testing.assert_allclose(mine, ref, atol=p_atol)
    else:
        err = np.abs(mine - ref)
        assert np.mean(err <= p_atol) >= 0.999, np.sort(err)[-10:]
        assert err.max() <= p_bound, err.max()
    return agent


@pytest.mark.gpu
@pytest.mark.parametrize("twin,rep,auto", MODES, ids=_MODE_IDS)
def test_agent_update_matches_port(twin, rep, auto):
    import torch
    torch.set_num_threads(4)
    agent = _compare_agent_and_port(twin, rep, auto)
    assert [type(t).__name__ for _, t in agent.target_networks] == [type(agent.vf).__name__]


@pytest.mark.gpu
def test_agent_update_with_grad_clip_matches_port():
    import torch
    torch.set_num_threads(4)
    _compare_agent_and_port(True, True, True, grad_clip=0.05)


def _build_pipeline(twin, N=32, T_rows=64, use_graph=True, seed=0, batch_rows=4, opt_times=6, num_epochs=3):
    import torch
    import torch.nn as nn
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import SAC, TwinSAC
    from torchrl_b200.collector import VecCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import BaseReplayBuffer
    from torchrl_b200.utils import NullLogger
    dev = torch.device("cuda:0")
    env = get_vec_env("SynthAnt-v0", {"reward_scale": 1, "obs_norm": False}, N)
    eval_env = get_vec_env("SynthAnt-v0", {"reward_scale": 1, "obs_norm": False}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    o, a = env.observation_space.shape[0], env.action_space.shape[0]
    buf = BaseReplayBuffer(env_nums=N, max_replay_buffer_size=T_rows * N, time_limit_filter=False)
    net = dict(hidden_shapes=[32, 32], append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=nn.ReLU)
    pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, tanh_action=True, **net)
    qfs = [networks.QNet(input_shape=o + a, output_shape=1, **net) for _ in range(2 if twin else 1)]
    vf = networks.Net(input_shape=o, output_shape=1, **net)
    col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=buf, device=dev, epoch_frames=8 * N,
                       max_episode_frames=20, use_cuda_graph=use_graph)
    common = dict(env=env, replay_buffer=buf, collector=col, logger=NullLogger(), discount=0.99,
                  batch_size=batch_rows * N, device=dev, save_dir=None, tau=0.005, use_soft_update=True,
                  opt_times=opt_times, pretrain_epochs=1, num_epochs=num_epochs, use_cuda_graph=use_graph, plr=3e-4,
                  vlr=3e-4, qlr=3e-4, policy_std_reg_weight=1e-3, policy_mean_reg_weight=1e-3)
    if twin:
        agent = TwinSAC(pf=pf, vf=vf, qf1=qfs[0], qf2=qfs[1], **common)
    else:
        agent = SAC(pf=pf, vf=vf, qf=qfs[0], **common)
    return agent, col, buf, env


@pytest.mark.gpu
@pytest.mark.parametrize("twin", [False, True])
def test_pipeline_graph_vs_eager(twin):
    import torch
    runs = []
    for use_graph in (False, True):
        agent, col, buf, env = _build_pipeline(twin, use_graph=use_graph)
        agent.pretrain()
        for epoch in range(3):
            agent.current_epoch = epoch
            col.train_one_epoch()
            agent.update_per_epoch()
        runs.append((agent, buf, [dict(i) for i in agent._last_infos]))
    (a0, b0, i0), (a1, b1, i1) = runs
    for k in ("obs", "next_obs", "acts", "rewards"):
        torch.testing.assert_close(getattr(b0, "_" + k), getattr(b1, "_" + k), rtol=1e-4, atol=1e-5, msg=k)
    torch.testing.assert_close(a0.opt.data, a1.opt.data, rtol=1e-3, atol=1e-5)
    torch.testing.assert_close(a0._target_flat.data, a1._target_flat.data, rtol=1e-3, atol=1e-5)
    assert len(i0) == len(i1) == 6
    for d0, d1 in zip(i0, i1):
        assert d0.keys() == d1.keys()
        assert "Training/vf_loss" in d0 and "Alpha" in d0
        for k in d0:
            assert abs(d0[k] - d1[k]) <= 2e-3 * max(1.0, abs(d0[k])), (k, d0[k], d1[k])
            assert np.isfinite(d0[k]), k


@pytest.mark.gpu
def test_twin_sac_resume_continues_identically(tmp_path):
    import torch
    path = str(tmp_path / "ck.pt")
    agent, col, buf, env = _build_pipeline(True, seed=1, use_graph=False)
    for e in range(3):
        agent.current_epoch = e
        col.train_one_epoch()
        agent.update_per_epoch()
    agent.save_checkpoint(path)
    agent.current_epoch = 3
    col.train_one_epoch()
    agent.update_per_epoch()
    want, want_t = agent.opt.data.clone(), agent._target_flat.data.clone()
    want_la, want_st = agent.log_alpha.clone(), agent._alpha_state.clone()
    agent2, col2, buf2, env2 = _build_pipeline(True, seed=77, use_graph=False)
    assert agent2.load_checkpoint(path) == 3
    agent2.current_epoch = 3
    col2.train_one_epoch()
    agent2.update_per_epoch()
    torch.testing.assert_close(agent2.opt.data, want, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(agent2._target_flat.data, want_t, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(agent2.log_alpha, want_la, rtol=1e-6, atol=1e-8)
    torch.testing.assert_close(agent2._alpha_state, want_st, rtol=1e-6, atol=1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("twin", [False, True])
def test_update_at_baseline_sizes_matches_port(twin):
    """One update at BASELINE config-3 sizes -- batch 4096 (1024 envs x 4 rows) of SynthAnt-shaped data, MLP(256,256),
    the default network mode: the value network runs through the wgmma GEMM and the 1-wide skinny head.
    Parameters: 99.9 % of the elements within atol 5e-4, every element within 2*lr + 5e-4 -- Adam's first step moves
    a weight by about lr * sign(g), so a gradient element that is zero up to rounding may step either way."""
    import torch
    from torchrl_b200.env.synth_spec import SPECS
    torch.set_num_threads(8)
    o, a = SPECS["SynthAnt-v0"][:2]
    batches = _batches(o=o, a=a, n=1, rows=4096, seed=11)
    _compare_agent_and_port(twin, True, True, batches=batches, o=o, a=a, hidden=(256, 256), rows=4096,
                            s_rtol=5e-3, s_atol=5e-4, p_atol=5e-4, p_bound=2 * 3e-4 + 5e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,agent_name", [("sac_synth_ant.json", "SAC"), ("twin_sac_synth_ant.json", "TwinSAC")])
def test_config_runs_through_compat(tmp_path, cfg_name, agent_name):
    """Each config drives 2 short epochs of `from torchrl.algo import SAC / TwinSAC` through compat/ (the alias of
    this package under the reference's name) and writes log.csv with the update's keys."""
    cfg = json.load(open(os.path.join(ROOT, "config", cfg_name)))
    n = 32
    cfg["replay_buffer"]["size"] = n * 64
    cfg["collector"].update(epoch_frames=n * 8, max_episode_frames=30)
    cfg["general_setting"].update(num_epochs=2, batch_size=n * 4, opt_times=5, eval_interval=1, save_interval=1,
                                  pretrain_epochs=1)
    cfg["net"]["hidden_shapes"] = [32, 32]
    cfg_path = tmp_path / cfg_name
    json.dump(cfg, open(cfg_path, "w"))
    key = "twin_sac" if agent_name == "TwinSAC" else "sac"
    critics = "qf1=qfs[0], qf2=qfs[1]" if agent_name == "TwinSAC" else "qf=qfs[0]"
    script = tmp_path / "run.py"
    script.write_text(_DRIVER % dict(agent=agent_name, key=key, nq=2 if agent_name == "TwinSAC" else 1,
                                     critics=critics))
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "compat"), ROOT, env.get("PYTHONPATH", "")])
    r = subprocess.run([sys.executable, str(script), "--config", str(cfg_path), "--vec_env_nums", str(n), "--seed",
                        "1", "--log_dir", str(tmp_path / "log"), "--overwrite"], capture_output=True, text=True,
                       timeout=900, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    work = tmp_path / "log" / os.path.splitext(cfg_name)[0] / cfg["env_name"] / "1"
    rows = open(work / "log.csv").read().strip().splitlines()
    assert len(rows) >= 3, rows
    crit = ["Training/qf1_loss", "Training/qf2_loss"] if agent_name == "TwinSAC" else ["Training/qf_loss"]
    for k in ["Reward_Mean", "Alpha", "Alpha_loss", "Training/policy_loss", "Training/vf_loss", "log_std/mean",
              "log_probs/std", "mean/max"] + crit:
        assert k + "_Mean" in rows[0], (k, rows[0])
    assert "model_vf_finish.pth" in set(os.listdir(work / "model"))


# a user's launcher written against the reference's API: every import resolves through compat/torchrl
_DRIVER = r"""
import random
import numpy as np
import torch
import torchrl.networks as networks
import torchrl.policies as policies
from torchrl.algo import %(agent)s
from torchrl.collector import VecCollector
from torchrl.env import get_vec_env
from torchrl.replay_buffers import BaseReplayBuffer
from torchrl.utils import Logger, get_args, get_params

args = get_args()
params = get_params(args.config)
dev = torch.device("cuda:0")
env = get_vec_env(params["env_name"], params["env"], args.vec_env_nums, device=dev)
eval_env = get_vec_env(params["env_name"], params["env"], args.vec_env_nums, device=dev)
env.seed(args.seed); torch.manual_seed(args.seed); np.random.seed(args.seed); random.seed(args.seed)
logger = Logger(args.config.split("/")[-1][:-5], params["env_name"], args.seed, params, args.log_dir, args.overwrite)
o, a = env.observation_space.shape[0], env.action_space.shape[0]
trunk = dict(params["net"], base_type=networks.MLPBase, activation_func=torch.nn.ReLU)
pf = policies.GuassianContPolicy(input_shape=o, output_shape=2 * a, **trunk, **params["policy"])
qfs = [networks.QNet(input_shape=o + a, output_shape=1, **trunk) for _ in range(%(nq)d)]
vf = networks.Net(input_shape=o, output_shape=1, **trunk)
rb = params["replay_buffer"]
ring = BaseReplayBuffer(env_nums=args.vec_env_nums, max_replay_buffer_size=int(rb["size"]),
                        time_limit_filter=rb["time_limit_filter"])
col = VecCollector(env=env, eval_env=eval_env, pf=pf, replay_buffer=ring, device=dev, train_render=False,
                   **params["collector"])
agent = %(agent)s(pf=pf, vf=vf, %(critics)s, env=env, replay_buffer=ring, collector=col, logger=logger, device=dev,
                  save_dir=logger.work_dir + "/model", **params["general_setting"], **params["%(key)s"])
agent.train()
"""
