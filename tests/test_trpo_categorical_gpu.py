"""Discrete TRPO on the H100: the three TRPO kernels against fp64 at their edges, the agent's Fisher-vector product,
conjugate-gradient solve and update(batch) against the executed reference (tests/golden/trpo_categorical_reference.npz,
oracle/make_golden_trpo_categorical.py), launch counts, the pixel epoch with and without CUDA graphs, checkpoint
resume, the launcher and the refusal of unsupported policies."""
import csv
import math
import os

import numpy as np
import pytest

from oracle import make_golden_categorical as cat
from oracle import make_golden_trpo_categorical as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trpo_categorical_reference.npz")


def _softmax64(z):
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _logits(M, A, seed, saturate=True):
    rs = np.random.RandomState(seed)
    z = rs.randn(M, A).astype(np.float32) * 2.0
    if saturate and A > 1:
        sat = np.arange(M) % 3 == 0
        z[sat] = (rs.randn(int(sat.sum()), A) * 12.0).astype(np.float32)
        z[sat, rs.randint(0, A, int(sat.sum()))] += 20.0
    return z, rs.randn(M, A).astype(np.float32)


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("M", [1, 31, 32, 33, 65537])
@pytest.mark.parametrize("A", [1, 2, 6, 18])
def test_fisher_vp_matches_fp64(M, A):
    import torch
    from torchrl_b200 import ops
    z, t = _logits(M, A, M * 31 + A)
    scale = 0.37
    g = ops.categorical_fisher_vp(torch.as_tensor(z, device="cuda"), torch.as_tensor(t, device="cuda"), scale)
    p = _softmax64(z)
    want = scale * (p * t - p * (p * t).sum(-1, keepdims=True))
    got = g.cpu().numpy()
    # per row: relative to the row's scale (p * |t|), which is what fp32 resolves
    tol = 1e-6 * scale * (p * np.abs(t)).sum(-1, keepdims=True) + 1e-30
    assert np.all(np.abs(got - want) <= tol + 2e-6 * np.abs(want)), np.abs(got - want).max()
    if A == 1:
        assert not got.any()


def test_fisher_vp_on_the_golden_kernel_cases():
    """Against the reference's own double backward with the logits as parameters (its mean over rows: 1 / M)."""
    import torch
    from torchrl_b200 import ops
    r = G.load(GOLDEN)
    for case, (M, A, _) in G.KERNEL_CASES.items():
        z, t = G.kernel_inputs(case)
        got = ops.categorical_fisher_vp(torch.as_tensor(z, device="cuda"), torch.as_tensor(t, device="cuda"),
                                        1.0 / M).cpu().numpy().astype(np.float64)
        want = r[case]["hvp"]["float64"]
        if A == 1:
            assert not got.any()
            continue
        assert np.linalg.norm(got - want) <= 1e-6 * np.linalg.norm(want), case


@pytest.mark.parametrize("layout", ["nchw", "mh", "odd"])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_tangent_bias_act_is_bit_identical_to_torch(layout, act):
    import torch
    from torchrl_b200 import ops
    torch.manual_seed(7 + act)
    shape = {"nchw": (33, 16, 20, 20), "mh": (65537, 6), "odd": (7, 3, 5, 3)}[layout]
    t = torch.randn(shape, device="cuda")
    y = torch.randn(shape, device="cuda")
    if act == 1:
        y = torch.tanh(y)
    elif act == 2:
        y = torch.relu(y)
        t[0].fill_(float("inf"))                                     # inf * 0 = nan where y == 0, as in torch
    db = torch.randn(shape[1], device="cuda")
    bshape = (1, shape[1]) + (1,) * (len(shape) - 2)
    want = t + db.view(bshape)
    if act == 1:
        want = want * (1 - y * y)
    elif act == 2:
        want = want * (y > 0)
    got = ops.tangent_bias_act(t.clone(), db, y, act)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    # an unaligned view takes the scalar path with the same result
    flat = torch.empty(t.numel() + 1, device="cuda")
    tv = flat[1:].view(shape)
    tv.copy_(t)
    ops.tangent_bias_act(tv, db, y, act)
    assert torch.equal(tv.view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("M", [1, 31, 32, 33, 65537])
@pytest.mark.parametrize("A", [1, 2, 6, 18])
def test_surrogate_matches_fp64_and_is_deterministic(M, A):
    import torch
    from torchrl_b200 import ops
    z, _ = _logits(M, A, 5 * M + A)
    rs = np.random.RandomState(M + A)
    acts = rs.randint(0, A, M).astype(np.float32)
    advn = rs.randn(M).astype(np.float32)
    zd = torch.as_tensor(z, device="cuda")
    ad = torch.as_tensor(acts, device="cuda")
    old = ops.categorical_log_prob(zd + 0.1 * torch.as_tensor(_logits(M, A, 9)[1], device="cuda"), ad)
    sc = ops.SurrogateScratch(M, "cuda")
    a = ops.categorical_surrogate(zd, ad, old, torch.as_tensor(advn, device="cuda"), sc).clone()
    b = ops.categorical_surrogate(zd, ad, old, torch.as_tensor(advn, device="cuda"), sc).clone()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))                 # bit for bit, run to run
    logp = ops.categorical_log_prob(zd, ad)                                      # the same clamp
    ratio = np.exp(logp.cpu().numpy().astype(np.float64) - old.cpu().numpy().astype(np.float64))
    want = -np.mean(ratio * advn)
    assert abs(float(a) - want) <= 1e-5 * np.mean(np.abs(ratio * advn)) + 1e-7, (float(a), want)


# ------------------------------------------------------------------------------------------ the agent
class _Logger(cat._NullLogger):
    def __init__(self):
        self.infos = []

    def add_update_info(self, info):
        self.infos.append(info)


def _state(rec, net):
    import torch
    return {k[len(net) + 1:]: torch.as_tensor(v) for k, v in rec.items() if k.startswith(net + ".")}


def _golden_agent(case, r, **kw):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import TRPO
    from torchrl_b200.spaces import Box, Discrete
    arch, act = G.CASES[case][:2]

    class Env:
        action_space = Discrete(G.A)
        observation_space = Box(-np.ones(11), np.ones(11))
    nk = cat.net_kwargs(networks, torch, arch)
    nk["activation_func"] = torch.nn.Tanh if act == "tanh" else torch.nn.ReLU
    pf = policies.CategoricalDisPolicy(output_shape=G.A, **nk)
    vf = networks.Net(output_shape=1, **nk)
    pf.load_state_dict(_state(r["init"], "pf"))
    vf.load_state_dict(_state(r["init"], "vf"))
    args = dict(G.KW, **kw)
    return TRPO(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=cat._Col(), logger=_Logger(), discount=0.99,
                num_epochs=10, batch_size=64, gae=True, device="cuda:0", save_dir=None, shuffle=True, tau=0.95,
                use_cuda_graph=False, **args)


@pytest.fixture
def no_tf32():
    import torch
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


@pytest.fixture
def deterministic_cudnn():
    import torch
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_fisher_vector_product_matches_the_reference(case, no_tf32):
    import torch
    r = G.load(GOLDEN)[case]
    agent = _golden_agent(case, r)
    arch, act, n, B, seed, lead = G.CASES[case]
    batch = G.batches(arch, n, B, seed, lead)[0]
    nparam = sum(p.numel() for p in agent.pf.parameters())
    assert [n for n, _ in agent.pf.named_parameters()] == list(r["meta"]["names"])
    for s in G.HVP_SEEDS:
        v = torch.as_tensor(G.directions(nparam, s), device="cuda")
        got = agent.fisher_vector_product(batch, v).cpu().numpy().astype(np.float64)
        want = r["hvp32"][str(s)].astype(np.float64)
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-5 * np.abs(want).max(), err_msg=str(s))
    # the first update's conjugate-gradient solve of F x = -g (fp64 dot products, 10 iterations)
    b = torch.as_tensor(r["cg"]["b"], device="cuda")
    x = agent._conjugate_gradient(lambda p: agent.fisher_vector_product(batch, p), b).cpu().numpy()
    want = r["cg"]["x"]
    assert np.linalg.norm(x - want) <= 2e-3 * np.linalg.norm(want), np.linalg.norm(x - want) / np.linalg.norm(want)


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_update_matches_reference(case, no_tf32):
    """Tolerances of test_onpolicy_algos.py::test_trpo_update_matches_reference: infos rtol 5e-3 + atol 5e-4,
    parameters atol 2e-2 * step + 1e-5, each update continuing from the reference's parameters."""
    r = G.load(GOLDEN)[case]
    agent = _golden_agent(case, r)
    arch, act, n, B, seed, lead = G.CASES[case]
    p0 = {k: v for k, v in r["init"].items() if k.startswith("pf.")}
    for u, b in enumerate(G.batches(arch, n, B, seed, lead)):
        info = agent.update(b)
        want = r["info%d" % u]
        assert set(want) == set(info), (sorted(want), sorted(info))
        for k, v in want.items():
            assert abs(info[k] - v) <= 5e-3 * abs(v) + 5e-4, (u, k, info[k], v)
        pr = r["pf%d" % u]
        step = max(float(np.abs(pr[k] - p0[k]).max()) for k in pr)
        assert step > 1e-5, "the reference took no step: the test would be vacuous"
        mine = agent.pf.state_dict()
        for k in pr:
            np.testing.assert_allclose(mine[k[3:]].cpu().numpy(), pr[k], atol=2e-2 * step + 1e-5, err_msg=k)
        agent.pf.load_state_dict(_state(pr, "pf"))
        p0 = pr


def test_one_fisher_launch_per_product_and_one_surrogate_launch_per_candidate():
    from torchrl_b200 import _lib
    case = "trpo_cnn"
    r = G.load(GOLDEN)[case]
    agent = _golden_agent(case, r)
    arch, act, n, B, seed, lead = G.CASES[case]
    counts, products, candidates = {}, [0], [0]
    call, fvp, score = _lib.call, agent._fvp, agent._head.trpo_score

    def counting(name, *a, **kw):
        counts[name] = counts.get(name, 0) + 1
        return call(name, *a, **kw)

    def counted_fvp(*a, **kw):
        products[0] += 1
        return fvp(*a, **kw)

    def counted_score(*a, **kw):
        candidates[0] += 1
        return score(*a, **kw)
    _lib.call, agent._fvp, agent._head.trpo_score = counting, counted_fvp, counted_score
    try:
        agent.update(G.batches(arch, n, B, seed, lead)[0])
    finally:
        _lib.call = call
    assert products[0] == G.KW["cg_iters"] + 1 and candidates[0] >= 2, (products, candidates)
    assert counts["trl_categorical_fisher_vp"] == products[0], counts
    assert counts["trl_categorical_surrogate"] == candidates[0], counts
    # the conv layers' and the linear layers' bias / activation steps: one launch per layer per product
    assert counts["trl_tangent_bias_act"] == products[0] * len(agent._plan), counts


def test_unsupported_policies_are_rejected():
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import TRPO
    from torchrl_b200.spaces import Box, Discrete

    class Env:
        action_space = Discrete(G.A)
        observation_space = Box(-np.ones(11), np.ones(11))
    kw = dict(input_shape=(11,), hidden_shapes=[32, 32], base_type=networks.MLPBase, activation_func=torch.nn.Tanh)
    bad = [policies.CategoricalDisPolicy(output_shape=G.A, add_ln=True, **kw),
           policies.GuassianContPolicy(output_shape=3, **kw)]
    for pf in bad:
        with pytest.raises(NotImplementedError, match="CategoricalDisPolicy"):
            TRPO(pf=pf, vf=networks.Net(output_shape=1, **kw), env=Env(), replay_buffer=None, collector=cat._Col(),
                 logger=_Logger(), discount=0.99, num_epochs=10, batch_size=64, device="cuda:0", save_dir=None,
                 **G.KW)


# ------------------------------------------------------------------------------------------ the pixel path
def _pixel_agent(N=16, T=8, use_graph=True, seed=0, max_frames=5, batch_rows=4):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import TRPO
    from torchrl_b200.collector import VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    dev = torch.device("cuda:0")
    env = get_vec_env("SynthAtari-v0", {}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    net = dict(input_shape=(4, 84, 84), hidden_shapes=cat.CNN["hidden"], append_hidden_shapes=[16],
               base_type=networks.CNNBase, activation_func=torch.nn.ReLU)
    pf, vf = policies.CategoricalDisPolicy(output_shape=6, **net), networks.Net(output_shape=1, **net)
    col = VecOnPolicyCollector(vf, env=env, pf=pf, replay_buffer=buf, device=dev, train_render=False,
                               epoch_frames=T * N, max_episode_frames=max_frames, eval_episodes=1,
                               use_cuda_graph=use_graph)
    agent = TRPO(pf=pf, vf=vf, env=env, replay_buffer=buf, collector=col, logger=_Logger(), discount=0.99,
                 num_epochs=10, batch_size=batch_rows * N, gae=True, device=dev, save_dir=None, shuffle=True,
                 tau=0.95, use_cuda_graph=use_graph, plr=3e-4, vlr=3e-4, max_kl=0.01, cg_damping=0.1, cg_iters=10,
                 residual_tol=1e-10, entropy_coeff=0.01, v_opt_times=2)
    return agent, col, buf, env


def test_pixel_epoch_graph_path_equals_eager_path(no_tf32):
    import torch
    runs = []
    for g in (False, True):
        agent, col, buf, env = _pixel_agent(use_graph=g, seed=2)
        p0 = agent.opt.data.clone()
        for epoch in range(2):
            agent.current_epoch = epoch
            col.train_one_epoch()
            agent.update_per_epoch()
        infos = agent.logger.infos
        assert infos and all(math.isfinite(v) for i in infos for v in i.values())
        keys = set().union(*infos)
        assert {"advs/mean", "Training/policy_loss", "logprob/mean", "Training/vf_loss", "grad_norm/vf"} <= keys
        seg = slice(agent.opt.seg_begin[0], agent.opt.seg_begin[1])
        assert float((agent.opt.data[seg] - p0[seg]).abs().max()) > 0, "no policy step was taken"
        runs.append((agent.opt.data.clone(), infos))
    (d0, i0), (d1, i1) = runs
    torch.testing.assert_close(d0, d1, rtol=1e-3, atol=2e-5)
    assert len(i0) == len(i1)
    for a, b in zip(i0, i1):
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-3 * max(1.0, abs(a[k])), (k, a[k], b[k])


def test_resume_continues_identically(tmp_path, deterministic_cudnn):
    """With deterministic cuDNN algorithms (the conjugate-gradient solve amplifies the last-bit differences of
    cuDNN's atomics-based weight gradients), the resumed run repeats the uninterrupted one."""
    import torch
    path = str(tmp_path / "ck.pt")

    def epochs(agent, col, first, n):
        out = []
        for e in range(first, first + n):
            agent.current_epoch = e
            out.append(col.train_one_epoch()["train_epoch_reward"])
            agent.update_per_epoch()
        return out
    agent, col, buf, env = _pixel_agent(use_graph=False, seed=3)
    epochs(agent, col, 0, 2)
    agent.save_checkpoint(path)
    want_r = epochs(agent, col, 2, 2)
    want = agent.opt.data.clone()
    want_acts = buf._acts.clone()
    agent2, col2, buf2, env2 = _pixel_agent(use_graph=False, seed=99)
    assert agent2.load_checkpoint(path) == 2
    got_r = epochs(agent2, col2, 2, 2)
    np.testing.assert_allclose(got_r, want_r, rtol=1e-5)
    assert torch.equal(buf2._acts, want_acts)
    torch.testing.assert_close(agent2.opt.data, want, rtol=1e-5, atol=1e-7)


def test_launcher_trains_on_a_shrunken_config(tmp_path):
    from tests.test_examples import _run

    def patch(c):
        n = 16
        c["replay_buffer"]["size"] = n * 16
        c["collector"].update(epoch_frames=n * 16, max_episode_frames=40)
        c["general_setting"].update(num_epochs=3, batch_size=n * 4, eval_interval=1, save_interval=1)
        c["net"].update(hidden_shapes=cat.CNN["hidden"], append_hidden_shapes=[32])
    work = _run("trpo_atari_vec.py", "trpo_synth_atari.json", patch, 16, tmp_path)
    assert "model_pf_finish.pth" in set(os.listdir(work / "model"))
    rows = list(csv.DictReader(open(work / "log.csv")))
    assert len(rows) == 3
    for key in ("Training/policy_loss", "Training/vf_loss", "logprob/mean", "Train_Epoch_Reward"):
        cols = [c for c in rows[0] if c.startswith(key)]
        assert cols, (key, list(rows[0]))
        assert all(math.isfinite(float(r[c])) for r in rows for c in cols), key
