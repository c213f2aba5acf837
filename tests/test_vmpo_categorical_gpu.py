"""Discrete V-MPO on the device: the top-half selection kernel exactly against NumPy, the categorical V-MPO loss kernel
against the fp64 restatement at its edges (both KL modes), the agent against the reference's own updates
(tests/golden/vmpo_categorical_reference.npz; tolerances of test_onpolicy_algos.py), the captured epoch on the pixel
collector against eager updates of a twin, the launch counts, checkpoint resume and the launcher."""
import csv
import math
import os

import numpy as np
import pytest

from oracle import make_golden_categorical as cat
from oracle import make_golden_vmpo_categorical as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vmpo_categorical_reference.npz")


def _stats(x):
    """[mean, unbiased std, max, min] as float32, a (1, 4) row."""
    x = np.asarray(x, np.float64)
    sd = x.std(ddof=1) if x.size > 1 else 0.0
    return np.array([[x.mean(), sd, x.max(), x.min()]], np.float32)


# ------------------------------------------------------------------------------------------ selection
@pytest.mark.parametrize("B", [1, 2, 3, 255, 256, 257, 4096, 65537])
def test_selection_matches_numpy(B):
    import torch
    from torchrl_b200 import ops
    rs = np.random.RandomState(B)
    cases = [rs.randn(B), np.round(rs.randn(B) * 3) / 3, np.full(B, 0.5)]    # distinct, many ties, all equal
    for adv in cases:
        adv = adv.astype(np.float32)
        st = _stats(adv)
        got = ops.vmpo_select(torch.tensor(adv, device="cuda"), torch.tensor(st, device="cuda"), 1, B)
        want = G.select(G.normalise(adv, st[0, 0], st[0, 1]))
        np.testing.assert_array_equal(got.cpu().numpy().reshape(-1), want)


def test_selection_of_every_minibatch_in_one_launch():
    """Several groups per launch through a row permutation, in gather_rows order, with ties at each boundary."""
    import torch
    from torchrl_b200 import ops
    rs = np.random.RandomState(0)
    T, N, b = 24, 37, 4
    passes = 2
    adv = (np.round(rs.randn(T, N, 1) * 2) / 2).astype(np.float32)
    adv[5] = 0.25                                                   # a whole row of equal values
    perm = np.concatenate([rs.permutation(T) for _ in range(passes)])
    U = passes * T // b
    groups = [adv[perm[u * b:(u + 1) * b]].reshape(-1) for u in range(U)]
    table = np.concatenate([_stats(g) for g in groups])
    got = ops.vmpo_select(torch.tensor(adv, device="cuda").reshape(T, -1), torch.tensor(table, device="cuda"), U, b,
                          perm=torch.tensor(perm, device="cuda")).cpu().numpy()
    B = b * N
    assert got.shape == (U, B - B // 2)
    for u in range(U):
        np.testing.assert_array_equal(got[u], G.select(G.normalise(groups[u], table[u, 0], table[u, 1])), err_msg=u)


# ------------------------------------------------------------------------------------------ loss kernel
def _loss_case(k, A, seed, saturate=False, zero_q=False, big=False):
    rs = np.random.RandomState(seed)
    z = (rs.randn(k, A) * 2).astype(np.float32)
    if saturate:
        z[::2, 0] += 40.0                                          # p_0 > 1 - eps: the clamp is active
    zq = (z + rs.randn(k, A) * 0.5).astype(np.float32)
    if zero_q and A > 1:
        zq[0, 1] -= 300.0                                          # q_1 == 0 exactly: that row's KL is inf
        z[min(1, k - 1), A - 1] -= 300.0                           # p == 0: the term is 0
    acts = rs.randint(0, A, k).astype(np.float32)
    adv = (rs.randn(k) * (30.0 if big else 1.0)).astype(np.float32)
    mean, std = np.float32(0.1), np.float32(0.9)
    return z, zq, acts, adv, np.array([[9.0, 9.0, 0, 0], [mean, std, 0, 0]], np.float32)


EDGES = {"k1": dict(k=1, A=6), "A1": dict(k=50, A=1), "A32": dict(k=300, A=32), "sat": dict(k=600, A=6, saturate=True),
         "zero_q": dict(k=97, A=6, zero_q=True), "big": dict(k=513, A=4, big=True)}


@pytest.mark.parametrize("per_row", [False, True])
@pytest.mark.parametrize("edge", sorted(EDGES))
def test_loss_kernel_matches_fp64(edge, per_row):
    import torch
    from torchrl_b200 import ops
    kw = dict(EDGES[edge])
    k, A = kw.pop("k"), kw.pop("A")
    z, zq, acts, adv, table = _loss_case(k, A, seed=k * 33 + A, **kw)
    eta, alpha = (0.05 if edge == "big" else 0.8), 0.3                # big: advn / eta reaches well beyond 88
    d = lambda x: torch.tensor(x, device="cuda")  # noqa: E731
    dual = d(np.array([eta, alpha], np.float32))
    g_dual = torch.zeros(2, device="cuda")
    info = torch.full((12,), 7.0, device="cuda")
    scratch = ops.VMPOScratch(k, "cuda")
    pos = torch.ones(1, dtype=torch.int32, device="cuda")           # statistics row 1
    g = ops.vmpo_categorical_loss(d(z), d(zq), d(acts), d(adv), d(table), dual, 0.02, 0.1, per_row, scratch, g_dual,
                                  info, stats_pos=pos)
    advn = G.normalise(adv, table[1, 0], table[1, 1])
    if edge == "big":
        assert np.abs(advn).max() / eta > 88.0
    want, gz, geta, galpha = G.vmpo_loss(z, zq, acts, advn, np.float32(eta), np.float32(alpha), 0.02, 0.1,
                                         per_row_kl=per_row)
    got = info.cpu().numpy().astype(np.float64)
    keys = ["Training/policy_loss", "Training/alpha_loss", None, None] + \
           ["logprob/" + s for s in ("mean", "std", "max", "min")] + ["KL/" + s for s in ("mean", "std", "max", "min")]
    for i, key in enumerate(keys):
        if key is None:
            assert got[i] == 7.0                                     # slots 2, 3 are not written
            continue
        w = want[key]
        if np.isnan(w):
            assert np.isnan(got[i]), key
        elif np.isinf(w):
            assert got[i] == w, (key, got[i])
        else:
            assert abs(got[i] - w) <= 1e-4 * abs(w) + 1e-5, (key, got[i], w)
    if k == 1:
        assert np.isnan(got[5]) and np.isnan(got[9])
    if not per_row:
        assert np.isnan(got[9]) and got[8] == got[10] == got[11]
    gk = g.cpu().numpy()
    assert np.all(np.isfinite(gk))
    np.testing.assert_allclose(gk, gz, rtol=2e-4, atol=2e-6)
    gd = g_dual.cpu().numpy()
    assert abs(gd[0] - geta) <= 1e-4 * abs(geta) + 1e-5, (gd[0], geta)
    if np.isinf(galpha):
        assert gd[1] == galpha
    else:
        assert abs(gd[1] - galpha) <= 1e-4 * abs(galpha) + 1e-5, (gd[1], galpha)
    if edge == "zero_q":
        assert np.isinf(want["KL/max"])


# ------------------------------------------------------------------------------------------ the agent
class _Logger(cat._NullLogger):
    def __init__(self):
        self.infos = []

    def add_update_info(self, info):
        self.infos.append(info)


def _state(rec, net):
    import torch
    return {k[len(net) + 1:]: torch.as_tensor(v) for k, v in rec.items() if k.startswith(net + ".")}


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_update_matches_reference(case):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import VMPO
    from torchrl_b200.spaces import Box, Discrete
    arch, n, B, seed = G.CASES[case]
    r = G.load(GOLDEN)[case]

    class Env:
        action_space = Discrete(G.A)
        observation_space = Box(-np.ones(11), np.ones(11))
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        kw = cat.net_kwargs(networks, torch, arch)
        pf = policies.CategoricalDisPolicy(output_shape=G.A, **kw)
        vf = networks.Net(output_shape=1, **kw)
        pf.load_state_dict(_state(r["init"], "pf"))
        vf.load_state_dict(_state(r["init"], "vf"))
        mine = VMPO(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=cat._Col(), logger=_Logger(),
                    discount=0.99, num_epochs=10, batch_size=64, gae=True, device="cuda:0", save_dir=None,
                    shuffle=True, tau=0.95, use_cuda_graph=False, **G.KW)
        infos = [mine.update(b) for b in G.batches(arch, n, B, seed)]
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    for u, m in enumerate(infos):
        want = r["info%d" % u]
        assert set(want) == set(m), (sorted(want), sorted(m))
        for k, v in want.items():
            if math.isnan(v):
                assert math.isnan(m[k]), (u, k)
            else:
                assert abs(m[k] - v) <= 2e-3 * abs(v) + 2e-4, (u, k, m[k], v)
    for net in ("pf", "vf"):
        for k, v in getattr(mine, net).state_dict().items():
            np.testing.assert_allclose(v.detach().cpu().numpy(), r["final"]["%s.%s" % (net, k)], atol=2e-4,
                                       err_msg=k)
    np.testing.assert_allclose(mine.dual.detach().cpu().numpy(), r["final"]["dual"], atol=2e-4)


def _pixel_agent(N=16, T=8, use_graph=True, seed=0, max_frames=5, batch_rows=4, opt_epochs=2):
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    from torchrl_b200.algo import VMPO
    from torchrl_b200.collector import VecOnPolicyCollector
    from torchrl_b200.env import get_vec_env
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    dev = torch.device("cuda:0")
    env = get_vec_env("SynthAtari-v0", {}, N)
    env.seed(seed); torch.manual_seed(seed); np.random.seed(seed)
    buf = OnPolicyReplayBuffer(env_nums=N, max_replay_buffer_size=T * N, time_limit_filter=True)
    pf, vf = _pixel_nets()
    col = VecOnPolicyCollector(vf, env=env, pf=pf, replay_buffer=buf, device=dev, train_render=False,
                               epoch_frames=T * N, max_episode_frames=max_frames, eval_episodes=1,
                               use_cuda_graph=use_graph)
    agent = VMPO(pf=pf, vf=vf, env=env, replay_buffer=buf, collector=col, logger=_Logger(), discount=0.99,
                 num_epochs=10, batch_size=batch_rows * N, gae=True, device=dev, save_dir=None, shuffle=True,
                 tau=0.95, use_cuda_graph=use_graph, plr=3e-4, vlr=3e-4, opt_epochs=opt_epochs)
    return agent, col, buf, env


def _pixel_nets():
    import torch
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    net = dict(input_shape=(4, 84, 84), hidden_shapes=cat.CNN["hidden"], append_hidden_shapes=[16],
               base_type=networks.CNNBase, activation_func=torch.nn.Tanh)
    return policies.CategoricalDisPolicy(output_shape=6, **net), networks.Net(output_shape=1, **net)


def test_fused_epoch_equals_eager_updates_of_a_twin_agent():
    """The captured epoch (row gather of uint8 frames, per-epoch advantage table and top-half selection read through
    the device counter, the loss kernel on the selected rows) against `update(batch)` of a twin with the same weights
    fed the same minibatches; the twin normalises and selects per minibatch, independently of the epoch machinery.
    """
    import torch
    from torchrl_b200.algo import VMPO
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        N, T, rows, passes = 16, 32, 4, 2
        agent, col, buf, env = _pixel_agent(N=N, T=T, seed=7, max_frames=9, batch_rows=rows, opt_epochs=passes)
        agent.current_epoch = 0
        col.train_one_epoch()
        init = {n: {k: v.detach().clone() for k, v in getattr(agent, n).state_dict().items()} for n in ("pf", "vf")}
        rng = np.random.get_state()
        agent.update_per_epoch()
        assert agent._mb_graph is not None
        fused_infos = [dict(i) for i in agent._last_infos]
        pf, vf = _pixel_nets()
        pf.load_state_dict(init["pf"])
        vf.load_state_dict(init["vf"])
        twin = VMPO(pf=pf, vf=vf, env=env, replay_buffer=None, collector=cat._Col(), logger=_Logger(), discount=0.99,
                    num_epochs=10, batch_size=rows * N, gae=True, device="cuda:0", save_dir=None, shuffle=True,
                    tau=0.95, use_cuda_graph=False, plr=3e-4, vlr=3e-4, opt_epochs=passes)
        np.random.set_state(rng)
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
    U = passes * T // rows
    assert len(eager_infos) == len(fused_infos) == U
    for u, (m, want) in enumerate(zip(fused_infos, eager_infos)):
        assert set(m) == set(want), (sorted(m), sorted(want))
        for k, v in want.items():
            if math.isnan(v):
                assert math.isnan(m[k]), (u, k)
            else:
                assert abs(m[k] - v) <= 2e-3 * abs(v) + 2e-4, (u, k, m[k], v)
    for n in ("pf", "vf"):
        mine, ref = getattr(agent, n).state_dict(), getattr(twin, n).state_dict()
        assert max(float((mine[k] - init[n][k]).abs().max()) for k in mine) > 1e-4, "no step was taken"
        for k in ref:
            np.testing.assert_allclose(mine[k].cpu().numpy(), ref[k].cpu().numpy(), atol=2e-4, err_msg=n + "." + k)
    np.testing.assert_allclose(agent.dual.detach().cpu().numpy(), twin.dual.detach().cpu().numpy(), atol=2e-4)


def test_one_selection_per_epoch_and_one_loss_launch_per_minibatch():
    from torchrl_b200 import _lib
    agent, col, buf, env = _pixel_agent(use_graph=False, seed=5)
    col.train_one_epoch()
    counts = {}
    call = _lib.call

    def counting(name, *a, **kw):
        counts[name] = counts.get(name, 0) + 1
        return call(name, *a, **kw)
    _lib.call = counting
    try:
        before = _lib.launch_count()
        agent.update_per_epoch()
        launched = _lib.launch_count() - before
    finally:
        _lib.call = call
    U = agent._mb_state["U"]
    assert U == 4
    assert counts["trl_vmpo_select"] == 1 and counts["trl_vmpo_categorical_loss"] == U, counts
    assert "trl_ppo_categorical_actor_loss" not in counts
    assert launched >= sum(counts.values())


@pytest.mark.parametrize("quirks", [True, False])
def test_epoch_loop_graph_path_equals_eager_path(quirks):
    import torch
    runs = []
    for g in (False, True):
        agent, col, buf, env = _pixel_agent(use_graph=g, seed=2)
        agent.reference_quirks = quirks
        for epoch in range(3):
            agent.current_epoch = epoch
            col.train_one_epoch()
            agent.update_per_epoch()
        runs.append((agent.opt.data.clone(), [dict(i) for i in agent._last_infos]))
        assert all(np.isfinite(i["Training/policy_loss"]) and np.isfinite(i["Training/eta"])
                   for i in agent._last_infos)
        assert all(np.isnan(i["KL/std"]) == quirks for i in agent._last_infos)
    (p0, i0), (p1, i1) = runs
    torch.testing.assert_close(p0, p1, rtol=1e-3, atol=2e-5)
    for d0, d1 in zip(i0, i1):
        for k in d0:
            if not math.isnan(d0[k]):
                assert abs(d0[k] - d1[k]) <= 2e-3 * max(1.0, abs(d0[k])), (k, d0[k], d1[k])


def test_resume_continues_identically(tmp_path):
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
        c["vmpo"]["opt_epochs"] = 2
    work = _run("vmpo_atari_vec.py", "vmpo_synth_atari.json", patch, 16, tmp_path)
    assert "model_pf_finish.pth" in set(os.listdir(work / "model"))
    rows = list(csv.DictReader(open(work / "log.csv")))
    assert len(rows) == 3
    for key in ("Training/policy_loss", "Training/eta", "Training/alpha", "KL/mean", "Train_Epoch_Reward"):
        cols = [c for c in rows[0] if c.startswith(key)]
        assert cols, (key, list(rows[0]))
        assert all(math.isfinite(float(r[c])) for r in rows for c in cols), key
