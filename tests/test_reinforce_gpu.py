"""REINFORCE on the device (torchrl_b200/algo/on_policy/reinforce.py) against the executed reference's updates
(tests/golden/reinforce_reference.npz; the tolerances of the A2C / V-MPO golden tests) and against an fp64 torch
restatement of reinforce.py:33-75, eagerly and through the captured minibatch epoch; the captured graph's host
syncs and launch count; and the launcher on CartPole and on the pixel env."""
import csv
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import make_golden_reinforce as G
from tests.test_reinforce_cpu import reinforce_fp64, reference_nets

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reinforce_reference.npz")


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


def _agent(case, r, use_graph=False, buf=None, collector=None):
    import torch
    from torchrl_b200.algo import Reinforce
    from torchrl_b200.spaces import Box, Discrete
    O, A = G.CASES[case][:2]

    class Env:
        action_space = Box(-np.ones(A), np.ones(A)) if case == "gauss" else Discrete(A)
        observation_space = Box(-np.ones(O), np.ones(O))
    pf = reference_nets(case, torch)
    pf.load_state_dict({k[3:]: torch.as_tensor(v, dtype=torch.float32) for k, v in r["init"].items()})
    return Reinforce(pf=pf, env=Env(), replay_buffer=buf, collector=collector or G._Col(), logger=_Logger(),
                     discount=0.99, num_epochs=10, batch_size=64, device="cuda:0", save_dir=None, shuffle=False,
                     use_cuda_graph=use_graph, **G.KW)


def _check_infos(got, want):
    assert list(got) == list(want), (list(got), list(want))
    for k, v in want.items():
        assert abs(got[k] - v) <= 2e-3 * abs(v) + 2e-4, (k, got[k], v)


def _check_params(pf, want):
    for k, v in pf.state_dict().items():
        np.testing.assert_allclose(v.detach().cpu().numpy(), want["pf." + k], atol=2e-4, err_msg=k)


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_eager_update_matches_reference_and_fp64(case):
    r = G.load(GOLDEN)[case]
    agent = _agent(case, r)
    bs = G.batches(case)
    infos = [agent.update(b) for b in bs]
    for u, info in enumerate(infos):
        _check_infos(info, r["info%d" % u])
    _check_params(agent.pf, r["pf%d" % (len(bs) - 1)])
    f64_infos, f64_params = reinforce_fp64(case, r["init"], bs)
    for info, want in zip(infos, f64_infos):
        _check_infos(info, want)
    _check_params(agent.pf, f64_params)


def _filled_buffer(case, bs):
    """The golden batches as the rows of a rollout buffer: N = 64 envs, row t = batch t."""
    import torch
    from torchrl_b200.replay_buffers import OnPolicyReplayBuffer
    O, A, n, B, _ = G.CASES[case]
    buf = OnPolicyReplayBuffer(env_nums=B, max_replay_buffer_size=n * B)
    buf.allocate("obs", (B, O))
    buf.allocate("acts", (B, A) if case == "gauss" else (B,))
    buf.allocate("rewards", (B, 1))
    buf.allocate("advs", (B, 1))
    for t, b in enumerate(bs):
        buf._obs[t] = torch.as_tensor(b["obs"])
        buf._acts[t] = torch.as_tensor(b["acts"], dtype=torch.float32).reshape(buf._acts[t].shape)
        buf._advs[t] = torch.as_tensor(b["advs"], dtype=torch.float32)
    return buf


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_captured_epoch_matches_reference(case):
    """Every minibatch of the epoch replays the captured graph (the warm-up ran on a twin agent): advantage table,
    loss kernel, log-prob statistics, clip + Adam, one info read-back."""
    import torch
    r = G.load(GOLDEN)[case]
    bs = G.batches(case)
    twin = _agent(case, r, use_graph=True, buf=_filled_buffer(case, bs))
    twin._minibatch_epoch(True)                       # three eager minibatches, then capture: shared scratch is warm
    buf = _filled_buffer(case, bs)
    agent = _agent(case, r, use_graph=True, buf=buf)
    agent._mb_eager_runs = 3
    agent._minibatch_epoch(True)
    assert agent._mb_graph is not None
    for u, info in enumerate(agent._last_infos):
        _check_infos(info, r["info%d" % u])
    _check_params(agent.pf, r["pf%d" % (len(bs) - 1)])
    # the replays issue no host synchronisation
    agent._mb_state["upd"].zero_()
    agent._epoch_adv_stats()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(len(bs)):
            agent._run_minibatch()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def profile_epoch_launches():
    """(graph?, _lib.launch_count() delta, library kernels the profiler saw) of one eager and one captured epoch."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from torchrl_b200 import _lib
    r = G.load(GOLDEN)["cat"]
    bs = G.batches("cat")
    agent = _agent("cat", r, use_graph=True, buf=_filled_buffer("cat", bs))
    agent._minibatch_epoch(True)
    out = []
    for graph in (False, True):
        agent.use_cuda_graph = graph
        torch.cuda.synchronize()
        before = _lib.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            agent._minibatch_epoch(True)
            torch.cuda.synchronize()
        out.append((graph, _lib.launch_count() - before, [e.name for e in prof.events() if "trl::" in e.name]))
    return out


def test_launch_count_matches_the_profiler():
    """Run in a fresh process, so that what the profiler records does not depend on what the suite ran before."""
    code = ("import json\nfrom tests.test_reinforce_gpu import profile_epoch_launches\n"
            "print(json.dumps(profile_epoch_launches()))\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    for graph, counted, kernels in json.loads(res.stdout.strip().splitlines()[-1]):
        assert counted == len(kernels), (graph, counted, len(kernels))
        assert sum("vec_stats" in k for k in kernels) == len(G.batches("cat"))      # logprob/* once per minibatch


# ------------------------------------------------------------------------------------------ launcher
def test_launcher_on_cartpole_and_on_pixels(tmp_path):
    from tests.test_examples import _run

    def cartpole(c):
        c["general_setting"].update(num_epochs=3, epoch_frames=512, batch_size=256, save_interval=1)
        c["replay_buffer"]["size"] = 512

    def atari(c):
        n = 16
        c["replay_buffer"]["size"] = n * 16
        c["collector"].update(epoch_frames=n * 16, max_episode_frames=40)
        c["general_setting"].update(num_epochs=3, batch_size=n * 4, eval_interval=1, save_interval=1)
        c["net"].update(hidden_shapes=[[8, [8, 8], [4, 4], [0, 0]], [8, [4, 4], [2, 2], [0, 0]]],
                        append_hidden_shapes=[16])
    for name, cfg, patch, n in (("cp", "reinforce_cartpole.json", cartpole, 8),
                                ("atari", "reinforce_synth_atari.json", atari, 16)):
        d = tmp_path / name
        d.mkdir()
        work = _run("reinforce_vec.py", cfg, patch, n, d)
        assert "model_pf_finish.pth" in set(os.listdir(work / "model"))
        rows = list(csv.DictReader(open(work / "log.csv")))
        assert len(rows) == 3
        for key in ("advs/mean", "advs/std", "Training/policy_loss", "ent", "logprob/mean", "logprob/std",
                    "logprob/max", "logprob/min", "Train_Epoch_Reward", "Running_Average_Rewards"):
            cols = [c for c in rows[0] if c.startswith(key)]
            assert cols, (key, list(rows[0]))
            assert all(math.isfinite(float(r[c])) for r in rows for c in cols), key
