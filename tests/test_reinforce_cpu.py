"""REINFORCE without a GPU: the golden recording against an fp64 torch restatement of the reference's update
(reinforce.py:33-75), its inputs regenerated from their seeds, and the agent's reachability through compat/."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import make_golden_reinforce as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reinforce_reference.npz")


def reference_nets(case, torch):
    """The policy of a golden case, built from torchrl_b200 (the weights come from the recording)."""
    import torchrl_b200.networks as networks
    import torchrl_b200.policies as policies
    O, A = G.CASES[case][:2]
    net = dict(hidden_shapes=list(G.HID), append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=torch.nn.Tanh)
    if case == "gauss":
        return policies.GuassianContPolicyBasicBias(input_shape=O, output_shape=A, tanh_action=True, **net)
    return policies.CategoricalDisPolicy(input_shape=O, output_shape=A, **net)


def reinforce_fp64(case, init, bs):
    """reinforce.py:33-75 in float64 on the CPU: the infos of every update (advs/* as NumPy computes them) and the final
    policy parameters, from the recorded initial weights."""
    import torch
    pf = reference_nets(case, torch).double()
    pf.load_state_dict({k[3:]: torch.as_tensor(v, dtype=torch.float64) for k, v in init.items()})
    opt = torch.optim.Adam(pf.parameters(), lr=G.KW["plr"])
    infos = []
    for b in bs:
        advs_np = np.asarray(b["advs"], np.float64)
        info = {'advs/mean': advs_np.mean(), 'advs/std': advs_np.std(), 'advs/max': advs_np.max(),
                'advs/min': advs_np.min()}
        obs = torch.as_tensor(b["obs"], dtype=torch.float64)
        acts = torch.as_tensor(b["acts"], dtype=torch.float64)
        advs = torch.as_tensor(advs_np)
        out = pf.update(obs, acts if case == "gauss" else acts.long())
        log_probs, ent = out["log_prob"], out["ent"]
        advs = (advs - advs.mean()) / (advs.std() + 1e-5)
        assert log_probs.shape == advs.shape
        loss = (-log_probs * advs).mean() - G.KW["entropy_coeff"] * ent.mean()
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(pf.parameters(), 0.5)
        opt.step()
        info['Training/policy_loss'] = loss.item()
        info['ent'] = ent.mean().item()
        for k, f in (("mean", torch.mean), ("std", torch.std), ("max", torch.max), ("min", torch.min)):
            info['logprob/' + k] = f(log_probs).item()
        infos.append({k: float(v) for k, v in info.items()})
    return infos, {"pf." + k: v.detach().numpy() for k, v in pf.state_dict().items()}


@pytest.fixture(scope="module")
def golden():
    return G.load(GOLDEN)


def test_recorded_inputs_regenerate_from_their_seeds(golden):
    assert sorted(golden) == sorted(G.CASES)
    for case, (O, A, n, B, seed) in G.CASES.items():
        bs = G.batches(case)
        assert len(bs) == n
        for u, b in enumerate(bs):
            want = golden[case]["info%d" % u]
            assert b["obs"].shape == (B, O) and b["advs"].shape == (B, 1)
            assert b["acts"].shape == ((B, A) if case == "gauss" else (B,))
            # the recorded advs/* are the NumPy statistics of the regenerated advantages
            assert abs(want["advs/mean"] - b["advs"].mean()) <= 1e-12 * abs(b["advs"].mean()) + 1e-12
            assert abs(want["advs/std"] - b["advs"].std()) <= 1e-12 * b["advs"].std()
            assert want["advs/max"] == b["advs"].max() and want["advs/min"] == b["advs"].min()
        assert sorted(golden[case]["init"]) == sorted(golden[case]["pf%d" % (n - 1)])


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_fp64_restatement_matches_the_recording(golden, case):
    r = golden[case]
    infos, params = reinforce_fp64(case, r["init"], G.batches(case))
    for u, info in enumerate(infos):
        want = r["info%d" % u]
        assert list(info) == list(want)
        for k, v in want.items():
            assert abs(info[k] - v) <= 1e-4 * abs(v) + 1e-5, (u, k, info[k], v)
    for k, v in params.items():
        np.testing.assert_allclose(v, r["pf%d" % (len(infos) - 1)][k], atol=1e-5, err_msg=k)


@pytest.mark.reference
def test_generator_reproduces_the_committed_golden_data():
    fresh = G.record()
    with np.load(GOLDEN) as z:
        assert sorted(fresh) == sorted(z.files)
        for k, v in fresh.items():
            np.testing.assert_allclose(v, z[k], rtol=1e-6, atol=1e-7, err_msg=k)


def test_reinforce_resolves_through_compat(tmp_path):
    code = ("import torchrl\nfrom torchrl.algo import Reinforce\nimport torchrl_b200.algo as a\n"
            "assert Reinforce is a.Reinforce and 'Reinforce' in a.__all__\n"
            "from torchrl.networks.nets import ZeroNet\nprint('ok')\n")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "compat"), ROOT])
    env["TORCHRL_B200_NO_AUTOBUILD"] = "1"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


def test_reinforce_keeps_the_reference_constructor():
    import inspect
    from torchrl_b200.algo import Reinforce
    sig = inspect.signature(Reinforce.__init__)
    assert list(sig.parameters)[:5] == ["self", "pf", "plr", "optimizer_class", "entropy_coeff"]
    assert sig.parameters["entropy_coeff"].default == 0.001
    assert Reinforce.adam_eps == 1e-8
