"""Golden data of tests/test_reinforce_*.py: the reference's own `Reinforce.update(batch)` executed on torch CPU (the
unmodified reference behind oracle/shims), recorded so that the device agent can be checked on a machine without a
copy of the reference.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/reference_loader.available()):

    python oracle/make_golden_reinforce.py         # -> tests/golden/reinforce_reference.npz

Recorded per case, keys "<case>|<what>|<name>": the initial policy state_dict (the device agent starts from it), the
infos of every update ("info<u>") and the policy after every update ("pf<u>").  Cases:
  * "gauss": GuassianContPolicyBasicBias (tanh actions) on an MLP, O = 11, A = 3, acts (B, A), advs (B, 1);
  * "cat":   CategoricalDisPolicy on CartPole's MLP shape, O = 4, A = 2, acts (B,), advs (B, 1).
These are the two batch layouts the reference's `assert log_probs.shape == advs.shape` accepts.  The batches are
regenerated from their seeds by the tests (`batches`).
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "reinforce_reference.npz")

HID = (32, 32)
KW = dict(plr=3e-3, entropy_coeff=0.01)
# case -> (obs dim, action dim / number of actions, number of updates, batch rows, batch seed)
CASES = {"gauss": (11, 3, 4, 64, 30), "cat": (4, 2, 4, 64, 31)}


def batches(case):
    O, A, n, B, seed = CASES[case]
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        obs = rs.randn(B, O).astype(np.float32)
        if case == "gauss":
            acts = np.tanh(0.4 * rs.randn(B, A))
        else:
            acts = rs.randint(0, A, B).astype(np.float64)
        # discounted-return-like advantages: positive, with a spread, as a REINFORCE batch has them
        advs = 5.0 + 3.0 * rs.randn(B, 1)
        out.append(dict(obs=obs, acts=acts, advs=advs))
    return out


class _NullLogger:
    def add_update_info(self, info):
        pass

    def add_epoch_info(self, *a, **k):
        pass

    def log(self, *a):
        pass

    def finish(self):
        pass


class _Col:
    epoch_frames = 64


def _reference_agent(case, save_dir):
    import torch
    from oracle import reference_loader
    reference_loader.load()                  # puts the gym / tensorboardX shims on sys.path
    import gym
    import torchrl.networks as networks
    import torchrl.policies as policies
    from torchrl.algo import Reinforce

    O, A = CASES[case][:2]

    class Env:
        action_space = gym.spaces.Box(-np.ones(A), np.ones(A)) if case == "gauss" else gym.spaces.Discrete(A)
        observation_space = gym.spaces.Box(-np.ones(O), np.ones(O))
    torch.manual_seed(4)
    net = dict(hidden_shapes=list(HID), append_hidden_shapes=[], base_type=networks.MLPBase,
               activation_func=torch.nn.Tanh)
    if case == "gauss":
        pf = policies.GuassianContPolicyBasicBias(input_shape=O, output_shape=A, tanh_action=True, **net)
    else:
        pf = policies.CategoricalDisPolicy(input_shape=O, output_shape=A, **net)
    return Reinforce(pf=pf, env=Env(), replay_buffer=None, collector=_Col(), logger=_NullLogger(), discount=0.99,
                     num_epochs=10, batch_size=64, device="cpu", save_dir=save_dir, shuffle=True, **KW)


def _put_params(rec, case, what, agent):
    for k, v in agent.pf.state_dict().items():
        rec["%s|%s|pf.%s" % (case, what, k)] = v.detach().cpu().numpy().astype(np.float64)


def record():
    rec = {}
    for case in CASES:
        with tempfile.TemporaryDirectory() as tmp:
            ref = _reference_agent(case, tmp)
            _put_params(rec, case, "init", ref)
            for u, b in enumerate(batches(case)):
                for k, v in ref.update(b).items():
                    rec["%s|info%d|%s" % (case, u, k)] = np.float64(v)
                _put_params(rec, case, "pf%d" % u, ref)
    return rec


def load(path=OUT):
    """{case: {what: {name: value}}} of a recorded file."""
    out = {}
    with np.load(path) as z:
        for key in z.files:
            case, what, name = key.split("|", 2)
            v = z[key]
            out.setdefault(case, {}).setdefault(what, {})[name] = v if v.ndim else float(v)
    return out


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    rec = record()
    np.savez_compressed(OUT, **rec)
    print("%s: %d arrays, %d bytes" % (OUT, len(rec), os.path.getsize(OUT)))
