"""Golden data of the categorical (discrete on-policy) path, tests/test_categorical_*.py: the unmodified reference
executed on torch CPU behind oracle/shims, recorded so that the device kernels and algorithms can be checked against it
on a machine without a copy of the reference.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/reference_loader.available()):

    python oracle/make_golden_categorical.py      # -> tests/golden/categorical_reference.npz

Recorded:
  * "dist": torch's Categorical(softmax(x)) -- what CategoricalDisPolicy.update builds -- over seeded logits, a third
    of the rows saturated (logit gaps above 16, where the probability clamp of probs_to_logits is active): log_prob and
    entropy per row, and the autograd gradients of sum(w1 * log_prob) and sum(w2 * entropy) wrt the logits;
  * the reference's A2C.update and PPO.update on an MLP (O = 11, A = 6) and on a small CNN over 4x84x84 inputs: the
    initial state_dicts (one per architecture: A2C and PPO start from the same weights), the logged scalars of every
    update and the parameters after the last one.  The reference's PPO reads out['log_std'] (ppo.py:52), which its
    CategoricalDisPolicy.update does not return; the recorded PPO runs wrap the policy so that update() also returns a
    dummy log_std, and the four log_std/* keys this produces are not recorded.
The inputs (logits, weights, batches) are regenerated from their seeds by the tests (`dist_inputs`, `batches`).
Keys: "<case>|<what>|<name>".
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "categorical_reference.npz")

A = 6
MLP = dict(obs=(11,), hidden=[32, 32], append=[])
CNN = dict(obs=(4, 84, 84), hidden=[[8, [8, 8], [4, 4], [0, 0]], [8, [4, 4], [2, 2], [0, 0]]], append=[16])
KW = {
    "a2c": dict(plr=1e-3, vlr=1e-3, entropy_coeff=0.01),
    "ppo": dict(plr=1e-3, vlr=1e-3, entropy_coeff=0.01, clip_para=0.2, opt_epochs=1),
}
# case -> (algorithm, architecture, number of batches, batch rows, batch seed)
CASES = {
    "a2c_mlp": ("a2c", "mlp", 4, 64, 10),
    "ppo_mlp": ("ppo", "mlp", 4, 64, 11),
    "a2c_cnn": ("a2c", "cnn", 2, 32, 12),
    "ppo_cnn": ("ppo", "cnn", 2, 32, 13),
}
DIST_M = 300


def dist_inputs(M=DIST_M, seed=0):
    """Seeded (M, A) logits -- rows 0, 3, 6, ... saturated -- integer actions and the two gradient weights."""
    rs = np.random.RandomState(seed)
    x = rs.randn(M, A).astype(np.float32) * 2.0
    sat = np.arange(M) % 3 == 0
    x[sat] = (rs.randn(int(sat.sum()), A) * 12.0).astype(np.float32)
    x[sat, rs.randint(0, A, int(sat.sum()))] += 20.0
    acts = rs.randint(0, A, M)
    return x, acts, rs.randn(M).astype(np.float32), rs.randn(M).astype(np.float32)


def batches(arch, n, B, seed):
    rs = np.random.RandomState(seed)
    spec = MLP if arch == "mlp" else CNN
    out = []
    for _ in range(n):
        obs = rs.randn(B, *spec["obs"]) if arch == "mlp" else rs.rand(B, *spec["obs"])
        out.append(dict(obs=obs.astype(np.float32), acts=rs.randint(0, A, B).astype(np.float32),
                        advs=rs.randn(B, 1), estimate_returns=rs.randn(B, 1), values=rs.randn(B, 1)))
    return out


def net_kwargs(networks, torch, arch):
    spec = MLP if arch == "mlp" else CNN
    base = networks.MLPBase if arch == "mlp" else networks.CNNBase
    return dict(input_shape=spec["obs"], hidden_shapes=spec["hidden"], append_hidden_shapes=list(spec["append"]),
                base_type=base, activation_func=torch.nn.Tanh)


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


def _reference_nets(arch):
    import torch
    from oracle import reference_loader
    reference_loader.load()
    import torchrl.networks as networks
    import torchrl.policies as policies

    class PolicyWithDummyLogStd(policies.CategoricalDisPolicy):
        def update(self, obs, actions):
            out = super().update(obs, actions)
            out["log_std"] = torch.zeros(1)
            return out

    torch.manual_seed(3)
    kw = net_kwargs(networks, torch, arch)
    pf = PolicyWithDummyLogStd(output_shape=A, **kw)
    vf = networks.Net(output_shape=1, **kw)
    return pf, vf


def _reference_agent(kind, arch, save_dir):
    pf, vf = _reference_nets(arch)           # loads the reference and its shims first
    import gym
    from torchrl.algo import A2C, PPO

    class Env:
        action_space = gym.spaces.Discrete(A)
        observation_space = gym.spaces.Box(-np.ones(MLP["obs"]), np.ones(MLP["obs"]))
    cls = {"a2c": A2C, "ppo": PPO}[kind]
    return cls(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=_Col(), logger=_NullLogger(), discount=0.99,
               num_epochs=10, batch_size=64, gae=True, device="cpu", save_dir=save_dir, shuffle=True, tau=0.95,
               **KW[kind])


def _put_params(rec, case, what, agent):
    for n in ("pf", "vf"):
        for k, v in getattr(agent, n).state_dict().items():
            rec["%s|%s|%s.%s" % (case, what, n, k)] = v.detach().cpu().numpy().astype(np.float32)


def record():
    import torch
    rec = {}
    # ---- the distribution itself
    x, acts, w1, w2 = dist_inputs()
    xt = torch.tensor(x, requires_grad=True)
    dis = torch.distributions.Categorical(torch.softmax(xt, dim=-1))
    lp = dis.log_prob(torch.as_tensor(acts))
    ent = dis.entropy()
    g_lp, = torch.autograd.grad((lp * torch.as_tensor(w1)).sum(), xt, retain_graph=True)
    g_ent, = torch.autograd.grad((ent * torch.as_tensor(w2)).sum(), xt)
    for k, v in (("log_prob", lp), ("entropy", ent), ("grad_log_prob", g_lp), ("grad_entropy", g_ent)):
        rec["dist|out|%s" % k] = v.detach().numpy().astype(np.float32)
    # ---- updates
    inits = {}
    for case, (kind, arch, n, B, seed) in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            ref = _reference_agent(kind, arch, tmp)
            if arch not in inits:
                inits[arch] = True
                _put_params(rec, arch, "init", ref)
            for u, b in enumerate(batches(arch, n, B, seed)):
                for k, v in ref.update(b).items():
                    if not k.startswith("log_std/"):
                        rec["%s|info%d|%s" % (case, u, k)] = np.float64(v)
            _put_params(rec, case, "final", ref)
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
