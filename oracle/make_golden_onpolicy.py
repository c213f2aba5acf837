"""Golden data of tests/test_onpolicy_algos.py: the reference's own A2C, V-MPO and TRPO `update(batch)` executed on
torch CPU (the unmodified reference behind oracle/shims), recorded so that the device algorithms can be checked
against it on a machine without a copy of the reference.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/reference_loader.available()):

    python oracle/make_golden_onpolicy.py         # -> tests/golden/onpolicy_reference.npz

Recorded per case: the initial policy / value state_dicts (the device agents start from them), the logged scalars of
every update, the parameters after the last one; TRPO also the sampled actions of each batch, the policy after every
update and the value-function sweeps (`update_vf`); V-MPO the final temperature / KL multiplier.  The batches
themselves are regenerated from their seeds by the test (`batches`).  Keys: "<case>|<what>|<name>".
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "onpolicy_reference.npz")

O, A, HID = 11, 3, (32, 32)
KW = {
    "a2c": dict(plr=1e-3, vlr=1e-3, entropy_coeff=0.01),
    "vmpo": dict(plr=1e-3, vlr=1e-3, opt_epochs=2, alpha_eps=0.01),
    "trpo": dict(plr=3e-4, vlr=1e-3, max_kl=0.01, cg_damping=0.1, cg_iters=10, residual_tol=1e-10, entropy_coeff=0.01,
                 v_opt_times=2),
}
# case -> (algorithm, number of batches, batch rows, batch seed, leading batch shape)
CASES = {
    "a2c": ("a2c", 4, 64, 0, None),
    "vmpo": ("vmpo", 4, 64, 1, None),
    "trpo_flat": ("trpo", 2, 128, 2, None),
    "trpo_lead": ("trpo", 2, 128, 2, (8, 16)),
}


def batches(n, B, seed, lead=None):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        shape = (B,) if lead is None else lead
        obs = rs.randn(*shape, O)
        acts = np.tanh(0.4 * rs.randn(*shape, A))
        out.append(dict(obs=obs, acts=acts, advs=rs.randn(*shape, 1), estimate_returns=rs.randn(*shape, 1),
                        values=rs.randn(*shape, 1)))
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


def _reference_agent(kind, save_dir):
    import torch
    from oracle import reference_loader
    reference_loader.load()                  # puts the gym / tensorboardX shims on sys.path
    import gym
    import torchrl.networks as networks
    import torchrl.policies as policies
    from torchrl.algo import A2C, TRPO, VMPO

    class Env:
        action_space = gym.spaces.Box(-np.ones(A), np.ones(A))
        observation_space = gym.spaces.Box(-np.ones(O), np.ones(O))
    torch.manual_seed(3)
    net = dict(hidden_shapes=list(HID), append_hidden_shapes=[], base_type=networks.MLPBase, activation_func=torch.nn.Tanh)
    pf = policies.GuassianContPolicyBasicBias(input_shape=O, output_shape=A, tanh_action=True, **net)
    vf = networks.Net(input_shape=(O,), output_shape=1, **net)
    cls = {"a2c": A2C, "vmpo": VMPO, "trpo": TRPO}[kind]
    return cls(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=_Col(), logger=_NullLogger(), discount=0.99,
               num_epochs=10, batch_size=64, gae=True, device="cpu", save_dir=save_dir, shuffle=True, tau=0.95,
               **KW[kind])


def _put_params(rec, case, what, agent, names=("pf", "vf")):
    for n in names:
        for k, v in getattr(agent, n).state_dict().items():
            rec["%s|%s|%s.%s" % (case, what, n, k)] = v.detach().cpu().numpy().astype(np.float64)


def _put_info(rec, case, what, info):
    for k, v in info.items():
        rec["%s|%s|%s" % (case, what, k)] = np.float64(v)


def record():
    import torch
    rec = {}
    for case, (kind, n, B, seed, lead) in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            ref = _reference_agent(kind, tmp)
            _put_params(rec, case, "init", ref)
            bs = batches(n, B, seed, lead)
            if kind != "trpo":
                for u, b in enumerate(bs):
                    _put_info(rec, case, "info%d" % u, ref.update(b))
                _put_params(rec, case, "final", ref)
                if kind == "vmpo":
                    rec["%s|dual|eta" % case] = np.float64(float(ref.eta))
                    rec["%s|dual|alpha" % case] = np.float64(float(ref.alpha))
                continue
            # actions the policy could have produced (log-probs of arbitrary actions underflow exp() in the ratio)
            for i, b in enumerate(bs):
                with torch.no_grad():
                    o = torch.as_tensor(b["obs"], dtype=torch.float32)
                    mean, std, _ = ref.pf(o)
                    b["acts"] = torch.tanh(mean + std * torch.randn_like(mean)).numpy().astype(np.float64)
                rec["%s|acts|%d" % (case, i)] = b["acts"]
            for i, b in enumerate(bs):
                _put_info(rec, case, "info%d" % i, ref.update(b))
                _put_params(rec, case, "pf%d" % i, ref, ("pf",))
            for i, b in enumerate(bs):
                flat = dict(obs=b["obs"].reshape(-1, O), estimate_returns=b["estimate_returns"].reshape(-1, 1))
                _put_info(rec, case, "vfinfo%d" % i, ref.update_vf(flat))
            _put_params(rec, case, "final", ref, ("vf",))
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
