"""Golden data of discrete TRPO, tests/test_trpo_categorical_*.py: the unmodified reference executed on torch CPU behind
oracle/shims, recorded so that the device kernels and the agent can be checked on a machine without a copy of the
reference.  Also the fp64 restatement of the Fisher-vector product that the tests compare the recording against.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/reference_loader.available()):

    python oracle/make_golden_trpo_categorical.py      # -> tests/golden/trpo_categorical_reference.npz

The reference's discrete TRPO does not run as shipped (DESIGN §6 deviation 20): CategoricalDisPolicy.update returns
the distribution under "dis" where trpo.py:54-57 expects its probabilities, and a whole-rollout batch with (T, N, 1)
actions fails in Categorical.log_prob.  The recording wraps the policy so that update() returns dis.probs under "dis"
(nothing else changes) and passes (T, N) actions in the whole-rollout layout.

Recorded, keys "<case>|<what>|<name>":
  * "trpo_mlp", "trpo_mlp_tn", "trpo_cnn": the reference's TRPO.update on the MLP (O = 11, A = 6, Tanh) in the flat
    and the (T, N) layout and on the small 4x84x84 CNN of make_golden_categorical with ReLU (flat): the initial
    state_dicts ("init"), every update's infos ("info<u>") and the policy after it ("pf<u>"); before the first update,
    hessian_vector_product(v) for the seeded directions of `directions` on the first batch, as the reference runs it
    in fp32 ("hvp32|<seed>") and with the policy and the inputs cast to float64 ("hvp64|<seed>"); and the first
    update's conjugate-gradient solve: its right-hand side -g ("cg|b") and step direction ("cg|x").  "meta|names" is
    the policy's parameter order of the flat vectors;
  * "kern_sat", "kern_uniform", "kern_a1", "kern_a18": the reference's hessian_vector_product for a policy whose
    parameters are the logits themselves (J = identity, cg_damping = 0) on the seeded logits and tangents of
    `kernel_inputs` -- saturated rows (logit gaps above 16), rows of equal logits, A = 1 and A = 18 -- in fp32 and fp64.
Inputs are regenerated from their seeds (`batches`, `directions`, `kernel_inputs`).
"""
import copy
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "trpo_categorical_reference.npz")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_golden_categorical as cat  # noqa: E402

A = cat.A
KW = dict(plr=3e-4, vlr=1e-3, max_kl=0.01, cg_damping=0.1, cg_iters=10, residual_tol=1e-10, entropy_coeff=0.01,
          v_opt_times=2)
# case -> (architecture, activation, number of batches, batch rows, batch seed, leading (T, N) shape or None)
CASES = {
    "trpo_mlp": ("mlp", "tanh", 2, 64, 30, None),
    "trpo_mlp_tn": ("mlp", "tanh", 2, 64, 31, (8, 8)),
    "trpo_cnn": ("cnn", "relu", 2, 32, 32, None),
}
HVP_SEEDS = (0, 1, 2)
# kernel case -> (rows M, actions A, seed)
KERNEL_CASES = {"kern_sat": (300, 6, 40), "kern_uniform": (64, 6, 41), "kern_a1": (33, 1, 42), "kern_a18": (65, 18, 43)}


def batches(arch, n, B, seed, lead=None):
    """Explicit whole batches: obs, integer actions as float ((B,) or (T, N)), advs (..., 1)."""
    rs = np.random.RandomState(seed)
    spec = cat.MLP if arch == "mlp" else cat.CNN
    shape = (B,) if lead is None else tuple(lead)
    out = []
    for _ in range(n):
        obs = rs.randn(*shape, *spec["obs"]) if arch == "mlp" else rs.rand(*shape, *spec["obs"])
        out.append(dict(obs=obs.astype(np.float32), acts=rs.randint(0, A, shape).astype(np.float32),
                        advs=rs.randn(*shape, 1), estimate_returns=rs.randn(*shape, 1)))
    return out


def directions(n, seed):
    """A seeded float32 direction in the policy's flat parameter space."""
    return np.random.RandomState(100 + seed).randn(n).astype(np.float32)


def kernel_inputs(case):
    """(logits (M, A), tangent (M, A)) float32 of a kernel case."""
    M, a, seed = KERNEL_CASES[case]
    rs = np.random.RandomState(seed)
    z = rs.randn(M, a).astype(np.float32) * 2.0
    if case == "kern_uniform":
        z[:] = rs.randn(M, 1).astype(np.float32)            # every row uniform
        z[::4] = 0.0
    elif a > 1:
        sat = np.arange(M) % 3 == 0
        z[sat] = (rs.randn(int(sat.sum()), a) * 12.0).astype(np.float32)
        z[sat, rs.randint(0, a, int(sat.sum()))] += 20.0    # gaps above 16: the other probabilities underflow 1e-7
    t = rs.randn(M, a).astype(np.float32)
    return z, t


def kl_scale(lead):
    """What the reference's KL over probs is in units of the mean per-sample KL: with a (T, N, A) batch
    torch.sum(kl, 1) sums over the N envs and the mean runs over (T, A), i.e. N / A (trpo.py:59-61)."""
    return 1.0 if lead is None else float(lead[1]) / A


# ------------------------------------------------------------------------------------------ fp64 restatement
def restated_hvp(net, obs, v, scale, damping):
    """J^T (diag p - p p^T) J v * scale / B + damping * v in float64 with J the Jacobian of the logits of `net` (a
    torch module, any dtype: it is cast to float64 on a copy) wrt its parameters, obs (B, ...) float."""
    import torch
    from torch.func import functional_call, jvp, vjp
    net = copy.deepcopy(net).double()
    names = [n for n, _ in net.named_parameters()]
    params = {n: p.detach() for n, p in net.named_parameters()}
    x = torch.as_tensor(np.asarray(obs), dtype=torch.float64)
    vv = torch.as_tensor(np.asarray(v), dtype=torch.float64)
    tang, o = {}, 0
    for n in names:
        k = params[n].numel()
        tang[n] = vv[o:o + k].view(params[n].shape)
        o += k

    def logits(p):
        return functional_call(net, p, (x,))
    z, jv = jvp(logits, (params,), (tang,))
    p = torch.softmax(z, dim=-1)
    u = (p * jv - p * (p * jv).sum(-1, keepdim=True)) * (scale / z.shape[0])
    _, back = vjp(logits, params)
    g, = back(u)
    return (torch.cat([g[n].reshape(-1) for n in names]) + damping * vv).numpy()


# ------------------------------------------------------------------------------------------ the executed reference
def _policy_class():
    import torch  # noqa: F401
    import torchrl.policies as policies

    class ProbsPolicy(policies.CategoricalDisPolicy):
        """The reference's policy with update()["dis"] = the distribution's probabilities (what trpo.py:54-57
        expects); nothing else changes."""

        def update(self, obs, actions):
            out = super().update(obs, actions)
            out["dis"] = out["dis"].probs
            return out
    return ProbsPolicy


def _reference_nets(arch, act):
    import torch
    from oracle import reference_loader
    reference_loader.load()
    import torchrl.networks as networks
    torch.manual_seed(3)
    kw = cat.net_kwargs(networks, torch, arch)
    kw["activation_func"] = torch.nn.Tanh if act == "tanh" else torch.nn.ReLU
    return _policy_class()(output_shape=A, **kw), networks.Net(output_shape=1, **kw)


def _reference_trpo(pf, vf, save_dir):
    import gym
    from torchrl.algo import TRPO

    class Env:
        action_space = gym.spaces.Discrete(A)
        observation_space = gym.spaces.Box(-np.ones(cat.MLP["obs"]), np.ones(cat.MLP["obs"]))
    return TRPO(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=cat._Col(), logger=cat._NullLogger(),
                discount=0.99, num_epochs=10, batch_size=64, gae=True, device="cpu", save_dir=save_dir, shuffle=True,
                tau=0.95, **KW)


def _hvp(ref, obs, acts, v, dtype):
    """The reference's hessian_vector_product(v) on (obs, acts) with the policy and inputs in `dtype`."""
    import torch
    pf = ref.pf
    ref.pf = copy.deepcopy(pf).to(dtype)
    try:
        ref.obs = torch.as_tensor(obs).to(dtype)
        ref.acts = torch.as_tensor(acts).to(dtype)
        return ref.hessian_vector_product(torch.as_tensor(v).to(dtype)).detach().numpy().astype(np.float64)
    finally:
        ref.pf = pf


def _record_updates(rec):
    import contextlib
    import io
    for case, (arch, act, n, B, seed, lead) in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            pf, vf = _reference_nets(arch, act)
            ref = _reference_trpo(pf, vf, tmp)
            cat._put_params(rec, case, "init", ref)
            names = [k for k, _ in ref.pf.named_parameters()]
            rec["%s|meta|names" % case] = np.array(names)
            nparam = sum(p.numel() for p in ref.pf.parameters())
            bs = batches(arch, n, B, seed, lead)
            for s in HVP_SEEDS:
                v = directions(nparam, s)
                rec["%s|hvp32|%d" % (case, s)] = _hvp(ref, bs[0]["obs"], bs[0]["acts"], v,
                                                      _dtype("float32")).astype(np.float32)
                rec["%s|hvp64|%d" % (case, s)] = _hvp(ref, bs[0]["obs"], bs[0]["acts"], v, _dtype("float64"))
            cg = ref.conjugate_gradient
            seen = {}

            def recording_cg(b):
                x = cg(b)
                if not seen:
                    seen["b"], seen["x"] = b.detach().numpy().copy(), x.detach().numpy().copy()
                return x
            ref.conjugate_gradient = recording_cg
            for u, b in enumerate(bs):
                with contextlib.redirect_stdout(io.StringIO()):              # the reference prints every backtrack
                    info = ref.update(b)
                for k, v in info.items():
                    rec["%s|info%d|%s" % (case, u, k)] = np.float64(v)
                for k, v in ref.pf.state_dict().items():
                    rec["%s|pf%d|pf.%s" % (case, u, k)] = v.detach().numpy().astype(np.float32)
            rec["%s|cg|b" % case] = seen["b"].astype(np.float32)
            rec["%s|cg|x" % case] = seen["x"].astype(np.float32)


def _dtype(name):
    import torch
    return getattr(torch, name)


def _record_kernels(rec):
    import torch
    from torch.distributions import Categorical

    class LogitTable(torch.nn.Module):
        """A policy whose parameters are the logits, looked up by the row index passed as the observation."""

        def __init__(self, table):
            super().__init__()
            self.table = torch.nn.Parameter(torch.as_tensor(table))

        def update(self, obs, actions):
            dis = Categorical(torch.softmax(self.table[obs.reshape(-1).long()], dim=-1))
            return {"dis": dis.probs, "log_prob": dis.log_prob(actions.reshape(-1)).unsqueeze(-1)}

    for case in KERNEL_CASES:
        z, t = kernel_inputs(case)
        with tempfile.TemporaryDirectory() as tmp:
            ref = _reference_trpo(LogitTable(z), LogitTable(z), tmp)
        ref.cg_damping = 0.0
        rows = np.arange(z.shape[0], dtype=np.float32).reshape(-1, 1)
        acts = np.zeros(z.shape[0], np.float32)
        for dt in ("float32", "float64"):
            rec["%s|hvp|%s" % (case, dt)] = _hvp(ref, rows, acts, t.reshape(-1), _dtype(dt)).reshape(z.shape).astype(dt)


def generate():
    from oracle import reference_loader
    reference_loader.load()
    rec = {}
    _record_updates(rec)
    _record_kernels(rec)
    return rec


def load(path=OUT):
    """{case: {what: {name: value}}} of a recorded file."""
    return cat.load(path)


if __name__ == "__main__":
    rec = generate()
    np.savez_compressed(OUT, **rec)
    print("%s: %d arrays, %d bytes" % (OUT, len(rec), os.path.getsize(OUT)))
