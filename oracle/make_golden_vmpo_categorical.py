"""Golden data of discrete V-MPO, tests/test_vmpo_categorical_*.py: the unmodified reference executed on torch CPU
behind oracle/shims, recorded so that the device kernels and the agent can be checked on a machine without a copy of
the reference.  Also the fp64 NumPy restatement of the selection rule and of the categorical V-MPO loss that the tests
compare both the recording and the kernels against.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/reference_loader.available()):

    python oracle/make_golden_vmpo_categorical.py      # -> tests/golden/vmpo_categorical_reference.npz

Recorded, keys "<case>|<what>|<name>":
  * "vmpo_mlp", "vmpo_cnn": the reference's VMPO.update with a CategoricalDisPolicy on the MLP (O = 11, A = 6) and the
    small CNN of make_golden_categorical (its nets and batch helpers): the initial state_dicts, every update's infos
    (NaN kept, e.g. KL/std), the final state_dicts and the final eta and alpha;
  * "loss", "loss_inf": the reference's VMPO.update_actor on a table of seeded logits (a policy whose update() looks
    its rows up by index): a third of the rows saturated (the probability clamp is active), ties of the normalised
    advantage across the selection boundary, and in "loss_inf" a selected target row with an exactly-zero probability
    (its KL is inf) and a policy row with one.  The logged infos and the autograd gradients wrt the logits, eta and
    alpha (the policy's gradient clip is bypassed for this recording, so the raw gradient is kept), and the rows the
    reference kept: its torch.sort is not stable, so among values tied at the boundary it may keep other positions
    than the lowest ones (DESIGN §6 deviation 19).
Inputs are regenerated from their seeds (`batches`, `loss_inputs`).
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "vmpo_categorical_reference.npz")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_golden_categorical as cat  # noqa: E402

A = cat.A
KW = dict(plr=1e-3, vlr=1e-3, opt_epochs=1, eta_eps=0.02, alpha_eps=0.1)
# case -> (architecture, number of batches, batch rows, batch seed)
CASES = {"vmpo_mlp": ("mlp", 4, 64, 20), "vmpo_cnn": ("cnn", 2, 32, 21)}
LOSS_B = 37                                  # k = 19
LOSS_DUAL = (0.7, 0.3)                       # eta, alpha of the loss cases


def batches(arch, n, B, seed):
    return cat.batches(arch, n, B, seed)


def loss_inputs(case):
    """(logits, target logits, actions, raw advantages) of a loss case, B = LOSS_B rows."""
    rs = np.random.RandomState(5 if case == "loss" else 6)
    B = LOSS_B
    z = rs.randn(B, A).astype(np.float32) * 2.0
    sat = np.arange(B) % 3 == 0
    z[sat] = (rs.randn(int(sat.sum()), A) * 12.0).astype(np.float32)
    z[sat, rs.randint(0, A, int(sat.sum()))] += 20.0
    zq = (z + rs.randn(B, A).astype(np.float32) * 0.5).astype(np.float32)
    acts = rs.randint(0, A, B).astype(np.float32)
    adv = np.round(rs.randn(B) * 4.0) / 4.0                 # quarter steps: many equal values
    k = B - B // 2
    order = np.argsort(-adv, kind="stable")
    adv[order[k - 2:k + 2]] = adv[order[k - 2]]             # a tie of four across the boundary (two kept)
    if case == "loss_inf":
        top = order[0]                                      # selected: its target has q_2 == 0, p_2 > 0
        zq[top] = z[top]
        zq[top, 2] -= 200.0
        z[order[1], 4] -= 200.0                             # selected: p_4 == 0
    return z, zq, acts, adv.astype(np.float32).reshape(B, 1)


# ------------------------------------------------------------------------------------------ fp64 restatement
def normalise(adv, mean, std):
    """(adv - mean) / (std + 1e-5) in float32, as the reference and the kernels compute it."""
    adv = np.asarray(adv, np.float32)
    return (adv - np.float32(mean)) / (np.float32(std) + np.float32(1e-5))


def select(advn):
    """Positions of the k = B - B // 2 largest values, ties to the lower position, in ascending order."""
    advn = np.asarray(advn).reshape(-1)
    B = advn.size
    order = np.argsort(-advn.astype(np.float64), kind="stable")
    return np.sort(order[:B - B // 2])


def _cat(z):
    """p, l = log(clamp(p, eps, 1 - eps)), the clamp mask of Categorical(softmax(z)), in fp64 from float32 logits."""
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(-1, keepdims=True))
    p = e / e.sum(-1, keepdims=True)
    eps = float(np.finfo(np.float32).eps)
    return p, np.log(np.clip(p, eps, 1 - eps)), ((p >= eps) & (p <= 1 - eps)).astype(np.float64)


def vmpo_loss(z, zq, acts, advn, eta, alpha, eta_eps, alpha_eps, per_row_kl=False):
    """The categorical V-MPO actor loss on the k selected rows: (info dict, dL/dz (k, A), dL/deta, dL/dalpha).
    Zero probabilities are decided on float32 softmax values, as torch decides them."""
    z32, zq32 = np.asarray(z, np.float32), np.asarray(zq, np.float32)
    k = z32.shape[0]
    p, l, m = _cat(z32)
    q, lq, _ = _cat(zq32)
    pz = _softmax32(z32) == 0
    qz = _softmax32(zq32) == 0
    a = np.asarray(acts).reshape(-1).astype(np.int64)
    advn32 = np.asarray(advn, np.float32).reshape(-1)
    x = (advn32 / np.float32(eta)).astype(np.float64)                  # float32, as torch and the kernel divide
    advn = advn32.astype(np.float64)
    mx = x.max()
    e = np.exp(x - mx)
    phi = e / e.sum()
    lme = mx + np.log(e.mean())
    rows = np.arange(k)
    logp = l[rows, a]
    live = ~pz & ~qz
    kl_t = np.where(live, p * (l - lq), 0.0)
    kl = np.where((qz & ~pz).any(-1), np.inf, kl_t.sum(-1))
    K = kl.mean() if per_row_kl else kl.sum()
    c = alpha / k if per_row_kl else alpha
    g = np.where(live, l - lq + m, 0.0)
    dkl = p * (g - (p * g).sum(-1, keepdims=True))
    onehot = np.eye(z32.shape[1])[a]
    dlogp = m[rows, a][:, None] * (onehot - p)
    gz = -(phi / k)[:, None] * dlogp + c * dkl
    with np.errstate(invalid="ignore"):
        info = {"Training/policy_loss": float(np.mean(-phi * logp) + alpha * K),
                "Training/alpha_loss": float(alpha * alpha_eps - alpha * K)}
        info.update(_four("logprob", logp))
        info.update(_four("KL", kl if per_row_kl else np.array([K])))
    return info, gz, float(eta_eps + lme - (phi * advn).sum() / eta), float(alpha_eps - K)


def _softmax32(z32):
    import torch
    return torch.softmax(torch.as_tensor(z32), dim=-1).numpy()


def _four(prefix, v):
    v = np.asarray(v, np.float64)
    std = float(np.std(v, ddof=1)) if v.size > 1 else float("nan")
    if not np.all(np.isfinite(v)):
        std = float("nan")
    return {prefix + "/mean": float(v.mean()), prefix + "/std": std, prefix + "/max": float(v.max()),
            prefix + "/min": float(v.min())}


# ------------------------------------------------------------------------------------------ the executed reference
def _reference_vmpo(pf, vf, save_dir):
    import gym
    from torchrl.algo import VMPO

    class Env:
        action_space = gym.spaces.Discrete(A)
        observation_space = gym.spaces.Box(-np.ones(cat.MLP["obs"]), np.ones(cat.MLP["obs"]))
    return VMPO(pf=pf, vf=vf, env=Env(), replay_buffer=None, collector=cat._Col(), logger=cat._NullLogger(),
                discount=0.99, num_epochs=10, batch_size=64, gae=True, device="cpu", save_dir=save_dir, shuffle=True,
                tau=0.95, **KW)


def _record_updates(rec):
    for case, (arch, n, B, seed) in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            pf, vf = cat._reference_nets(arch)
            ref = _reference_vmpo(pf, vf, tmp)
            cat._put_params(rec, case, "init", ref)
            for u, b in enumerate(batches(arch, n, B, seed)):
                for k, v in ref.update(b).items():
                    rec["%s|info%d|%s" % (case, u, k)] = np.float64(v)
            cat._put_params(rec, case, "final", ref)
            rec["%s|final|dual" % case] = np.array([ref.eta.item(), ref.alpha.item()], np.float32)


def _record_loss(rec, case):
    import torch
    from torch.distributions import Categorical
    z, zq, acts, adv = loss_inputs(case)

    class LogitTable(torch.nn.Module):
        """A policy whose rows are free logits, looked up by the row index passed as the observation."""

        def __init__(self, table):
            super().__init__()
            self.table = torch.nn.Parameter(torch.as_tensor(table))
            self.rows = None

        def update(self, obs, actions):
            self.rows = obs.reshape(-1).long().numpy().copy()       # the rows the reference kept, in its order
            dis = Categorical(torch.softmax(self.table[obs.reshape(-1).long()], dim=-1))
            return {"dis": dis, "log_prob": dis.log_prob(actions).unsqueeze(-1)}

    with tempfile.TemporaryDirectory() as tmp:
        ref = _reference_vmpo(LogitTable(z), LogitTable(z), tmp)
    with torch.no_grad():
        ref.target_pf.table.copy_(torch.as_tensor(zq))
        ref.eta.fill_(LOSS_DUAL[0])
        ref.alpha.fill_(LOSS_DUAL[1])
    advs = torch.as_tensor(adv)
    advn = (advs - advs.mean()) / (advs.std() + 1e-5)          # VMPO.update's normalisation
    info = {}
    clip = torch.nn.utils.clip_grad_norm_
    torch.nn.utils.clip_grad_norm_ = lambda params, max_norm, *a, **kw: clip(params, float("inf"))
    try:
        ref.update_actor(info, torch.arange(LOSS_B, dtype=torch.float32).reshape(-1, 1), torch.as_tensor(acts), advn)
    finally:
        torch.nn.utils.clip_grad_norm_ = clip
    for k, v in info.items():
        if k not in ("Training/alpha", "Training/eta"):
            rec["%s|info|%s" % (case, k)] = np.float64(v)
    rec["%s|grad|logits" % case] = ref.pf.table.grad.numpy().astype(np.float32)
    rec["%s|grad|dual" % case] = np.array([ref.eta.grad.item(), ref.alpha.grad.item()], np.float32)
    rec["%s|input|advn" % case] = advn.numpy().astype(np.float32)
    rec["%s|input|kept" % case] = ref.pf.rows.astype(np.int64)
    rec["%s|input|stats" % case] = np.array([advs.mean().item(), advs.std().item()], np.float32)


def generate():
    from oracle import reference_loader
    reference_loader.load()
    rec = {}
    _record_updates(rec)
    for case in ("loss", "loss_inf"):
        _record_loss(rec, case)
    return rec


def load(path=OUT):
    """{case: {what: {name: value}}} of a recorded file."""
    return cat.load(path)


if __name__ == "__main__":
    rec = generate()
    np.savez_compressed(OUT, **rec)
    print("%s: %d arrays, %d bytes" % (OUT, len(rec), os.path.getsize(OUT)))
