"""Discrete V-MPO without a GPU: the golden data against the executed reference, the fp64 NumPy restatement of the
selection rule and of the categorical V-MPO loss (oracle/make_golden_vmpo_categorical.py) against that data and
against torch autograd in the per-row KL mode, and the argument checks of the two entry points (csrc/categorical.cu)."""
import ctypes
import os

import numpy as np
import pytest

from oracle import make_golden_vmpo_categorical as G

KW = G.KW


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "vmpo_categorical_reference.npz")))


@pytest.mark.reference
def test_generator_reproduces_the_committed_golden_data(golden):
    fresh = G.generate()
    assert sorted(fresh) == sorted(golden)
    for k, v in fresh.items():
        assert v.dtype == golden[k].dtype and v.shape == golden[k].shape, k
        # the reference's CPU convolutions may round differently on another CPU: last-bit differences only
        np.testing.assert_allclose(v, golden[k], rtol=1e-6, atol=1e-7, err_msg=k)


def _inputs(golden, case):
    z, zq, acts, adv = G.loss_inputs(case)
    advn = golden["%s|input|advn" % case].reshape(-1)
    mean, std = golden["%s|input|stats" % case]
    np.testing.assert_array_equal(G.normalise(adv.reshape(-1), mean, std), advn)
    return z, zq, acts, advn


def _close(got, want, rtol, atol, what):
    if np.isnan(want):
        assert np.isnan(got), what
    elif np.isinf(want):
        assert got == want, (what, got, want)
    else:
        assert abs(got - want) <= rtol * abs(want) + atol, (what, got, want)


@pytest.mark.parametrize("case", ["loss", "loss_inf"])
def test_restatement_matches_the_reference_loss(golden, case):
    """Selection, logged scalars and gradients wrt the logits, eta and alpha of the reference's update_actor (summed
    KL).  The reference computes in float32, the restatement in fp64 from the same float32 inputs."""
    z, zq, acts, advn = _inputs(golden, case)
    sel = G.select(advn)
    k = G.LOSS_B - G.LOSS_B // 2
    assert sel.size == k
    # a tie straddles the boundary: its lower positions are kept
    order = np.argsort(-advn.astype(np.float64), kind="stable")
    tie = np.flatnonzero(advn == advn[order[k - 1]])
    kept = k - int((advn > advn[order[k - 1]]).sum())
    assert 0 < kept < tie.size
    assert np.isin(tie[:kept], sel).all() and not np.isin(tie[kept:], sel).any()
    # the reference's unstable sort keeps the same values, possibly other positions among the tied ones
    ref_rows = golden["%s|input|kept" % case]
    assert ref_rows.size == k
    np.testing.assert_array_equal(np.sort(advn[ref_rows]), np.sort(advn[sel]))
    assert set(ref_rows) ^ set(sel) <= set(tie)
    sel = np.sort(ref_rows)                         # the loss on the rows the reference kept
    eta, alpha = G.LOSS_DUAL
    info, gz, geta, galpha = G.vmpo_loss(z[sel], zq[sel], acts[sel], advn[sel], eta, alpha, KW["eta_eps"],
                                         KW["alpha_eps"])
    for key, v in info.items():
        _close(v, golden["%s|info|%s" % (case, key)], 1e-5, 1e-6, key)
    assert np.isnan(info["KL/std"])
    g = np.zeros_like(z, dtype=np.float64)
    g[sel] = gz
    want = golden["%s|grad|logits" % case]
    assert np.all(np.isfinite(want)) and np.all(want[np.setdiff1d(np.arange(G.LOSS_B), sel)] == 0)
    np.testing.assert_allclose(g, want, rtol=1e-4, atol=1e-7)
    _close(geta, float(golden["%s|grad|dual" % case][0]), 1e-5, 1e-6, "d eta")
    _close(galpha, float(golden["%s|grad|dual" % case][1]), 1e-5, 1e-6, "d alpha")
    if case == "loss_inf":
        assert info["KL/mean"] == np.inf and galpha == -np.inf
        assert np.isfinite(gz).all()


@pytest.mark.parametrize("case", ["loss", "loss_inf"])
def test_restatement_per_row_kl_matches_torch_autograd(golden, case):
    import torch
    from torch.distributions import Categorical, kl_divergence
    z, zq, acts, advn = _inputs(golden, case)
    sel = G.select(advn)
    eta, alpha = G.LOSS_DUAL
    info, gz, geta, galpha = G.vmpo_loss(z[sel], zq[sel], acts[sel], advn[sel], eta, alpha, KW["eta_eps"],
                                         KW["alpha_eps"], per_row_kl=True)
    zt = torch.tensor(z[sel], requires_grad=True)
    et = torch.tensor([eta], requires_grad=True)
    at = torch.tensor([alpha], requires_grad=True)
    adv = torch.as_tensor(advn[sel]).reshape(-1, 1)
    dis = Categorical(torch.softmax(zt, -1))
    tdis = Categorical(torch.softmax(torch.as_tensor(zq[sel]), -1))
    logp = dis.log_prob(torch.as_tensor(acts[sel])).unsqueeze(-1)
    kl = kl_divergence(dis, tdis).unsqueeze(-1)                     # one KL per row
    phi = torch.softmax(adv / et.detach(), dim=0)
    eta_loss = et * KW["eta_eps"] + et * torch.log(torch.mean(torch.exp(adv / et)))
    alpha_loss = at * KW["alpha_eps"] - at * kl.detach().mean()
    policy_loss = (-phi * logp + at.detach() * kl).mean()
    (policy_loss + eta_loss + alpha_loss).sum().backward()
    _close(info["Training/policy_loss"], policy_loss.item(), 1e-5, 1e-6, "policy_loss")
    _close(info["Training/alpha_loss"], alpha_loss.item(), 1e-5, 1e-6, "alpha_loss")
    _close(info["KL/mean"], kl.mean().item(), 1e-5, 1e-6, "KL/mean")
    if case == "loss":
        _close(info["KL/std"], kl.std().item(), 1e-4, 1e-6, "KL/std")
    np.testing.assert_allclose(gz, zt.grad.numpy(), rtol=1e-4, atol=1e-7)
    _close(geta, et.grad.item(), 1e-5, 1e-6, "d eta")
    _close(galpha, at.grad.item(), 1e-5, 1e-6, "d alpha")


def test_selection_rule_edges():
    assert G.select(np.array([3.0])).tolist() == [0]
    assert G.select(np.array([1.0, 2.0])).tolist() == [1]
    assert G.select(np.array([1.0, 1.0, 1.0])).tolist() == [0, 1]
    assert G.select(np.array([0.0, -0.0, 0.0, -0.0])).tolist() == [0, 1]
    assert G.select(np.array([5.0, 1.0, 5.0, 1.0, 1.0])).tolist() == [0, 1, 2]


def test_log_mean_exp_stays_finite_where_the_unshifted_form_overflows():
    z = np.zeros((3, 4), np.float32)
    info, gz, geta, galpha = G.vmpo_loss(z, z, np.zeros(3), np.array([100.0, 0.0, -1.0]), 1.0, 0.1, 0.02, 0.1)
    assert np.isfinite(geta) and np.isfinite(info["Training/policy_loss"])


def test_golden_agent_cases_are_complete(golden):
    for case, (arch, n, B, seed) in G.CASES.items():
        for u in range(n):
            assert np.isnan(golden["%s|info%d|KL/std" % (case, u)])          # the summed KL is one value
            assert golden["%s|info%d|KL/mean" % (case, u)] == golden["%s|info%d|KL/max" % (case, u)]
        assert golden["%s|final|dual" % case].shape == (2,)


# ------------------------------------------------------------------------------------------ argument checks
def _sel(lib, b=4, n=1, groups=1, advs=8, stats=8, sel=8):
    p = lambda v: ctypes.c_void_p(v) if v else None  # noqa: E731
    return lib.trl_vmpo_select(p(advs), None, groups, b, n, p(stats), p(sel), None)


def test_select_rejects_bad_arguments(native_lib):
    for kw in (dict(b=0), dict(n=0), dict(groups=0), dict(advs=0), dict(stats=0), dict(sel=0), dict(b=1 << 16, n=1 << 15)):
        assert _sel(native_lib, **kw) == -1, kw
        assert b"trl_vmpo_select" in native_lib.trl_last_error()


def _loss(lib, k=4, A=6, **null):
    names = ("logits", "target", "actions", "advs", "stats", "dual", "g_logits", "g_dual", "info", "scratch",
             "ticket")
    ptr = {n: (None if n in null else ctypes.c_void_p(8)) for n in names}
    return lib.trl_vmpo_categorical_loss(ptr["logits"], ptr["target"], ptr["actions"], ptr["advs"], ptr["stats"], None,
                                         ptr["dual"], k, A, 0.02, 0.1, 0, ptr["g_logits"], ptr["g_dual"], ptr["info"],
                                         ptr["scratch"], ptr["ticket"], None)


def test_loss_rejects_bad_arguments(native_lib):
    for kw in (dict(A=0), dict(A=33), dict(k=0), dict(k=-1)):
        assert _loss(native_lib, **kw) == -1, kw
        assert b"bad sizes" in native_lib.trl_last_error()
    for n in ("logits", "target", "actions", "advs", "stats", "dual", "g_logits", "g_dual", "info", "scratch",
              "ticket"):
        assert _loss(native_lib, **{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()


def test_scratch_size_query(native_lib):
    assert native_lib.trl_vmpo_categorical_scratch_doubles(1) == 10
    assert native_lib.trl_vmpo_categorical_scratch_doubles(257) == 20
