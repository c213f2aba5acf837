"""Discrete TRPO without a GPU: the golden data against the executed reference and the fp64 restatement of its
Fisher-vector product, J^T (diag p - p p^T) J v * scale + damping * v (oracle/make_golden_trpo_categorical.py), in both
batch layouts, and the argument checks of the three TRPO entry points (csrc/categorical.cu)."""
import ctypes
import os

import numpy as np
import pytest

from oracle import make_golden_trpo_categorical as G


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "trpo_categorical_reference.npz")))


@pytest.mark.reference
def test_generator_reproduces_the_committed_golden_data(golden):
    fresh = G.generate()
    assert sorted(fresh) == sorted(golden)
    for k, v in fresh.items():
        assert v.dtype == golden[k].dtype and v.shape == golden[k].shape, k
        if v.dtype.kind == "U":
            assert (v == golden[k]).all(), k
        else:
            # the reference's CPU convolutions may round differently on another CPU: last-bit differences only
            np.testing.assert_allclose(v, golden[k], rtol=1e-5, atol=1e-7, err_msg=k)


def _logits_net(golden, case):
    """The policy of `case` at its initial weights as a networks.Net on the CPU (its forward is the logits)."""
    import torch
    import torchrl_b200.networks as networks
    from oracle import make_golden_categorical as cat
    arch, act, n, B, seed, lead = G.CASES[case]
    kw = cat.net_kwargs(networks, torch, arch)
    kw["activation_func"] = torch.nn.Tanh if act == "tanh" else torch.nn.ReLU
    net = networks.Net(output_shape=G.A, **kw)
    pre = "%s|init|pf." % case
    net.load_state_dict({k[len(pre):]: torch.as_tensor(v) for k, v in golden.items() if k.startswith(pre)})
    names = [n for n, _ in net.named_parameters()]
    assert names == list(golden["%s|meta|names" % case])
    return net


def _rel(got, want):
    return float(np.linalg.norm(np.asarray(got, np.float64) - want) / np.linalg.norm(want))


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_restated_fisher_product_matches_the_reference(golden, case):
    """Without the O(1e-8) terms of the reference's KL (DESIGN §6 deviation 20) the product matches the reference's
    double backward run in fp64 to 1e-6 and in fp32 to 1e-5, norm-wise: the omitted terms are below fp32 resolution."""
    arch, act, n, B, seed, lead = G.CASES[case]
    net = _logits_net(golden, case)
    obs = G.batches(arch, n, B, seed, lead)[0]["obs"]
    obs = obs.reshape((-1,) + obs.shape[len(lead or (B,)):])
    nparam = sum(p.numel() for p in net.parameters())
    for s in G.HVP_SEEDS:
        v = G.directions(nparam, s)
        mine = G.restated_hvp(net, obs, v, G.kl_scale(lead), G.KW["cg_damping"])
        assert _rel(mine, golden["%s|hvp64|%d" % (case, s)]) < 1e-6, (s, _rel(mine, golden["%s|hvp64|%d" % (case, s)]))
        assert _rel(mine, golden["%s|hvp32|%d" % (case, s)]) < 1e-5, (s, _rel(mine, golden["%s|hvp32|%d" % (case, s)]))
        # the damping alone would not pass: the Fisher term is a sizeable part of the product
        assert _rel(G.KW["cg_damping"] * v, golden["%s|hvp64|%d" % (case, s)]) > 1e-2


def test_kl_scale_of_both_layouts_matches_the_reference(golden):
    """The (T, N) whole-rollout batch: the reference's KL is N / A times the per-sample KL (trpo.py:59-61).  The
    per-sample restatement misses the recorded product by far; scaled by N / A it matches."""
    case = "trpo_mlp_tn"
    arch, act, n, B, seed, lead = G.CASES[case]
    assert G.kl_scale(lead) == lead[1] / G.A and G.kl_scale(None) == 1.0
    net = _logits_net(golden, case)
    obs = G.batches(arch, n, B, seed, lead)[0]["obs"].reshape(-1, 11)
    v = G.directions(sum(p.numel() for p in net.parameters()), 0)
    want = golden["%s|hvp64|0" % case]
    assert _rel(G.restated_hvp(net, obs, v, lead[1] / G.A, G.KW["cg_damping"]), want) < 1e-6
    assert _rel(G.restated_hvp(net, obs, v, 1.0, G.KW["cg_damping"]), want) > 1e-2


def _kernel_restatement(z, t):
    """(diag p - p p^T) t per row in fp64 from float32 logits."""
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(-1, keepdims=True))
    p = e / e.sum(-1, keepdims=True)
    t = np.asarray(t, np.float64)
    return p * t - p * (p * t).sum(-1, keepdims=True)


@pytest.mark.parametrize("case", sorted(G.KERNEL_CASES))
def test_logit_space_product_matches_the_reference(golden, case):
    """The kernel's formula on the kernel cases against the reference's double backward with the logits as the
    parameters (its KL is the mean over rows: scale 1 / M)."""
    z, t = G.kernel_inputs(case)
    mine = _kernel_restatement(z, t) / z.shape[0]
    want64, want32 = golden["%s|hvp|float64" % case], golden["%s|hvp|float32" % case]
    if case == "kern_a1":
        assert not mine.any() and not want64.any() and not want32.any()       # p = 1: no curvature
        return
    assert _rel(mine, want64) < 1e-6 and _rel(mine, want32) < 1e-5, (_rel(mine, want64), _rel(mine, want32))


def test_recorded_conjugate_gradient_is_complete(golden):
    """cg|b is the first update's -g and cg|x the reference's 10-iteration solve of F x = -g: one finite vector each
    in the policy's parameter space (the agent's solve is compared with it on the GPU)."""
    for case in G.CASES:
        b, x = golden["%s|cg|b" % case], golden["%s|cg|x" % case]
        assert b.shape == x.shape and np.linalg.norm(b) > 0 and np.all(np.isfinite(x))


def test_golden_cases_are_complete(golden):
    for case, (arch, act, n, B, seed, lead) in G.CASES.items():
        for u in range(n):
            info = {k.split("|", 2)[2] for k in golden if k.startswith("%s|info%d|" % (case, u))}
            assert info == {"advs/mean", "advs/std", "advs/max", "advs/min", "Training/policy_loss", "logprob/mean",
                            "logprob/std", "logprob/max", "logprob/min"}, info
        moved = max(float(np.abs(golden["%s|pf0|%s" % (case, k)] - golden["%s|init|%s" % (case, k)]).max())
                    for k in ("pf." + n for n in golden["%s|meta|names" % case]))
        assert moved > 1e-5, (case, moved)


# ------------------------------------------------------------------------------------------ argument checks
def _p(v):
    return ctypes.c_void_p(8) if v else None


def test_fisher_vp_rejects_bad_arguments(native_lib):
    def call(M=4, A=6, **null):
        return native_lib.trl_categorical_fisher_vp(_p("logits" not in null), _p("tangent" not in null), M, A, 1.0,
                                                    _p("g" not in null), None)
    for kw in (dict(A=0), dict(A=33), dict(M=-1)):
        assert call(**kw) == -1, kw
        assert b"bad sizes" in native_lib.trl_last_error()
    for n in ("logits", "tangent", "g"):
        assert call(**{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
    assert call(M=0) == 0                                      # nothing to do, nothing launched


def test_tangent_bias_act_rejects_bad_arguments(native_lib):
    def call(M=4, C=3, S=1, act=1, **null):
        return native_lib.trl_tangent_bias_act(_p("t" not in null), _p("db" not in null), _p("y" not in null), M, C,
                                               S, act, None)
    for kw in (dict(C=0), dict(S=0), dict(M=-1), dict(act=3), dict(act=-1)):
        assert call(**kw) == -1, kw
        assert b"bad sizes" in native_lib.trl_last_error()
    for n in ("t", "db"):
        assert call(**{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
    assert call(y=True, act=1) == -1 and call(y=True, act=2) == -1
    assert call(M=0, y=True, act=0) == 0                       # no activation: y is not read


def test_surrogate_rejects_bad_arguments(native_lib):
    names = ("logits", "actions", "logp_old", "advn", "out", "scratch", "ticket")

    def call(M=4, A=6, **null):
        ptr = {n: _p(n not in null) for n in names}
        return native_lib.trl_categorical_surrogate(ptr["logits"], ptr["actions"], ptr["logp_old"], ptr["advn"], M, A,
                                                    ptr["out"], ptr["scratch"], ptr["ticket"], None)
    for kw in (dict(A=0), dict(A=33), dict(M=0), dict(M=-1)):
        assert call(**kw) == -1, kw
        assert b"bad sizes" in native_lib.trl_last_error()
    for n in names:
        assert call(**{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()


def test_new_entry_points_are_exported(native_lib):
    from torchrl_b200 import ops
    for name in ("trl_categorical_fisher_vp", "trl_tangent_bias_act", "trl_categorical_surrogate"):
        assert hasattr(native_lib, name)
    for fn in ("categorical_fisher_vp", "tangent_bias_act", "categorical_surrogate"):
        assert callable(getattr(ops, fn))


def test_wrappers_refuse_cpu_tensors():
    import torch
    from torchrl_b200 import ops
    z = torch.zeros(4, 6)
    with pytest.raises(ValueError, match="CUDA"):
        ops.categorical_fisher_vp(z, z, 1.0, out=torch.zeros(4, 6))
    with pytest.raises(ValueError, match="CUDA"):
        ops.tangent_bias_act(z, torch.zeros(6), z, 1)
    with pytest.raises(ValueError, match="per channel"):
        ops.tangent_bias_act(z, torch.zeros(5), z, 1)


def test_unsupported_policies_are_rejected_without_a_gpu():
    import torch
    import torchrl_b200.networks as networks
    from torchrl_b200.algo.on_policy.trpo import layer_plan
    kw = dict(input_shape=(11,), hidden_shapes=[32, 32], base_type=networks.MLPBase, activation_func=torch.nn.Tanh)
    assert [type(l).__name__ for l, _ in layer_plan(networks.Net(output_shape=6, append_hidden_shapes=[16], **kw))] \
        == ["Linear"] * 4
    assert layer_plan(networks.Net(output_shape=6, add_ln=True, **kw)) is None
    kw["activation_func"] = torch.nn.ELU
    assert layer_plan(networks.Net(output_shape=6, **kw)) is None
