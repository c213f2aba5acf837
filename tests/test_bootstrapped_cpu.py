"""Bootstrapped DQN without a GPU: the golden data against the executed reference, the NumPy restatement of the loss
against that data, and the argument checks of the two entry points (csrc/bootstrapped.cu)."""
import ctypes

import numpy as np
import pytest

from oracle import make_golden_bootstrapped as G
from oracle import ref_bootstrapped as R


@pytest.fixture(scope="module")
def golden(golden_dir):
    import os
    return dict(np.load(os.path.join(golden_dir, "bootstrapped_dqn_reference.npz")))


@pytest.mark.reference
def test_generator_reproduces_the_committed_golden_data(golden):
    fresh = G.generate()
    assert sorted(fresh) == sorted(golden)
    for k, v in fresh.items():
        assert v.dtype == golden[k].dtype and v.shape == golden[k].shape, k
        np.testing.assert_array_equal(v, golden[k], err_msg=k)


def test_golden_batches_are_regenerated_from_their_seeds(golden):
    for name, (H, n, _, seed) in G.CASES.items():
        for u, b in enumerate(G.batches(H, n, seed)):
            for k, v in b.items():
                np.testing.assert_array_equal(golden["%s|batch%d|%s" % (name, u, k)], v)
            assert b["masks"][0].sum() == 0 and b["masks"][1].sum() == H and b["terminals"].any()


@pytest.mark.parametrize("case", sorted(G.CASES))
def test_numpy_restatement_matches_the_executed_reference(golden, case):
    """Loss, gradient wrt every head's outputs and the mean reward of every recorded update; the reference computes
    in float32, the restatement in fp64 on the same float32 network outputs."""
    H, n, _, _ = G.CASES[case]
    for u in range(n):
        g = lambda k: golden["%s|update%d|%s" % (case, u, k)]  # noqa: E731
        b = lambda k: golden["%s|batch%d|%s" % (case, u, k)]  # noqa: E731
        assert g("pred").shape == (H, G.B, G.A)
        loss, grad, info = R.bootstrapped_dqn_loss(g("pred"), g("next"), b("acts"), b("rewards"), b("terminals"),
                                                   b("masks"), G.GAMMA)
        np.testing.assert_allclose(loss, g("info")[0], rtol=1e-6)
        np.testing.assert_allclose(info[2], g("info")[1], rtol=0, atol=1e-7)
        np.testing.assert_allclose(grad, g("grad"), rtol=1e-5, atol=1e-8)
        assert np.all(grad[:, 0, :] == 0)                       # the all-zero mask row gets no gradient


def test_act_rule_draws_heads_only_at_episode_starts():
    rs = np.random.RandomState(0)
    H, N, A = 4, 9, 5
    q = rs.randn(H, N, A).astype(np.float32)
    q[:, 0, :] = 1.0                                            # ties: the lowest index wins
    step = np.array([0, 3, 0, 1, 0, 0, 7, 0, 2])
    old = np.full(N, 2, np.int32)
    u = np.array([0.0, 0.5, 0.999999, 0.3, 0.25, 1 - 2 ** -24, 0.7, 0.74999, 0.1], np.float32)
    um = rs.rand(N, H).astype(np.float32)
    head, act, mask = R.bootstrapped_act(q, step, old, u, um, 0.5)
    np.testing.assert_array_equal(head, [0, 2, 3, 2, 1, 3, 2, 2, 2])
    assert act[0] == 0
    np.testing.assert_array_equal(act, q[head, np.arange(N)].argmax(-1))
    np.testing.assert_array_equal(mask, (um < 0.5).astype(np.uint8))


def test_entry_points_reject_bad_arguments(native_lib):
    lib = native_lib
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def loss(B, H, A, ptr=p):
        return lib.trl_bootstrapped_dqn_loss(ptr, ptr, ptr, ptr, ptr, ptr, B, H, A, 0.99, ptr, ptr, ptr, ptr, None)

    for B, H, A in ((0, 1, 2), (-1, 1, 2), (4, 0, 2), (4, 1, 1)):
        assert loss(B, H, A) == -1 and b"bad sizes" in lib.trl_last_error()
    assert loss(4, 2, 2, ptr=None) == -1 and b"null" in lib.trl_last_error()

    def act(N, H, A, prob=0.5, u=p, um=p, ctr=None, ticket=None, q=p):
        return lib.trl_bootstrapped_act(q, p, p, p, p, p, u, um, 0, ctr, ticket, N, H, A, prob, None)

    for N, H, A in ((-1, 1, 2), (4, 0, 2), (4, 1, 0)):
        assert act(N, H, A) == -1 and b"bad sizes" in lib.trl_last_error()
    for prob in (-0.1, 1.5, float("nan")):
        assert act(4, 2, 2, prob=prob) == -1 and b"bernoulli_p" in lib.trl_last_error()
    assert act(4, 2, 2, q=None) == -1 and b"null" in lib.trl_last_error()
    assert act(4, 2, 2, um=None) == -1 and b"u_head and u_mask" in lib.trl_last_error()
    assert act(4, 2, 2, u=None, um=None) == -1 and b"rng_counter" in lib.trl_last_error()
    assert act(4, 2, 2, u=None, um=None, ctr=p) == -1 and b"rng_counter" in lib.trl_last_error()
    assert act(0, 2, 2) == 0                                    # no envs: nothing to launch
