"""CPU checks of the categorical entry points: argument validation happens before any CUDA call (so a bad call
returns -1 with a message on a machine without a GPU), and the recorded reference data regenerates identically where
the reference is present."""
import os

import numpy as np
import pytest


def test_categorical_argument_errors_without_gpu(native_lib):
    lib = native_lib
    x = 16  # any non-null address: validation fails before it is touched
    for A in (0, 33):
        assert lib.trl_categorical_sample(x, x, 0, None, 4, A, x, None, None, None) == -1
        assert b"bad sizes" in lib.trl_last_error()
        assert lib.trl_categorical_log_prob(x, x, 4, A, x, None) == -1
        assert b"bad sizes" in lib.trl_last_error()
        assert lib.trl_ppo_categorical_actor_loss(x, x, None, x, None, None, 4, A, 0.2, 0.0, x, None, x, x, x,
                                                  None) == -1
        assert b"bad sizes" in lib.trl_last_error()
    assert lib.trl_categorical_sample(None, x, 0, None, 4, 6, x, None, None, None) == -1
    assert b"null" in lib.trl_last_error()
    assert lib.trl_categorical_sample(x, None, 0, None, 4, 6, x, None, None, None) == -1   # neither u nor counter
    assert b"null" in lib.trl_last_error()
    assert lib.trl_categorical_log_prob(x, None, 4, 6, x, None) == -1
    assert b"null" in lib.trl_last_error()
    assert lib.trl_ppo_categorical_actor_loss(x, x, None, x, None, None, 4, 6, 0.2, 0.0, None, None, x, x, x,
                                              None) == -1
    assert b"null" in lib.trl_last_error()
    assert lib.trl_ppo_categorical_actor_loss(x, x, None, x, None, None, 0, 6, 0.2, 0.0, x, None, x, x, x,
                                              None) == -1
    assert lib.trl_ppo_categorical_actor_scratch_doubles(1000) == 4 * 9
    assert lib.trl_categorical_log_prob(x, x, 0, 6, x, None) == 0               # empty batch: no-op


@pytest.mark.reference
def test_golden_categorical_regenerates_identically():
    from oracle import make_golden_categorical as gold
    rec = gold.record()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "categorical_reference.npz")
    with np.load(path) as z:
        assert sorted(z.files) == sorted(rec)
        for k in z.files:
            np.testing.assert_array_equal(z[k], rec[k], err_msg=k)
