"""CartPole without a GPU: the NumPy statement (oracle/cartpole.py) against gym's constants and a hand-derived step,
the time limits and rewards, the argument checks of trl_cartpole_step, and the env-id routing."""
import ctypes
import math

import numpy as np
import pytest

from oracle import cartpole as C
from oracle import synth_env


def test_constants_and_thresholds():
    assert (C.GRAVITY, C.MASS_CART, C.MASS_POLE, C.LENGTH, C.FORCE_MAG, C.TAU) == (9.8, 1.0, 0.1, 0.5, 10.0, 0.02)
    assert C.TOTAL_MASS == 1.1 and C.POLE_MASS_LENGTH == 0.05
    assert C.THETA_THRESHOLD == 0.20943951023931953 == 12 * 2 * math.pi / 360
    assert C.X_THRESHOLD == 2.4 and C.INIT_SCALE == 0.05
    assert C.MAX_EPISODE_STEPS == {"CartPole-v0": 200, "CartPole-v1": 500}


def test_the_kernel_states_the_same_constants():
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "torchrl_b200", "csrc",
                            "cartpole.cu")).read()
    for line in ("kGravity = 9.8;", "kMassCart = 1.0;", "kMassPole = 0.1;", "kLength = 0.5;", "kForceMag = 10.0;",
                 "kTau = 0.02;", "kXThreshold = 2.4;", "kFourThirds = 4.0 / 3.0;",
                 "kThetaThreshold = 12.0 * 2.0 * 3.141592653589793 / 360.0;"):
        assert line in src, line
    assert 12.0 * 2.0 * 3.141592653589793 / 360.0 == C.THETA_THRESHOLD


def test_one_step_from_the_zero_state():
    s = np.zeros((2, 4), np.float32)
    n64 = C.dynamics64(s, [1, 0])
    assert n64[0].tolist() == [0.0, 0.1951219512195122, 0.0, -0.2926829268292683]
    assert n64[1].tolist() == [0.0, -0.1951219512195122, 0.0, 0.2926829268292683]
    n32, done = C.dynamics(s, [1, 0])
    np.testing.assert_array_equal(n32, n64.astype(np.float32))
    assert not done.any()


def test_termination_thresholds_are_strict():
    f = np.float32
    x = f(C.X_THRESHOLD)
    th = f(C.THETA_THRESHOLD)
    up = lambda v: np.nextafter(v, f(np.inf))         # noqa: E731
    down = lambda v: np.nextafter(v, f(-np.inf))      # noqa: E731
    # fp32(2.4) lies above 2.4: it already terminates; the fp32 value below does not
    states = np.array([[x, 0, 0, 0], [down(x), 0, 0, 0], [-x, 0, 0, 0], [0, 0, th, 0], [0, 0, down(th), 0],
                       [0, 0, -up(th), 0]], np.float32)
    assert float(x) > 2.4 and float(down(x)) < 2.4
    assert float(th) > C.THETA_THRESHOLD and float(down(th)) < C.THETA_THRESHOLD
    assert C.terminated(states).tolist() == [True, False, True, True, False, True]


@pytest.mark.parametrize("env_id", ["CartPole-v0", "CartPole-v1"])
def test_time_limits_and_rewards(env_id):
    limit = C.MAX_EPISODE_STEPS[env_id]
    s = np.zeros((3, 4), np.float32)
    s[2, 0] = 2.39                                      # pushed out by this step
    s[2, 1] = 1.0
    el = np.array([limit - 1, limit - 2, limit - 1])
    nxt, r, done, tl, el2 = C.step(s, [1, 0, 1], el, limit, reward_scale=0.5)
    assert done.tolist() == [True, False, True] and tl.tolist() == [True, False, True]
    assert r.tolist() == [0.5, 0.5, 0.5] and el2.tolist() == [limit, limit - 1, limit]
    _, r, done, tl, _ = C.step(s, [1, 0, 1], [0, 0, 0], limit)
    assert done.tolist() == [False, False, True] and not tl.any()
    assert r.tolist() == [1.0, 1.0, 1.0]                # the terminating step is rewarded too


def test_reset_uses_the_synth_hash():
    seeds, eps = np.arange(5) * 7 + 3, np.arange(5)
    s = C.reset_state(seeds, eps)
    want = (0.05 / synth_env.INIT_SCALE) * synth_env.reset_state(seeds, eps, 4)
    np.testing.assert_allclose(s, want.astype(np.float32), rtol=1e-6)
    assert s.dtype == np.float32 and np.abs(s).max() <= 0.05


def _step(lib, N=4, max_steps=500, **null):
    names = ("state", "actions", "elapsed", "reward", "done", "time_limit", "action_error")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_cartpole_step(p["state"], p["actions"], p["elapsed"], None, p["reward"], p["done"], p["time_limit"],
                                 p["action_error"], None, None, None, None, None, None, None, None, N, 1.0, max_steps,
                                 1 << 30, 0, None)


def test_step_rejects_bad_arguments(native_lib):
    for kw in (dict(N=-1), dict(max_steps=0)):
        assert _step(native_lib, **kw) == -1, kw
        assert b"trl_cartpole_step: bad sizes" in native_lib.trl_last_error()
    for n in ("state", "actions", "elapsed", "reward", "done", "time_limit", "action_error"):
        assert _step(native_lib, **{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
    p = ctypes.c_void_p(16)
    assert native_lib.trl_cartpole_step(p, p, p, None, p, p, p, p, p, None, None, None, None, None, None, None, 4, 1.0,
                                        500, 1 << 30, 0, None) == -1
    assert b"ticket" in native_lib.trl_last_error()
    assert native_lib.trl_cartpole_step(p, p, p, None, p, p, p, p, p, None, None, None, None, p, None, None, 4, 1.0,
                                        500, 1 << 30, 1, None) == -1
    assert b"merge_stats" in native_lib.trl_last_error()
    assert native_lib.trl_cartpole_step(p, p, p, None, p, p, p, p, None, None, None, None, None, None, None, p, 4, 1.0,
                                        500, 1 << 30, 0, None) == -1
    assert b"any_reset" in native_lib.trl_last_error()
    assert _step(native_lib, N=0, state=True) == 0          # nothing to do: no pointer is read


def test_cta_count(native_lib):
    assert [native_lib.trl_cartpole_num_ctas(n) for n in (1, 256, 257, 4099)] == [1, 1, 2, 17]


def test_ops_wrapper_checks_operands():
    import torch
    from torchrl_b200 import ops
    s = torch.zeros(4, 4)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.cartpole_step(s, torch.zeros(4), torch.zeros(4, dtype=torch.int32), None, torch.zeros(4),
                          torch.zeros(4, dtype=torch.uint8), torch.zeros(4, dtype=torch.uint8),
                          torch.zeros(1, dtype=torch.int32), None, None, None, None, None,
                          torch.zeros(1, dtype=torch.int32), torch.zeros(2, dtype=torch.int32), None, 1.0, 500, 1000,
                          False)
    with pytest.raises(ValueError, match="one action per env"):
        ops.cartpole_step(s, torch.zeros(3), *([None] * 18))


def test_cartpole_ids_are_routed_to_the_device_env():
    import importlib
    ge = importlib.import_module("torchrl_b200.env.get_env")
    assert ge.is_cartpole("CartPole-v0") and ge.is_cartpole("CartPole-v1") and not ge.is_cartpole("CartPole-v2")
    with pytest.raises(NotImplementedError):
        ge.get_vec_env("Pendulum-v0", {}, 2, device="cuda")
