"""MountainCar-v0 and MountainCarContinuous-v0 without a GPU: the NumPy statement (oracle/mountain_car.py) against gym's
constants and steps derived by hand, the wall, the goals, NormAct's float32 rounding and the NumPy-1.x promotion of the
force, the time limits, the reset hash, the random-policy baselines, the scripted controller, the argument checks of
trl_mountain_car_step / trl_mountain_car_reset, the ops wrappers' operand checks and the env-id routing."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import mountain_car as M
from oracle import synth_env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V0, CONT = "MountainCar-v0", "MountainCarContinuous-v0"


def test_constants():
    assert (M.MIN_POSITION, M.MAX_POSITION, M.MAX_SPEED, M.GRAVITY, M.FORCE, M.POWER) == (-1.2, 0.6, 0.07, 0.0025,
                                                                                          0.001, 0.0015)
    assert M.SPECS == {V0: (0.5, 200, False), CONT: (0.45, 999, True)}
    src = open(os.path.join(ROOT, "torchrl_b200", "csrc", "mountain_car.cu")).read()
    for line in ("kCarMinPosition = -1.2;", "kCarMaxPosition = 0.6;", "kCarMaxSpeed = 0.07;", "kCarGoalV0 = 0.5;",
                 "kCarGoalCont = 0.45;", "kCarForce = 0.001;", "kCarGravity = 0.0025;", "kCarPower = 0.0015;"):
        assert line in src, line


def test_v0_step_derived_by_hand():
    phys = np.array([[-0.5, 0.0], [0.1, 0.02], [-0.3, -0.01]])
    nxt, term, base = M.dynamics(phys, [2.0, 1.0, 0.0], V0)
    v0 = 0.0 + (1.0 * 0.001 + math.cos(3 * -0.5) * (-0.0025))
    v1 = 0.02 + (0.0 * 0.001 + math.cos(3 * 0.1) * (-0.0025))
    v2 = -0.01 + (-1.0 * 0.001 + math.cos(3 * -0.3) * (-0.0025))
    np.testing.assert_allclose(nxt[:, 1], [v0, v1, v2], rtol=1e-15, atol=0)
    np.testing.assert_allclose(nxt[:, 0], [-0.5 + v0, 0.1 + v1, -0.3 + v2], rtol=1e-15, atol=0)
    assert not term.any() and base.tolist() == [-1.0] * 3
    _, obs, r, *_ = M.step(phys, [2.0, 1.0, 0.0], [0, 0, 0], V0, reward_scale=0.5)
    assert obs.dtype == np.float32 and obs.tolist() == np.float32(nxt).tolist() and r.tolist() == [-0.5] * 3


def test_continuous_step_derived_by_hand():
    phys = np.array([[-0.5, 0.0], [0.55, 0.07], [0.0, 0.0]])
    a = np.float32([0.3, 1.0, -2.0])
    nxt, term, base = M.dynamics(phys, a, CONT)
    u = M.norm_act(a)
    assert u[1] == 1.0 and u[2] == -1.0                                    # clipped by NormAct
    f = u.astype(np.float64)
    v0 = 0.0 + (f[0] * 0.0015 - 0.0025 * math.cos(3 * -0.5))
    v2 = 0.0 + (-1.0 * 0.0015 - 0.0025 * math.cos(0.0))
    assert nxt[[0, 2], 1].tolist() == [v0, v2] and nxt[[0, 2], 0].tolist() == [-0.5 + v0, v2]
    # 0.07 + 0.0015 - 0.0025 cos(1.65) > 0.07: both clips hold the car at the right end, past the goal
    assert nxt[1].tolist() == [0.6, 0.07] and term.tolist() == [False, True, False]
    assert base[1] == 100.0 - 1.0 * 0.1 and base[0] == -(f[0] * f[0]) * 0.1


def test_force_is_widened_before_the_power():
    """NumPy 1.x promotes float32 scalar * Python float to float64; NumPy 2 (NEP 50) would keep the product in float32.
    The oracle and the kernel follow NumPy 1.x: the float32 force meets the float64 power exactly widened."""
    a = np.float32([0.3, -0.7, 0.123])
    u = M.norm_act(a)
    nxt, _, _ = M.dynamics(np.array([[0.0, 0.0]] * 3), a, CONT)
    want = u.astype(np.float64) * 0.0015 - 0.0025 * 1.0
    assert nxt[:, 1].tolist() == want.tolist()
    nep50 = (u * np.float32(0.0015)).astype(np.float64) - 0.0025
    assert np.any(nxt[:, 1] != nep50)


def test_the_wall_zeroes_a_negative_velocity():
    for env_id, act in ((V0, 0.0), (CONT, -1.0)):
        nxt, term, _ = M.dynamics(np.array([[-1.19, -0.07], [-1.19, 0.01]]), [act, act], env_id)
        assert nxt[0].tolist() == [-1.2, 0.0]                             # clipped to the wall, stopped
        assert nxt[1, 0] > -1.2 and nxt[1, 1] != 0.0 and not term.any()


def test_goal_boundaries():
    assert M.terminal(np.array([[0.5, 0.0], [np.nextafter(0.5, 0), 0.0], [0.5, -1e-12]]), V0).tolist() == [True, False,
                                                                                                         False]
    assert M.terminal(np.array([[0.45, 0.0], [np.nextafter(0.45, 0), 0.01], [0.46, -1e-12]]), CONT).tolist() == [
        True, False, False]
    assert not M.terminal(np.array([[0.45, 0.0]]), V0)[0]
    # a step that lands on the right clip at 0.6 is done for both
    for env_id, act in ((V0, 2.0), (CONT, 1.0)):
        nxt, term, _ = M.dynamics(np.array([[0.59, 0.07]]), [act], env_id)
        assert nxt[0].tolist() == [0.6, 0.07] and term[0]


def test_normact_rounding():
    a = np.float32([-1.0, 1.0, 0.0, 0.5, -0.3, 0.1, 0.7, 1.5, -3.0])
    got = M.norm_act(a)
    f = np.float32
    want = [f(-1.0) + (f(x) + f(1.0)) * f(0.5) * (f(1.0) - f(-1.0)) for x in a]
    assert got.dtype == np.float32 and got.tolist() == np.clip(np.float32(want), -1, 1).tolist()
    assert got[:4].tolist() == [-1.0, 1.0, 0.0, 0.5] and got[7:].tolist() == [1.0, -1.0]
    small = np.float32([1e-3, -1e-5])
    assert np.all(M.norm_act(small) != small)                            # the affine map is not the identity in fp32


def test_invalid_v0_actions_raise():
    with pytest.raises(ValueError):
        M.dynamics(np.zeros((2, 2)), [0.0, 3.0], V0)


def test_time_limits():
    for env_id, limit in ((V0, 200), (CONT, 999)):
        phys = np.array([[-0.5, 0.0]] * 3)
        _, _, _, done, tl, el = M.step(phys, [1.0 if env_id == V0 else 0.0] * 3, [limit - 2, limit - 1, 0], env_id)
        assert done.tolist() == [False, True, False] and tl.tolist() == [False, True, False]
        assert el.tolist() == [limit - 1, limit, 1]


def test_reset_uses_the_synth_hash():
    seeds, eps = np.arange(6) * 5 + 1, np.arange(6)
    phys = M.reset_phys(seeds, eps)
    u = synth_env.hash_uniform(seeds.astype(np.uint64), eps.astype(np.uint64), np.uint64(0))
    assert phys[:, 0].tolist() == (-0.6 + 0.2 * u).tolist() and phys[:, 1].tolist() == [0.0] * 6
    big = M.reset_phys(np.arange(10000), np.zeros(10000))
    assert big[:, 0].min() >= -0.6 and big[:, 0].max() < -0.4


def test_random_policy_baselines():
    """A uniformly random policy never reaches either goal from the hash resets: v0 returns -200 (256 envs, seed 0, and
    1024 envs, seed 1); the continuous variant returns about -33.3 (0.1 E[a^2] = 1/30 per step for 999 steps)."""
    assert M.random_policy_return(V0) == -200.0
    r = M.random_policy_return(CONT)
    assert abs(r - (-33.3367190372268)) < 1e-6, r


@pytest.mark.parametrize("env_id", [V0, CONT])
def test_scripted_controller_reaches_the_goal(env_id):
    n = 4096
    ret, length, reached = M.episodes(lambda s: M.push(s, env_id), M.reset_phys(np.arange(n), np.arange(n) % 3),
                                      env_id)
    assert reached.all()
    assert (length.min(), length.max()) == ((113, 125) if env_id == V0 else (105, 111))
    if env_id == V0:
        np.testing.assert_array_equal(ret, -length.astype(np.float64))
    else:
        assert np.all(ret > 100.0 - 0.1 * length - 1e-3) and np.all(ret < 100.0)


# ------------------------------------------------------------------------------------------ C ABI
def _step(lib, N=4, max_steps=200, continuous=0, **null):
    names = ("phys", "obs", "actions", "elapsed", "reward", "done", "time_limit", "action_error")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_mountain_car_step(p["phys"], p["obs"], p["actions"], p["elapsed"], None, p["reward"], p["done"],
                                     p["time_limit"], p["action_error"], None, None, None, None, None, None, None,
                                     None, N, 1.0, max_steps, 1 << 30, 0, continuous, None)


def test_step_rejects_bad_arguments(native_lib):
    for kw in (dict(N=-1), dict(max_steps=0)):
        assert _step(native_lib, **kw) == -1, kw
        assert b"trl_mountain_car_step: bad sizes" in native_lib.trl_last_error()
    assert _step(native_lib, continuous=2) == -1
    assert b"continuous must be 0 or 1" in native_lib.trl_last_error()
    for n in ("phys", "obs", "actions", "elapsed", "reward", "done", "time_limit", "action_error"):
        assert _step(native_lib, **{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
    p = ctypes.c_void_p(16)
    assert native_lib.trl_mountain_car_step(p, p, p, p, None, p, p, p, p, p, None, None, None, None, None, None, None,
                                            4, 1.0, 200, 1 << 30, 0, 1, None) == -1
    assert b"ticket" in native_lib.trl_last_error()
    assert native_lib.trl_mountain_car_step(p, p, p, p, None, p, p, p, p, p, None, None, None, None, p, None, None, 4,
                                            1.0, 200, 1 << 30, 1, 0, None) == -1
    assert b"merge_stats" in native_lib.trl_last_error()
    assert native_lib.trl_mountain_car_step(p, p, p, p, None, p, p, p, p, None, None, None, None, None, None, None, p,
                                            4, 1.0, 200, 1 << 30, 0, 0, None) == -1
    assert b"any_reset" in native_lib.trl_last_error()
    assert _step(native_lib, N=0, phys=True) == 0


def _reset(lib, N=4, mask=None, step_count=None, next_norm=None, cur_ob=None, any_reset=None, t_ptr=None,
           norm_mean=None, norm_var=None, **null):
    names = ("phys", "obs", "elapsed", "episode", "seeds")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_mountain_car_reset(p["phys"], p["obs"], p["elapsed"], p["episode"], p["seeds"], mask, step_count,
                                      next_norm, cur_ob, any_reset, t_ptr, norm_mean, norm_var, N, 10.0, 1, None)


def test_reset_rejects_bad_arguments(native_lib):
    p = ctypes.c_void_p(16)
    assert _reset(native_lib, N=-1) == -1
    assert b"trl_mountain_car_reset: bad size" in native_lib.trl_last_error()
    for n in ("phys", "obs", "elapsed", "episode", "seeds"):
        assert _reset(native_lib, **{n: True}) == -1, n
        assert b"trl_mountain_car_reset: null pointer" in native_lib.trl_last_error()
    assert _reset(native_lib, mask=p, step_count=p) == -1
    assert b"not both" in native_lib.trl_last_error()
    for missing in ("step_count", "next_norm", "any_reset", "t_ptr"):
        kw = dict(step_count=p, next_norm=p, any_reset=p, t_ptr=p)
        kw[missing] = None
        assert _reset(native_lib, cur_ob=p, **kw) == -1, missing
        assert b"cur_ob needs" in native_lib.trl_last_error()
    assert _reset(native_lib, norm_mean=p) == -1
    assert b"norm_var" in native_lib.trl_last_error()
    assert _reset(native_lib, N=0, phys=True) == 0


def test_cta_count(native_lib):
    assert [native_lib.trl_mountain_car_num_ctas(n) for n in (1, 256, 257, 4099, 1 << 20)] == [1, 1, 2, 17, 4096]


def test_ops_wrappers_check_operands():
    import torch
    from torchrl_b200 import ops
    i32, u8, f64 = torch.int32, torch.uint8, torch.float64
    phys, obs = torch.zeros(4, 2, dtype=f64), torch.zeros(4, 2)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.mountain_car_step(phys, obs, torch.zeros(4), torch.zeros(4, dtype=i32), None, torch.zeros(4),
                              torch.zeros(4, dtype=u8), torch.zeros(4, dtype=u8), torch.zeros(1, dtype=i32), None,
                              None, None, None, None, torch.zeros(1, dtype=i32), torch.zeros(2, dtype=i32), None, 1.0,
                              200, 1000, False, True)
    with pytest.raises(ValueError, match="one action per env"):
        ops.mountain_car_step(phys, obs, torch.zeros(3), *([None] * 19))
    with pytest.raises(ValueError, match=r"\(N, 2\) and obs \(N, 2\)"):
        ops.mountain_car_step(torch.zeros(4, 3, dtype=f64), obs, torch.zeros(4), *([None] * 19))
    with pytest.raises(ValueError, match=r"\(N, 2\)"):
        ops.mountain_car_reset(phys, torch.zeros(4, 3), None, None, None)
    with pytest.raises(ValueError, match="not both"):
        ops.mountain_car_reset(phys, obs, None, None, None, mask=torch.zeros(4, dtype=u8),
                               step_count=torch.zeros(4, dtype=i32))
    with pytest.raises(ValueError, match="cur_ob needs"):
        ops.mountain_car_reset(phys, obs, None, None, None, step_count=torch.zeros(4, dtype=i32), cur_ob=obs)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.mountain_car_reset(phys, obs, torch.zeros(4, dtype=i32), torch.zeros(4, dtype=i32),
                               torch.zeros(4, dtype=i32))


def test_both_ids_are_routed():
    import importlib
    ge = importlib.import_module("torchrl_b200.env.get_env")
    from torchrl_b200.env import MountainCarVecEnv
    assert ge.is_mountain_car(V0) and ge.is_mountain_car(CONT) and not ge.is_mountain_car("MountainCar-v1")
    assert not MountainCarVecEnv.lockstep and MountainCarVecEnv.resets_itself and not MountainCarVecEnv._host_mirror_ok
    for other in ("MountainCar-v1", "MountainCarContinuous-v1", "mountaincar-v0"):
        with pytest.raises(NotImplementedError):
            ge.get_vec_env(other, {}, 2, device="cuda")
    import torch
    if not torch.cuda.is_available():
        for env_id in (V0, CONT):
            with pytest.raises((RuntimeError, AssertionError)):
                ge.get_vec_env(env_id, {}, 2)
