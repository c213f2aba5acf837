"""Pendulum-v1 without a GPU: the NumPy statement (oracle/pendulum.py) against gym's constants and hand-derived steps,
the v1 order of the velocity clip, angle_normalize, NormAct's float32 rounding, the time limit, the argument checks of
trl_pendulum_step / trl_pendulum_reset, the env-id routing and the random-policy baseline of the learning tests."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import pendulum as P
from oracle import synth_env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_constants():
    assert (P.G, P.M, P.L, P.DT, P.MAX_SPEED, P.MAX_TORQUE) == (10.0, 1.0, 1.0, 0.05, 8.0, 2.0)
    assert P.MAX_EPISODE_STEPS == 200 and P.ENV_ID == "Pendulum-v1"
    src = open(os.path.join(ROOT, "torchrl_b200", "csrc", "pendulum.cu")).read()
    for line in ("kPendG = 10.0;", "kPendM = 1.0;", "kPendL = 1.0;", "kPendDt = 0.05;", "kPendMaxSpeed = 8.0;",
                 "kPendMaxTorque = 2.0f;", "kPi = 3.141592653589793;"):
        assert line in src, line
    assert 3.141592653589793 == math.pi


def test_one_step_derived_by_hand():
    phys = np.array([[0.0, 0.0], [math.pi / 2, 1.0], [0.0, 0.0]])
    nxt, cost = P.dynamics(phys, [1.0, 0.0, -1.0])
    # th = 0, thdot = 0, u = 2: newthdot = (15 * 0 + 3 * 2) * 0.05, newth = newthdot * 0.05, cost = 0.001 * 4
    assert nxt[0].tolist() == [0.30000000000000004 * 0.05, 6.0 * 0.05] and cost[0] == 0.001 * (2.0 * 2.0)
    # th = pi/2, thdot = 1, u = 0: newthdot = 1 + 15 * sin(pi/2) * 0.05 = 1.75; cost = (pi/2)^2 + 0.1
    assert nxt[1, 1] == 1.75 and nxt[1, 0] == math.pi / 2 + 1.75 * 0.05
    assert cost[1] == (math.pi / 2) ** 2 + 0.1 * 1.0 + 0.0
    assert nxt[2].tolist() == [-0.015000000000000003, -0.30000000000000004]
    obs = P.observe(nxt)
    assert obs.dtype == np.float32 and obs[0].tolist() == np.float32([math.cos(0.015000000000000003),
                                                                     math.sin(0.015000000000000003),
                                                                     0.30000000000000004]).tolist()
    _, _, r, _, _, _ = P.step(phys, [1.0, 0.0, -1.0], [0, 0, 0], reward_scale=0.5)
    assert r.dtype == np.float32 and r.tolist() == np.float32(-cost * 0.5).tolist()


def test_v1_moves_the_angle_with_the_clipped_velocity():
    # |thdot| near 8 and a torque pushing it past: the clipped 8 moves the angle, not the unclipped 8.2 (v0's order)
    phys = np.array([[0.3, 7.9], [-0.3, -7.95]])
    nxt, _ = P.dynamics(phys, [1.0, -1.0])
    unclipped = 7.9 + (15.0 * math.sin(0.3) + 3.0 * 2.0) * 0.05
    assert unclipped > 8.0
    assert nxt[0].tolist() == [0.3 + 8.0 * 0.05, 8.0]
    assert nxt[1].tolist() == [-0.3 - 8.0 * 0.05, -8.0]
    assert nxt[0, 0] != 0.3 + unclipped * 0.05


def test_angle_normalize():
    pi = math.pi
    xs = [pi, -pi, 0.0, 2 * pi, -2 * pi, 4 * pi, -6 * pi, 3 * pi, 0.5, -0.5, 7.0, -7.0]
    got = P.angle_normalize(xs).tolist()
    want = [((x + pi) % (2 * pi)) - pi for x in xs]          # Python's float %
    assert got == want
    assert got[:6] == [-pi, -pi, 0.0, 0.0, 0.0, 0.0]
    assert all(-pi <= g < pi for g in got)


def test_normact_rounding():
    a = np.float32([-1.0, 1.0, 0.0, 0.5, -0.3, 0.1, 0.7, 1.5, -3.0])
    got = P.torque(a)
    assert got.dtype == np.float32
    f = np.float32
    want = [f(-2.0) + (f(x) + f(1.0)) * f(0.5) * (f(2.0) - f(-2.0)) for x in a]
    assert got.tolist() == np.clip(np.float32(want), -2, 2).tolist()
    assert got[:4].tolist() == [-2.0, 2.0, 0.0, 1.0]
    assert got[4] == np.float32(-0.6000000238418579) and got[5] == np.float32(0.20000004768371582)
    assert got[7:].tolist() == [2.0, -2.0]                   # NormAct clips actions outside [-1, 1]


def test_time_limit():
    phys = np.zeros((3, 2))
    _, _, _, done, tl, el = P.step(phys, [0.0, 0.0, 0.0], [198, 199, 0])
    assert done.tolist() == [False, True, False] and tl.tolist() == [False, True, False]
    assert el.tolist() == [199, 200, 1]
    _, _, _, done, tl, _ = P.step(phys, [0.0] * 3, [200, 10, 0], max_episode_steps=11)
    assert done.tolist() == [True, True, False] and tl.tolist() == [False, True, False]


def test_reset_uses_the_synth_hash():
    seeds, eps = np.arange(6) * 5 + 1, np.arange(6)
    phys = P.reset_phys(seeds, eps)
    u0 = synth_env.hash_uniform(seeds.astype(np.uint64), eps.astype(np.uint64), np.uint64(0))
    u1 = synth_env.hash_uniform(seeds.astype(np.uint64), eps.astype(np.uint64), np.uint64(1))
    assert phys[:, 0].tolist() == (math.pi * (2.0 * u0 - 1.0)).tolist()
    assert phys[:, 1].tolist() == (2.0 * u1 - 1.0).tolist()
    assert np.abs(phys[:, 0]).max() <= math.pi and np.abs(phys[:, 1]).max() <= 1.0


def test_random_policy_baseline():
    """A uniformly random policy from the hash resets returns about -1230 per 200-step episode (256 and 1024 envs,
    two seeds: -1230.2 and -1229.7).  The learning tests' thresholds sit far above it."""
    r = P.random_policy_return()
    assert -1300 < r < -1150, r
    assert abs(r - (-1230.24)) < 0.01


# ------------------------------------------------------------------------------------------ C ABI
def _step(lib, N=4, max_steps=200, **null):
    names = ("phys", "obs", "actions", "elapsed", "reward", "done", "time_limit", "action_error")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_pendulum_step(p["phys"], p["obs"], p["actions"], p["elapsed"], None, p["reward"], p["done"],
                                 p["time_limit"], p["action_error"], None, None, None, None, None, None, None, None,
                                 N, 1.0, max_steps, 1 << 30, 0, None)


def test_step_rejects_bad_arguments(native_lib):
    for kw in (dict(N=-1), dict(max_steps=0)):
        assert _step(native_lib, **kw) == -1, kw
        assert b"trl_pendulum_step: bad sizes" in native_lib.trl_last_error()
    for n in ("phys", "obs", "actions", "elapsed", "reward", "done", "time_limit", "action_error"):
        assert _step(native_lib, **{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
    p = ctypes.c_void_p(16)
    assert native_lib.trl_pendulum_step(p, p, p, p, None, p, p, p, p, p, None, None, None, None, None, None, None, 4,
                                        1.0, 200, 1 << 30, 0, None) == -1
    assert b"ticket" in native_lib.trl_last_error()
    assert native_lib.trl_pendulum_step(p, p, p, p, None, p, p, p, p, p, None, None, None, None, p, None, None, 4,
                                        1.0, 200, 1 << 30, 1, None) == -1
    assert b"merge_stats" in native_lib.trl_last_error()
    assert native_lib.trl_pendulum_step(p, p, p, p, None, p, p, p, p, None, None, None, None, None, None, None, p, 4,
                                        1.0, 200, 1 << 30, 0, None) == -1
    assert b"any_reset" in native_lib.trl_last_error()
    assert _step(native_lib, N=0, phys=True) == 0           # nothing to do: no pointer is read


def _reset(lib, N=4, mask=None, step_count=None, next_norm=None, cur_ob=None, any_reset=None, t_ptr=None,
           norm_mean=None, norm_var=None, **null):
    names = ("phys", "obs", "elapsed", "episode", "seeds")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_pendulum_reset(p["phys"], p["obs"], p["elapsed"], p["episode"], p["seeds"], mask, step_count,
                                  next_norm, cur_ob, any_reset, t_ptr, norm_mean, norm_var, N, 10.0, 1, None)


def test_reset_rejects_bad_arguments(native_lib):
    p = ctypes.c_void_p(16)
    assert _reset(native_lib, N=-1) == -1
    assert b"trl_pendulum_reset: bad size" in native_lib.trl_last_error()
    for n in ("phys", "obs", "elapsed", "episode", "seeds"):
        assert _reset(native_lib, **{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
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
    assert [native_lib.trl_pendulum_num_ctas(n) for n in (1, 256, 257, 4099, 1 << 20)] == [1, 1, 2, 17, 4096]


def test_ops_wrappers_check_operands():
    import torch
    from torchrl_b200 import ops
    i32, u8, f64 = torch.int32, torch.uint8, torch.float64
    phys, obs = torch.zeros(4, 2, dtype=f64), torch.zeros(4, 3)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.pendulum_step(phys, obs, torch.zeros(4), torch.zeros(4, dtype=i32), None, torch.zeros(4),
                          torch.zeros(4, dtype=u8), torch.zeros(4, dtype=u8), torch.zeros(1, dtype=i32), None, None,
                          None, None, None, torch.zeros(1, dtype=i32), torch.zeros(2, dtype=i32), None, 1.0, 200,
                          1000, False)
    with pytest.raises(ValueError, match="one action per env"):
        ops.pendulum_step(phys, obs, torch.zeros(3), *([None] * 18))
    with pytest.raises(ValueError, match=r"\(N, 2\)"):
        ops.pendulum_step(torch.zeros(4, 3, dtype=f64), obs, torch.zeros(4), *([None] * 18))
    with pytest.raises(ValueError, match=r"\(N, 2\)"):
        ops.pendulum_reset(phys, torch.zeros(4, 4), None, None, None)
    with pytest.raises(ValueError, match="not both"):
        ops.pendulum_reset(phys, obs, None, None, None, mask=torch.zeros(4, dtype=u8),
                           step_count=torch.zeros(4, dtype=i32))
    with pytest.raises(ValueError, match="cur_ob needs"):
        ops.pendulum_reset(phys, obs, None, None, None, step_count=torch.zeros(4, dtype=i32), cur_ob=obs)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.pendulum_reset(phys, obs, torch.zeros(4, dtype=i32), torch.zeros(4, dtype=i32),
                           torch.zeros(4, dtype=i32))


def test_pendulum_v1_is_routed_and_v0_is_not():
    import importlib
    ge = importlib.import_module("torchrl_b200.env.get_env")
    from torchrl_b200.env import PendulumVecEnv
    assert ge.is_pendulum("Pendulum-v1") and not ge.is_pendulum("Pendulum-v0")
    assert PendulumVecEnv.lockstep and PendulumVecEnv.resets_itself
    with pytest.raises(NotImplementedError):
        ge.get_vec_env("Pendulum-v0", {}, 2, device="cuda")
    # construction allocates device tensors: on a CPU-only box, Pendulum-v1 reaches the env class and stops there
    import torch
    if not torch.cuda.is_available():
        with pytest.raises((RuntimeError, AssertionError)):
            ge.get_vec_env("Pendulum-v1", {}, 2)
