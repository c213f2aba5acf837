"""Acrobot-v1 without a GPU: the NumPy statement (oracle/acrobot.py) against gym's constants, a scalar transcription of
gym's step and a step from rest worked by hand, gym's wrap loop, the time limit, the reset hash, the random-policy
baseline, the scripted controller, the argument checks of trl_acrobot_step / trl_acrobot_reset, the ops wrappers'
operand checks and the env-id routing."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import acrobot as A
from oracle import synth_env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_constants():
    assert (A.DT, A.LINK_LENGTH_1, A.LINK_MASS_1, A.LINK_MASS_2, A.LINK_COM_POS_1, A.LINK_COM_POS_2, A.LINK_MOI,
            A.G) == (0.2, 1.0, 1.0, 1.0, 0.5, 0.5, 1.0, 9.8)
    assert A.MAX_VEL_1 == 4 * math.pi and A.MAX_VEL_2 == 9 * math.pi and A.AVAIL_TORQUE == (-1.0, 0.0, 1.0)
    assert A.MAX_EPISODE_STEPS == 500 and A.ENV_ID == "Acrobot-v1"
    src = open(os.path.join(ROOT, "torchrl_b200", "csrc", "acrobot.cu")).read()
    for line in ("kAcroDt = 0.2;", "kAcroL1 = 1.0;", "kAcroM1 = 1.0;", "kAcroM2 = 1.0;", "kAcroLc1 = 0.5;",
                 "kAcroLc2 = 0.5;", "kAcroI1 = 1.0;", "kAcroI2 = 1.0;", "kAcroG = 9.8;", "kAcroPi = 3.141592653589793;",
                 "kAcroMaxVel1 = 4.0 * kAcroPi;", "kAcroMaxVel2 = 9.0 * kAcroPi;"):
        assert line in src, line


# gym's AcrobotEnv.step, transcribed for one env with Python floats and the math module
def _gym_dsdt(s, a):
    m1 = m2 = l1 = 1.0
    lc1 = lc2 = 0.5
    I1 = I2 = 1.0
    g = 9.8
    pi = math.pi
    theta1, theta2, dtheta1, dtheta2 = s
    cos, sin = math.cos, math.sin
    d1 = m1 * lc1 ** 2 + m2 * (l1 ** 2 + lc2 ** 2 + 2 * l1 * lc2 * cos(theta2)) + I1 + I2
    d2 = m2 * (lc2 ** 2 + l1 * lc2 * cos(theta2)) + I2
    phi2 = m2 * lc2 * g * cos(theta1 + theta2 - pi / 2.0)
    phi1 = (-m2 * l1 * lc2 * dtheta2 ** 2 * sin(theta2) - 2 * m2 * l1 * lc2 * dtheta2 * dtheta1 * sin(theta2)
            + (m1 * lc1 + m2 * l1) * g * cos(theta1 - pi / 2) + phi2)
    ddtheta2 = (a + d2 / d1 * phi1 - m2 * l1 * lc2 * dtheta1 ** 2 * sin(theta2) - phi2) / (m2 * lc2 ** 2 + I2
                                                                                          - d2 ** 2 / d1)
    ddtheta1 = -(d2 * ddtheta2 + phi1) / d1
    return [dtheta1, dtheta2, ddtheta1, ddtheta2]


def _gym_wrap(x, m, M):
    diff = M - m
    while x > M:
        x = x - diff
    while x < m:
        x = x + diff
    return x


def _gym_step(s, action):
    torque = [-1.0, 0.0, +1][action]
    dt = 0.2
    dt2 = dt / 2.0
    k1 = _gym_dsdt(s, torque)
    k2 = _gym_dsdt([y + dt2 * k for y, k in zip(s, k1)], torque)
    k3 = _gym_dsdt([y + dt2 * k for y, k in zip(s, k2)], torque)
    k4 = _gym_dsdt([y + dt * k for y, k in zip(s, k3)], torque)
    ns = [y + dt / 6.0 * (a + 2 * b + 2 * c + d) for y, a, b, c, d in zip(s, k1, k2, k3, k4)]
    ns[0] = _gym_wrap(ns[0], -math.pi, math.pi)
    ns[1] = _gym_wrap(ns[1], -math.pi, math.pi)
    ns[2] = min(max(ns[2], -4 * math.pi), 4 * math.pi)
    ns[3] = min(max(ns[3], -9 * math.pi), 9 * math.pi)
    terminal = bool(-math.cos(ns[0]) - math.cos(ns[1] + ns[0]) > 1.0)
    return ns, terminal


def test_oracle_matches_a_scalar_transcription_of_gym():
    rs = np.random.RandomState(3)
    n = 200
    phys = np.stack([rs.uniform(-math.pi, math.pi, n), rs.uniform(-math.pi, math.pi, n),
                     rs.uniform(-4 * math.pi, 4 * math.pi, n), rs.uniform(-9 * math.pi, 9 * math.pi, n)], 1)
    phys[:20] = rs.uniform(-0.1, 0.1, (20, 4))
    acts = rs.randint(0, 3, n)
    got, term = A.dynamics(phys, acts.astype(np.float32))
    for i in range(n):
        want, wterm = _gym_step(list(phys[i]), int(acts[i]))
        # NumPy's vectorised sin / cos may differ from libm's in the last bit; the arithmetic around them is the same
        np.testing.assert_allclose(got[i], want, rtol=1e-12, atol=1e-12)
        if abs(A.goal_height(got[i:i + 1])[0] - 1.0) > 1e-9:
            assert term[i] == wterm
    assert np.abs(got[:, 2]).max() <= 4 * math.pi and np.abs(got[:, 3]).max() <= 9 * math.pi
    assert (np.abs(got[:, 3]) == 9 * math.pi).any()                  # the bound was exercised


def test_one_step_from_rest_worked_by_hand():
    """From rest with torque 0, gravity enters only through cos(theta - pi/2) at theta = 0, i.e. cos(-pi/2) =
    6.123233995736766e-17 in fp64: the link accelerates by that residue and the state moves off zero by ~1e-17."""
    c = math.cos(-math.pi / 2)
    assert c == 6.123233995736766e-17
    d1, d2 = 0.25 + (1.25 + 1.0) + 1.0 + 1.0, (0.25 + 0.5) + 1.0
    assert (d1, d2) == (4.5, 1.75)
    phi2 = 4.9 * c
    phi1 = ((-0.5 * 0.0) * 0.0 - 0.0) + (1.5 * 9.8) * c + phi2
    dd2 = (0.0 + d2 / d1 * phi1 - 0.0 - phi2) / (1.25 - (d2 * d2) / d1)
    dd1 = -(d2 * dd2 + phi1) / d1
    k1 = A.dsdt(np.zeros((1, 4)), np.zeros(1))[0]
    assert k1.tolist() == [0.0, 0.0, dd1, dd2]
    assert dd1 < 0 and dd2 > 0 and abs(dd1) < 1e-15 and abs(dd2) < 1e-15
    nxt, term = A.dynamics(np.zeros((1, 4)), [1.0])
    want, _ = _gym_step([0.0, 0.0, 0.0, 0.0], 1)
    np.testing.assert_allclose(nxt[0], want, rtol=1e-12, atol=0)
    assert not term[0] and np.all(nxt[0] != 0.0) and np.abs(nxt[0]).max() < 1e-15
    assert nxt[0, 0] < 0 and nxt[0, 2] < 0                          # the first link starts to fall one way
    _, obs, r, d, tl, el = A.step(np.zeros((1, 4)), [1.0], [0])
    assert obs.dtype == np.float32 and obs[0, [0, 2]].tolist() == [1.0, 1.0] and r.tolist() == [-1.0]
    assert not d[0] and not tl[0] and el.tolist() == [1]


def test_terminal_step_has_zero_reward():
    # link 1 up and link 2 in line: the tip is at height 2
    phys = np.array([[math.pi - 0.05, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0]])
    _, _, r, d, tl, _ = A.step(phys, [1.0, 1.0], [10, 10], reward_scale=0.5)
    assert d.tolist() == [True, False] and tl.tolist() == [False, False]
    assert r.tolist() == [0.0, -0.5]


@pytest.mark.parametrize("x", [0.0, 3.0, -3.0, math.pi, -math.pi, 3.2, -3.2, 7.0, -7.0, 20.0, -20.0, 100.5, -100.5,
                               2 * math.pi + 1e-9, 1e3])
def test_wrap_matches_the_loop(x):
    got = A.wrap(np.array([x]))[0]
    assert got == _gym_wrap(x, -math.pi, math.pi)
    assert -math.pi <= got <= math.pi
    if abs(x) > 3 * math.pi:
        # more than a turn out of range: the loop's repeated subtraction is not Python's %
        r = ((x + math.pi) % (2 * math.pi)) - math.pi
        assert abs(got - r) < 1e-9


def test_wrap_keeps_the_ends_and_differs_from_fmod():
    assert A.wrap([math.pi, -math.pi]).tolist() == [math.pi, -math.pi]   # the loop leaves +-pi where they are
    xs = np.linspace(-60, 60, 20001)
    got = A.wrap(xs)
    assert np.all(np.abs(got) <= math.pi)
    fm = np.fmod(xs + math.pi, 2 * math.pi)
    fm = np.where(fm < 0, fm + 2 * math.pi, fm) - math.pi
    assert np.max(np.abs(got - fm)) < 1e-13 and np.any(got != fm)      # fmod rounds differently


def test_invalid_actions_raise():
    with pytest.raises(ValueError):
        A.dynamics(np.zeros((2, 4)), [0.0, 1.5])


def test_time_limit():
    phys = np.zeros((3, 4))
    _, _, _, done, tl, el = A.step(phys, [1.0, 1.0, 1.0], [498, 499, 0])
    assert done.tolist() == [False, True, False] and tl.tolist() == [False, True, False]
    assert el.tolist() == [499, 500, 1]
    _, _, _, done, tl, _ = A.step(phys, [1.0] * 3, [500, 10, 0], max_episode_steps=11)
    assert done.tolist() == [True, True, False] and tl.tolist() == [False, True, False]


def test_reset_uses_the_synth_hash():
    seeds, eps = np.arange(6) * 5 + 1, np.arange(6)
    phys = A.reset_phys(seeds, eps)
    for j in range(4):
        u = synth_env.hash_uniform(seeds.astype(np.uint64), eps.astype(np.uint64), np.uint64(j))
        assert phys[:, j].tolist() == (0.1 * (2.0 * u - 1.0)).tolist()
    assert np.abs(phys).max() <= 0.1


def test_random_policy_baseline():
    """A uniformly random policy from the hash resets almost never lifts the tip within 500 steps: -499.5 over 256 envs
    (seed 0) and -498.6 over 1024 (seed 1).  The learning tests' thresholds sit far above it."""
    r = A.random_policy_return()
    assert abs(r - (-499.484375)) < 1e-9, r


def test_scripted_controller_reaches_the_goal():
    n = 2048
    ret, length, reached = A.episodes(A.pump, A.reset_phys(np.arange(n) * 7 + 3, np.zeros(n)))
    assert reached.all() and length.max() == 335 and 80 < length.mean() < 90
    np.testing.assert_array_equal(ret, -(length - 1.0))              # -1 per step, 0 on the terminal one


# ------------------------------------------------------------------------------------------ C ABI
def _step(lib, N=4, max_steps=500, **null):
    names = ("phys", "obs", "actions", "elapsed", "reward", "done", "time_limit", "action_error")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_acrobot_step(p["phys"], p["obs"], p["actions"], p["elapsed"], None, p["reward"], p["done"],
                                p["time_limit"], p["action_error"], None, None, None, None, None, None, None, None,
                                N, 1.0, max_steps, 1 << 30, 0, None)


def test_step_rejects_bad_arguments(native_lib):
    for kw in (dict(N=-1), dict(max_steps=0)):
        assert _step(native_lib, **kw) == -1, kw
        assert b"trl_acrobot_step: bad sizes" in native_lib.trl_last_error()
    for n in ("phys", "obs", "actions", "elapsed", "reward", "done", "time_limit", "action_error"):
        assert _step(native_lib, **{n: True}) == -1, n
        assert b"null pointer" in native_lib.trl_last_error()
    p = ctypes.c_void_p(16)
    assert native_lib.trl_acrobot_step(p, p, p, p, None, p, p, p, p, p, None, None, None, None, None, None, None, 4,
                                       1.0, 500, 1 << 30, 0, None) == -1
    assert b"ticket" in native_lib.trl_last_error()
    assert native_lib.trl_acrobot_step(p, p, p, p, None, p, p, p, p, p, None, None, None, None, p, None, None, 4,
                                       1.0, 500, 1 << 30, 1, None) == -1
    assert b"merge_stats" in native_lib.trl_last_error()
    assert native_lib.trl_acrobot_step(p, p, p, p, None, p, p, p, p, None, None, None, None, None, None, None, p, 4,
                                       1.0, 500, 1 << 30, 0, None) == -1
    assert b"any_reset" in native_lib.trl_last_error()
    assert _step(native_lib, N=0, phys=True) == 0           # nothing to do: no pointer is read


def _reset(lib, N=4, mask=None, step_count=None, next_norm=None, cur_ob=None, any_reset=None, t_ptr=None,
           norm_mean=None, norm_var=None, **null):
    names = ("phys", "obs", "elapsed", "episode", "seeds")
    p = {n: (None if n in null else ctypes.c_void_p(16)) for n in names}
    return lib.trl_acrobot_reset(p["phys"], p["obs"], p["elapsed"], p["episode"], p["seeds"], mask, step_count,
                                 next_norm, cur_ob, any_reset, t_ptr, norm_mean, norm_var, N, 10.0, 1, None)


def test_reset_rejects_bad_arguments(native_lib):
    p = ctypes.c_void_p(16)
    assert _reset(native_lib, N=-1) == -1
    assert b"trl_acrobot_reset: bad size" in native_lib.trl_last_error()
    for n in ("phys", "obs", "elapsed", "episode", "seeds"):
        assert _reset(native_lib, **{n: True}) == -1, n
        assert b"trl_acrobot_reset: null pointer" in native_lib.trl_last_error()
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
    assert [native_lib.trl_acrobot_num_ctas(n) for n in (1, 256, 257, 4099, 1 << 20)] == [1, 1, 2, 17, 4096]


def test_ops_wrappers_check_operands():
    import torch
    from torchrl_b200 import ops
    i32, u8, f64 = torch.int32, torch.uint8, torch.float64
    phys, obs = torch.zeros(4, 4, dtype=f64), torch.zeros(4, 6)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.acrobot_step(phys, obs, torch.zeros(4), torch.zeros(4, dtype=i32), None, torch.zeros(4),
                         torch.zeros(4, dtype=u8), torch.zeros(4, dtype=u8), torch.zeros(1, dtype=i32), None, None,
                         None, None, None, torch.zeros(1, dtype=i32), torch.zeros(2, dtype=i32), None, 1.0, 500,
                         1000, False)
    with pytest.raises(ValueError, match="one action per env"):
        ops.acrobot_step(phys, obs, torch.zeros(3), *([None] * 18))
    with pytest.raises(ValueError, match=r"\(N, 4\) and obs \(N, 6\)"):
        ops.acrobot_step(torch.zeros(4, 2, dtype=f64), obs, torch.zeros(4), *([None] * 18))
    with pytest.raises(ValueError, match=r"\(N, 4\)"):
        ops.acrobot_reset(phys, torch.zeros(4, 3), None, None, None)
    with pytest.raises(ValueError, match="not both"):
        ops.acrobot_reset(phys, obs, None, None, None, mask=torch.zeros(4, dtype=u8), step_count=torch.zeros(4, dtype=i32))
    with pytest.raises(ValueError, match="cur_ob needs"):
        ops.acrobot_reset(phys, obs, None, None, None, step_count=torch.zeros(4, dtype=i32), cur_ob=obs)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ops.acrobot_reset(phys, obs, torch.zeros(4, dtype=i32), torch.zeros(4, dtype=i32), torch.zeros(4, dtype=i32))


def test_acrobot_v1_is_routed():
    import importlib
    ge = importlib.import_module("torchrl_b200.env.get_env")
    from torchrl_b200.env import AcrobotVecEnv
    assert ge.is_acrobot("Acrobot-v1") and not ge.is_acrobot("Acrobot-v0")
    assert not AcrobotVecEnv.lockstep and AcrobotVecEnv.resets_itself and not AcrobotVecEnv._host_mirror_ok
    for other in ("Acrobot-v0", "Pendulum-v0", "LunarLander-v2"):
        with pytest.raises(NotImplementedError):
            ge.get_vec_env(other, {}, 2, device="cuda")
    import torch
    if not torch.cuda.is_available():
        # construction allocates device tensors: on a CPU-only box, Acrobot-v1 reaches the env class and stops there
        with pytest.raises((RuntimeError, AssertionError)):
            ge.get_vec_env("Acrobot-v1", {}, 2)
