"""NumPy statement of the device Pendulum-v1 (csrc/pendulum.cu): gym's PendulumEnv.step behind NormAct for a batch.

Constants: g = 10, m = 1, l = 1, dt = 0.05, max_speed = 8, max_torque = 2, time limit 200 steps.

    u        = clip(lb + (a + 1) * 0.5 * (ub - lb), lb, ub)     NormAct, float32, lb = -2, ub = 2; then widened exactly
    cost     = angle_normalize(th)**2 + 0.1 * thdot**2 + 0.001 * u**2
    newthdot = clip(thdot + (3*g/(2*l) * sin(th) + 3/(m*l**2) * u) * dt, -8, 8)
    newth    = th + newthdot * dt                                v1: the clipped velocity moves the angle
    reward   = float32(-cost * reward_scale)
    obs      = float32((cos newth, sin newth, newthdot))
    done     = elapsed >= 200 ;  time_limit = done and elapsed == 200

The state (th, thdot) is float64 and theta is never wrapped, as in gym.  angle_normalize(x) = ((x + pi) % (2 pi)) - pi
with Python's float %.  Resets draw th = pi (2U - 1), thdot = 2U - 1 from the counter hash of oracle/synth_env.py keyed
by (seed, episode, component).  Every dtype is explicit, so the result does not depend on NumPy's promotion rules.
"""
import math

import numpy as np

from . import synth_env

G = 10.0
M = 1.0
L = 1.0
DT = 0.05
MAX_SPEED = 8.0
MAX_TORQUE = 2.0
MAX_EPISODE_STEPS = 200
ENV_ID = "Pendulum-v1"


def torque(actions):
    """NormAct in float32: policy actions (n,) -> torques (n,) float32 in [-2, 2]."""
    a = np.asarray(actions, dtype=np.float32).reshape(-1)
    lb, ub = np.float32(-MAX_TORQUE), np.float32(MAX_TORQUE)
    u = lb + ((a + np.float32(1.0)) * np.float32(0.5)) * (ub - lb)
    return np.clip(u, lb, ub).astype(np.float32)


def angle_normalize(x):
    """((x + pi) % (2 pi)) - pi, float64, with Python's float % (the result takes the divisor's sign)."""
    x = np.asarray(x, dtype=np.float64)
    r = np.fmod(x + math.pi, 2.0 * math.pi)
    r = np.where(r < 0.0, r + 2.0 * math.pi, r)
    return r - math.pi


def dynamics(phys, actions):
    """phys (n, 2) float64, actions (n,) -> next phys (n, 2) float64 and cost (n,) float64."""
    s = np.asarray(phys, dtype=np.float64)
    th, thdot = s[:, 0], s[:, 1]
    u = torque(actions).astype(np.float64)
    an = angle_normalize(th)
    cost = (an * an + 0.1 * (thdot * thdot)) + 0.001 * (u * u)
    newthdot = thdot + ((3.0 * G / (2.0 * L)) * np.sin(th) + (3.0 / (M * L * L)) * u) * DT
    newthdot = np.clip(newthdot, -MAX_SPEED, MAX_SPEED)
    newth = th + newthdot * DT
    return np.stack([newth, newthdot], axis=1), cost


def observe(phys):
    """(cos th, sin th, thdot) rounded to float32."""
    s = np.asarray(phys, dtype=np.float64)
    return np.stack([np.cos(s[:, 0]), np.sin(s[:, 0]), s[:, 1]], axis=1).astype(np.float32)


def reset_phys(seeds, episodes):
    """Reset states (n, 2) float64 of the envs with these seeds and episode counters."""
    u = synth_env.hash_uniform(np.asarray(seeds, dtype=np.uint64).reshape(-1, 1),
                               np.asarray(episodes, dtype=np.uint64).reshape(-1, 1),
                               np.arange(2, dtype=np.uint64).reshape(1, -1)).astype(np.float64)
    return np.stack([math.pi * (2.0 * u[:, 0] - 1.0), 2.0 * u[:, 1] - 1.0], axis=1)


def step(phys, actions, elapsed, max_episode_steps=MAX_EPISODE_STEPS, reward_scale=1.0):
    """One step of the batch with the time limit: (next phys, obs, reward, done, time_limit, elapsed)."""
    nxt, cost = dynamics(phys, actions)
    el = np.asarray(elapsed, dtype=np.int64) + 1
    done = el >= max_episode_steps
    time_limit = done & (el == max_episode_steps)
    reward = (-cost * np.float64(np.float32(reward_scale))).astype(np.float32)
    return nxt, observe(nxt), reward, done, time_limit, el


def random_policy_return(n_envs=256, seed=0, steps=MAX_EPISODE_STEPS):
    """Mean undiscounted 200-step return of a uniformly random policy (actions U(-1, 1)) from the hash resets."""
    rs = np.random.RandomState(seed)
    phys = reset_phys(np.arange(n_envs), np.zeros(n_envs))
    ret = np.zeros(n_envs)
    el = np.zeros(n_envs, np.int64)
    for _ in range(steps):
        phys, _, r, _, _, el = step(phys, rs.uniform(-1, 1, n_envs).astype(np.float32), el)
        ret += r.astype(np.float64)
    return float(ret.mean())
