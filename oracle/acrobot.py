"""NumPy statement of the device Acrobot-v1 (csrc/acrobot.cu): gym's AcrobotEnv.step ("book" dynamics, no torque
noise) for a batch.

Constants: dt = 0.2; link lengths l1 = l2 = 1, masses m1 = m2 = 1, centres of mass lc1 = lc2 = 0.5, moments of inertia
I1 = I2 = 1, g = 9.8; velocity bounds 4 pi and 9 pi; torques (-1, 0, +1) for the actions (0, 1, 2); time limit 500.

    d1       = m1 lc1^2 + m2 (l1^2 + lc2^2 + 2 l1 lc2 cos t2) + I1 + I2
    d2       = m2 (lc2^2 + l1 lc2 cos t2) + I2
    phi2     = m2 lc2 g cos(t1 + t2 - pi/2)
    phi1     = -m2 l1 lc2 dt2^2 sin t2 - 2 m2 l1 lc2 dt2 dt1 sin t2 + (m1 lc1 + m2 l1) g cos(t1 - pi/2) + phi2
    ddt2     = (a + d2/d1 phi1 - m2 l1 lc2 dt1^2 sin t2 - phi2) / (m2 lc2^2 + I2 - d2^2/d1)
    ddt1     = -(d2 ddt2 + phi1) / d1
    s'       = RK4 over [0, dt]: k1..k4 at y, y + dt/2 k1, y + dt/2 k2, y + dt k3; y + dt/6 (k1 + 2 k2 + 2 k3 + k4)
    t1', t2' = wrap(., -pi, pi): add or remove 2 pi one turn at a time
    dt1',dt2'= clip to +-4 pi, +-9 pi
    terminal = -cos t1' - cos(t2' + t1') > 1 ;  reward = 0 if terminal else -1, times reward_scale, in float32
    obs      = float32((cos t1', sin t1', cos t2', sin t2', dt1', dt2'))

Every expression is evaluated left to right with Python's precedence, as gym writes it, one rounding per operation, in
float64.  Resets draw each of the four state components as 0.1 (2U - 1) from the counter hash of oracle/synth_env.py
keyed by (seed, episode, component).
"""
import math

import numpy as np

from . import synth_env

DT = 0.2
LINK_LENGTH_1 = 1.0
LINK_MASS_1 = 1.0
LINK_MASS_2 = 1.0
LINK_COM_POS_1 = 0.5
LINK_COM_POS_2 = 0.5
LINK_MOI = 1.0
G = 9.8
MAX_VEL_1 = 4 * math.pi
MAX_VEL_2 = 9 * math.pi
AVAIL_TORQUE = (-1.0, 0.0, 1.0)
MAX_EPISODE_STEPS = 500
ENV_ID = "Acrobot-v1"


def dsdt(s, a):
    """_dsdt of states s (n, 4) with torques a (n,): (n, 4) float64."""
    m1, m2, l1, lc1, lc2, I1, I2, g = (LINK_MASS_1, LINK_MASS_2, LINK_LENGTH_1, LINK_COM_POS_1, LINK_COM_POS_2,
                                       LINK_MOI, LINK_MOI, G)
    pi = math.pi
    theta1, theta2, dtheta1, dtheta2 = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    cos, sin = np.cos, np.sin
    d1 = m1 * lc1 ** 2 + m2 * (l1 ** 2 + lc2 ** 2 + 2 * l1 * lc2 * cos(theta2)) + I1 + I2
    d2 = m2 * (lc2 ** 2 + l1 * lc2 * cos(theta2)) + I2
    phi2 = m2 * lc2 * g * cos(theta1 + theta2 - pi / 2.0)
    phi1 = (-m2 * l1 * lc2 * (dtheta2 * dtheta2) * sin(theta2)
            - 2 * m2 * l1 * lc2 * dtheta2 * dtheta1 * sin(theta2)
            + (m1 * lc1 + m2 * l1) * g * cos(theta1 - pi / 2)
            + phi2)
    ddtheta2 = ((a + d2 / d1 * phi1 - m2 * l1 * lc2 * (dtheta1 * dtheta1) * sin(theta2) - phi2)
                / (m2 * lc2 ** 2 + I2 - (d2 * d2) / d1))
    ddtheta1 = -(d2 * ddtheta2 + phi1) / d1
    return np.stack([dtheta1, dtheta2, ddtheta1, ddtheta2], axis=1)


def wrap(x, m=-math.pi, M=math.pi):
    """gym's wrap: whole turns of M - m added or removed one at a time, elementwise."""
    x = np.array(x, dtype=np.float64, copy=True)
    diff = M - m
    while True:
        hi = x > M
        if not hi.any():
            break
        x = np.where(hi, x - diff, x)
    while True:
        lo = x < m
        if not lo.any():
            break
        x = np.where(lo, x + diff, x)
    return x


def torque(actions):
    """Actions (n,) in {0, 1, 2} -> torques (n,) float64; anything else raises."""
    a = np.asarray(actions, dtype=np.float32).reshape(-1)
    if not np.all((a == 0) | (a == 1) | (a == 2)):
        raise ValueError("Acrobot actions are 0, 1 and 2")
    return a.astype(np.float64) - 1.0


def dynamics(phys, actions):
    """phys (n, 4) float64, actions (n,) -> next phys (n, 4) float64 and terminal (n,) bool."""
    y0 = np.asarray(phys, dtype=np.float64)
    a = torque(actions)
    dt = DT
    dt2 = dt / 2.0
    k1 = dsdt(y0, a)
    k2 = dsdt(y0 + dt2 * k1, a)
    k3 = dsdt(y0 + dt2 * k2, a)
    k4 = dsdt(y0 + dt * k3, a)
    ns = y0 + dt / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4)
    ns[:, 0] = wrap(ns[:, 0])
    ns[:, 1] = wrap(ns[:, 1])
    ns[:, 2] = np.clip(ns[:, 2], -MAX_VEL_1, MAX_VEL_1)
    ns[:, 3] = np.clip(ns[:, 3], -MAX_VEL_2, MAX_VEL_2)
    return ns, terminal(ns)


def terminal(phys):
    s = np.asarray(phys, dtype=np.float64)
    return -np.cos(s[:, 0]) - np.cos(s[:, 1] + s[:, 0]) > 1.0


def goal_height(phys):
    """-cos t1 - cos(t2 + t1): the tip's height; the episode ends above 1."""
    s = np.asarray(phys, dtype=np.float64)
    return -np.cos(s[:, 0]) - np.cos(s[:, 1] + s[:, 0])


def observe(phys):
    """(cos t1, sin t1, cos t2, sin t2, dt1, dt2) rounded to float32."""
    s = np.asarray(phys, dtype=np.float64)
    return np.stack([np.cos(s[:, 0]), np.sin(s[:, 0]), np.cos(s[:, 1]), np.sin(s[:, 1]), s[:, 2], s[:, 3]],
                    axis=1).astype(np.float32)


def reset_phys(seeds, episodes):
    """Reset states (n, 4) float64 of the envs with these seeds and episode counters."""
    u = synth_env.hash_uniform(np.asarray(seeds, dtype=np.uint64).reshape(-1, 1),
                               np.asarray(episodes, dtype=np.uint64).reshape(-1, 1),
                               np.arange(4, dtype=np.uint64).reshape(1, -1)).astype(np.float64)
    return 0.1 * (2.0 * u - 1.0)


def step(phys, actions, elapsed, max_episode_steps=MAX_EPISODE_STEPS, reward_scale=1.0):
    """One step of the batch with the time limit: (next phys, obs, reward, done, time_limit, elapsed)."""
    nxt, term = dynamics(phys, actions)
    el = np.asarray(elapsed, dtype=np.int64) + 1
    done = term | (el >= max_episode_steps)
    time_limit = done & (el == max_episode_steps)
    reward = (np.where(term, 0.0, -1.0) * np.float64(np.float32(reward_scale))).astype(np.float32)
    return nxt, observe(nxt), reward, done, time_limit, el


def pump(phys):
    """The scripted controller, energy pumping: torque along dtheta2 - dtheta1 - sin theta2 (the second joint's swing
    relative to the first, against a spring that keeps the links from folding), as actions (n,) float32 in {0, 2}, or
    1 (no torque) where that is exactly 0.  It reaches the goal within 500 steps from all 2048 resets of seeds
    7 i + 3 at episode 0 (at most 335 steps, 84 on average), and from 99.97 % of 16384 other resets."""
    s = np.asarray(phys, dtype=np.float64)
    return (1.0 + np.sign(s[:, 3] - s[:, 2] - np.sin(s[:, 1]))).astype(np.float32)


def episodes(policy, phys, max_steps=MAX_EPISODE_STEPS):
    """Run one episode of each env from `phys` under policy(phys) -> actions; returns (return, length, reached)."""
    phys = np.array(phys, dtype=np.float64)
    n = phys.shape[0]
    ret, length = np.zeros(n), np.zeros(n, np.int64)
    live = np.ones(n, bool)
    reached = np.zeros(n, bool)
    el = np.zeros(n, np.int64)
    for _ in range(max_steps):
        phys, _, r, d, tl, el = step(phys, policy(phys), el, max_steps)
        ret += np.where(live, r, 0.0)
        length += live
        reached |= live & d & ~tl
        live &= ~d
        if not live.any():
            break
    return ret, length, reached


def random_policy_return(n_envs=256, seed=0):
    """Mean undiscounted return of a uniformly random policy over one episode from the hash resets."""
    rs = np.random.RandomState(seed)
    ret, _, _ = episodes(lambda s: rs.randint(0, 3, s.shape[0]).astype(np.float32),
                         reset_phys(np.arange(n_envs), np.zeros(n_envs)))
    return float(ret.mean())
