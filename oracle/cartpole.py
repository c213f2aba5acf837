"""NumPy statement of the device CartPole (csrc/cartpole.cu): gym's CartPoleEnv.step for a batch.

The dynamics are gym's classic-control cart-pole (its constants, its Euler integrator, its termination thresholds),
computed in float64 from the float32 state and rounded to float32 once, every product and quotient in gym's order of
evaluation.  Resets use the counter hash of oracle/synth_env.py with a half-width of 0.05.

    temp      = (F + m_pole*l*theta_dot**2*sin(theta)) / (m_cart + m_pole)
    theta_acc = (g*sin(theta) - cos(theta)*temp) / (l*(4/3 - m_pole*cos(theta)**2/(m_cart + m_pole)))
    x_acc     = temp - m_pole*l*theta_acc*cos(theta)/(m_cart + m_pole)
    x += tau*x_dot ; x_dot += tau*x_acc ; theta += tau*theta_dot ; theta_dot += tau*theta_acc
    done      = |x| > 2.4 or |theta| > 12 degrees or elapsed >= max_episode_steps ; reward = 1 on every step
"""
import math

import numpy as np

from . import synth_env

GRAVITY = 9.8
MASS_CART = 1.0
MASS_POLE = 0.1
TOTAL_MASS = MASS_POLE + MASS_CART
LENGTH = 0.5                              # half the pole's length
POLE_MASS_LENGTH = MASS_POLE * LENGTH
FORCE_MAG = 10.0
TAU = 0.02
THETA_THRESHOLD = 12 * 2 * math.pi / 360
X_THRESHOLD = 2.4
INIT_SCALE = 0.05
MAX_EPISODE_STEPS = {"CartPole-v0": 200, "CartPole-v1": 500}


def dynamics64(state, actions):
    """state (n, 4) float32, actions (n,) in {0, 1} -> the next state (n, 4) in float64, before its rounding."""
    s = np.asarray(state, dtype=np.float32).astype(np.float64)
    x, x_dot, theta, theta_dot = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    force = np.where(np.asarray(actions).reshape(-1) == 1, FORCE_MAG, -FORCE_MAG)
    costh, sinth = np.cos(theta), np.sin(theta)
    temp = (force + POLE_MASS_LENGTH * (theta_dot * theta_dot) * sinth) / TOTAL_MASS
    thetaacc = (GRAVITY * sinth - costh * temp) / (LENGTH * (4.0 / 3.0 - MASS_POLE * (costh * costh) / TOTAL_MASS))
    xacc = temp - POLE_MASS_LENGTH * thetaacc * costh / TOTAL_MASS
    return np.stack([x + TAU * x_dot, x_dot + TAU * xacc, theta + TAU * theta_dot, theta_dot + TAU * thetaacc], axis=1)


def dynamics(state, actions):
    """state (n, 4) float32, actions (n,) in {0, 1} -> next state (n, 4) float32 and done_dyn (n,) bool."""
    nxt = dynamics64(state, actions).astype(np.float32)
    return nxt, terminated(nxt)


def terminated(state):
    """gym's termination test on the (float32) state, compared in float64."""
    s = np.asarray(state, dtype=np.float32).astype(np.float64)
    return (np.abs(s[:, 0]) > X_THRESHOLD) | (np.abs(s[:, 2]) > THETA_THRESHOLD)


def reset_state(seeds, episodes):
    """Reset states (n, 4) float32 of the envs with these seeds and episode counters."""
    u = synth_env.hash_uniform(np.asarray(seeds, dtype=np.uint64).reshape(-1, 1),
                               np.asarray(episodes, dtype=np.uint64).reshape(-1, 1),
                               np.arange(4, dtype=np.uint64).reshape(1, -1)).astype(np.float64)
    return (INIT_SCALE * (2.0 * u - 1.0)).astype(np.float32)


def step(state, actions, elapsed, max_episode_steps, reward_scale=1.0):
    """One step of the batch with the time limit: (next state, reward, done, time_limit, elapsed)."""
    nxt, done_dyn = dynamics(state, actions)
    el = np.asarray(elapsed, dtype=np.int64) + 1
    done = done_dyn | (el >= max_episode_steps)
    time_limit = done & (el == max_episode_steps)
    reward = np.full(len(el), np.float32(reward_scale), dtype=np.float32)
    return nxt, reward, done, time_limit, el
