"""NumPy statement of the device MountainCar-v0 and MountainCarContinuous-v0 (csrc/mountain_car.cu): gym's
MountainCarEnv.step and Continuous_MountainCarEnv.step (behind NormAct) for a batch.

Constants: positions in [-1.2, 0.6], speeds in [-0.07, 0.07], gravity 0.0025; v0: force 0.001, goal 0.5, time limit
200; continuous: power 0.0015, goal 0.45, time limit 999.

    v0          v  = clip(v + ((a - 1) * 0.001 + cos(3 x) * (-0.0025)), -0.07, 0.07)      a in {0, 1, 2}
    continuous  u  = clip(lb + (a + 1) * 0.5 * (ub - lb), lb, ub)     NormAct, float32, lb = -1, ub = 1
                f  = min(max(u, -1), 1) widened to float64 (NumPy 1.x promotion: float32 scalar * Python float is float64)
                v  = clip(v + (f * 0.0015 - 0.0025 * cos(3 x)), -0.07, 0.07)
    both        x  = clip(x + v, -1.2, 0.6) ;  v = 0 if x == -1.2 and v < 0
                terminal = x >= goal and v >= 0
    reward      v0: -1 ; continuous: (100 if terminal else 0) - u**2 * 0.1 ;  times reward_scale, in float32
    obs         float32((x, v))

The state (x, v) is float64; every operation is rounded once in gym's order.  Resets draw x = -0.6 + 0.2 U from the
counter hash of oracle/synth_env.py keyed by (seed, episode, 0), and v = 0.
"""
import numpy as np

from . import synth_env

MIN_POSITION = -1.2
MAX_POSITION = 0.6
MAX_SPEED = 0.07
GRAVITY = 0.0025
FORCE = 0.001
POWER = 0.0015
# id: (goal position, time limit, continuous)
SPECS = {"MountainCar-v0": (0.5, 200, False), "MountainCarContinuous-v0": (0.45, 999, True)}


def norm_act(actions):
    """NormAct in float32 with lb = -1, ub = 1: policy actions (n,) -> env actions (n,) float32 in [-1, 1]."""
    a = np.asarray(actions, dtype=np.float32).reshape(-1)
    lb, ub = np.float32(-1.0), np.float32(1.0)
    u = lb + ((a + np.float32(1.0)) * np.float32(0.5)) * (ub - lb)
    return np.clip(u, lb, ub).astype(np.float32)


def dynamics(phys, actions, env_id):
    """phys (n, 2) float64, actions (n,) -> next phys (n, 2) float64, terminal (n,) bool and the base reward (n,)
    float64 (before reward_scale)."""
    goal, _, continuous = SPECS[env_id]
    s = np.asarray(phys, dtype=np.float64)
    x, v = s[:, 0], s[:, 1]
    c = np.cos(3 * x)
    if continuous:
        act = norm_act(actions).astype(np.float64)
        force = np.minimum(np.maximum(act, -1.0), 1.0)
        v = v + (force * POWER - GRAVITY * c)
    else:
        a = np.asarray(actions, dtype=np.float32).reshape(-1)
        if not np.all((a == 0) | (a == 1) | (a == 2)):
            raise ValueError("MountainCar-v0 actions are 0, 1 and 2")
        v = v + ((a.astype(np.float64) - 1.0) * FORCE + c * (-GRAVITY))
    v = np.clip(v, -MAX_SPEED, MAX_SPEED)
    x = np.clip(x + v, MIN_POSITION, MAX_POSITION)
    v = np.where((x == MIN_POSITION) & (v < 0), 0.0, v)
    term = terminal(np.stack([x, v], axis=1), env_id)
    if continuous:
        base = np.where(term, 100.0, 0.0) - (act * act) * 0.1
    else:
        base = np.full(x.shape, -1.0)
    return np.stack([x, v], axis=1), term, base


def terminal(phys, env_id):
    """position >= goal and velocity >= 0, on the new state."""
    s = np.asarray(phys, dtype=np.float64)
    return (s[:, 0] >= SPECS[env_id][0]) & (s[:, 1] >= 0)


def observe(phys):
    return np.asarray(phys, dtype=np.float64).astype(np.float32)


def reset_phys(seeds, episodes):
    """Reset states (n, 2) float64 of the envs with these seeds and episode counters."""
    u = synth_env.hash_uniform(np.asarray(seeds, dtype=np.uint64).reshape(-1),
                               np.asarray(episodes, dtype=np.uint64).reshape(-1), np.uint64(0)).astype(np.float64)
    return np.stack([-0.6 + 0.2 * u, np.zeros_like(u)], axis=1)


def step(phys, actions, elapsed, env_id, max_episode_steps=None, reward_scale=1.0):
    """One step of the batch with the time limit: (next phys, obs, reward, done, time_limit, elapsed)."""
    nxt, term, base = dynamics(phys, actions, env_id)
    limit = SPECS[env_id][1] if max_episode_steps is None else max_episode_steps
    el = np.asarray(elapsed, dtype=np.int64) + 1
    done = term | (el >= limit)
    time_limit = done & (el == limit)
    reward = (base * np.float64(np.float32(reward_scale))).astype(np.float32)
    return nxt, observe(nxt), reward, done, time_limit, el


def push(phys, env_id):
    """The scripted controller: push in the direction of the velocity (right while it is 0).  v0: actions 2 / 0;
    continuous: policy actions +1 / -1.  From 4096 hash resets it reaches the goal every time, in 113-125 steps (v0)
    and 105-111 steps (continuous).  Pushing left at v = 0 instead never leaves the valley from x near -0.489 in v0."""
    v = np.asarray(phys, dtype=np.float64)[:, 1]
    if SPECS[env_id][2]:
        return np.where(v >= 0, 1.0, -1.0).astype(np.float32)
    return np.where(v >= 0, 2.0, 0.0).astype(np.float32)


def episodes(policy, phys, env_id):
    """Run one episode of each env from `phys` under policy(phys) -> actions; returns (return, length, reached)."""
    phys = np.array(phys, dtype=np.float64)
    n = phys.shape[0]
    ret, length = np.zeros(n), np.zeros(n, np.int64)
    live = np.ones(n, bool)
    reached = np.zeros(n, bool)
    el = np.zeros(n, np.int64)
    for _ in range(SPECS[env_id][1]):
        phys, _, r, d, tl, el = step(phys, policy(phys), el, env_id)
        ret += np.where(live, r.astype(np.float64), 0.0)
        length += live
        reached |= live & d & ~tl
        live &= ~d
        if not live.any():
            break
    return ret, length, reached


def random_policy_return(env_id, n_envs=256, seed=0):
    """Mean undiscounted return of a uniformly random policy over one episode from the hash resets (v0: actions
    uniform over {0, 1, 2}; continuous: U(-1, 1))."""
    rs = np.random.RandomState(seed)
    if SPECS[env_id][2]:
        pol = lambda s: rs.uniform(-1, 1, s.shape[0]).astype(np.float32)       # noqa: E731
    else:
        pol = lambda s: rs.randint(0, 3, s.shape[0]).astype(np.float32)        # noqa: E731
    ret, _, _ = episodes(pol, reset_phys(np.arange(n_envs), np.zeros(n_envs)), env_id)
    return float(ret.mean())
