"""A deterministic ALE-shaped game for the Atari host path (TEST INFRASTRUCTURE ONLY).

No ROM can be installed here, so this stands where `gym.make("PongNoFrameskip-v4")` stands in the reference
(/root/reference/torchrl/env/get_env.py:53): an env with the attributes wrap_deepmind reads
(`spec.id` containing NoFrameskip, `unwrapped.get_action_meanings()`, `unwrapped.ale.lives()`, `unwrapped.np_random`)
wrapped in a gym-style `TimeLimit` (`_max_episode_steps`, `_elapsed_steps`; its class name is what get_single_env
tests before applying TimeLimitAugment).

The game (integer state, one raw frame per step, no frame skip):
  * a cue bit picks the rewarded move: UP when cue == 0, DOWN when cue == 1.  A raw frame with the right move pays
    +2, with the wrong one -1, NOOP / FIRE 0 -- rewards outside {-1, 0, 1}, so the skip sum and the clipping matter;
  * the cue only changes on move frames: after the 2nd of every 4 move frames the next cue is drawn (and shown),
    after the 4th it takes effect.  Every agent step of MaxAndSkip is 4 frames of one action, so the cue is constant
    within a step and both max-pooled frames (the last two of the step) show the cue of the NEXT step: the optimal
    action is visible in the observation.  A life loss and a reset re-align the count;
  * a life is lost on every 6th wrong move frame since the last life loss (a wrong agent step never costs one alone;
    the second lands mid-skip, at its 2nd frame), and on every `hazard`-th raw frame since reset (policy-independent;
    it lands at any offset of a skip because NoopReset draws 1..30 noops);
  * game over when no life is left; like ALE, a step after the game is over changes nothing and reports done (the
    reference's chain does step there: EpisodicLife's NOOP reset can end the last life inside NoopReset's loop).

Analytic returns of the clipped game (EpisodicLife ends an episode at the first life loss): a uniformly random policy
earns 0 in expectation (each step's clipped reward is +1 or -1 with equal probability on a move, 0 otherwise, and the
cue is drawn independently of the past); the optimal policy never loses a life to a wrong move and earns +1 per agent
step until the hazard frame (see optimal_first_life_return).
"""
import numpy as np

H, W = 210, 160
ENV_ID = "FakeAleNoFrameskip-v4"
FIRE_MEANINGS = ["NOOP", "FIRE", "UP", "DOWN"]
PLAIN_MEANINGS = ["NOOP", "UP", "DOWN"]
RIGHT, WRONG = 2, -1
WRONG_PER_LIFE = 6


class Box:
    def __init__(self, low, high, shape, dtype):
        self.low = np.full(shape, low)
        self.high = np.full(shape, high)
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)


class Discrete:
    def __init__(self, n):
        self.n = int(n)
        self.shape = ()
        self.dtype = np.dtype(np.int64)


class Spec:
    def __init__(self, env_id):
        self.id = env_id


class _Ale:
    def __init__(self, game):
        self._game = game

    def lives(self):
        return self._game.lives_left


class FakeAle:
    def __init__(self, fire=True, lives=3, hazard=97, height=H, width=W):
        self.meanings = list(FIRE_MEANINGS if fire else PLAIN_MEANINGS)
        self.up, self.down = self.meanings.index("UP"), self.meanings.index("DOWN")
        self.start_lives, self.hazard = int(lives), int(hazard)
        self.observation_space = Box(0, 255, (height, width, 3), np.uint8)
        self.action_space = Discrete(len(self.meanings))
        self.spec = Spec(ENV_ID)
        self.ale = _Ale(self)
        self.np_random = np.random.RandomState(0)
        self.total_frames = 0                     # raw frames since construction (tests read it)
        r, c = np.arange(height)[:, None], np.arange(width)[None, :]
        self._bg = ((3 * r + 5 * c) % 61, (r * c) % 37, 40 + (c // 8 + r // 8) % 3 * 20)
        self._set_state(0)

    @property
    def unwrapped(self):
        return self

    def get_action_meanings(self):
        return list(self.meanings)

    def seed(self, seed=None):
        self.np_random = np.random.RandomState(seed)
        return [seed]

    def _set_state(self, cue):
        self.t = 0
        self.lives_left = self.start_lives
        self.moves = 0
        self.wrong = 0
        self.cue = self.next_cue = int(cue)
        self.game_over = False

    def reset(self):
        self._set_state(self.np_random.randint(2))
        return self.render()

    def step(self, action):
        action = int(action)
        assert 0 <= action < len(self.meanings)
        self.total_frames += 1
        if self.game_over:                        # as ALE: the game stays over until reset
            return self.render(), 0, True, {}
        self.t += 1
        reward = 0
        lost = False
        if action in (self.up, self.down):
            right = (action == self.up) == (self.cue == 0)
            reward = RIGHT if right else WRONG
            self.moves += 1
            if self.moves % 4 == 2:
                self.next_cue = int(self.np_random.randint(2))
            elif self.moves % 4 == 0:
                self.cue = self.next_cue
            if not right:
                self.wrong += 1
                lost = self.wrong % WRONG_PER_LIFE == 0
        lost = lost or self.t % self.hazard == 0
        if lost:
            self.lives_left -= 1
            self.moves, self.wrong, self.cue = 0, 0, self.next_cue
        self.game_over = self.lives_left <= 0
        return self.render(), reward, self.game_over, {}

    def render(self, mode="rgb_array"):
        """(H, W, 3) uint8: a moving background, the shown cue as a block on the left (0) or right (1) half, one
        square per life left along the top, and a bar whose length is the move count within the current 4."""
        b0, b1, b2 = self._bg
        f = np.empty(self.observation_space.shape, np.uint8)
        f[..., 0] = (b0 + 7 * self.t % 61) % 61
        f[..., 1] = (b1 + self.t % 37) % 37
        f[..., 2] = b2 if self.wrong % 2 == 0 else 100 - b2
        x0 = 8 if self.next_cue == 0 else f.shape[1] // 2 + 8
        f[40:150, x0:x0 + f.shape[1] // 2 - 16] = (230, 200, 40)
        for k in range(self.lives_left):
            f[8:20, 8 + 16 * k:20 + 16 * k] = (250, 250, 250)
        f[180:190, 8:8 + 9 * (self.moves % 4 + 1)] = (120, 255, 120)
        return f

    def close(self):
        pass


class TimeLimit:
    """gym.wrappers.TimeLimit as gym.make applies it: done once `_max_episode_steps` raw frames have elapsed."""

    def __init__(self, env, max_episode_steps):
        self.env = env
        self._max_episode_steps = int(max_episode_steps)
        self._elapsed_steps = None
        self.observation_space = env.observation_space
        self.action_space = env.action_space

    def step(self, action):
        ob, rew, done, info = self.env.step(action)
        self._elapsed_steps += 1
        if self._elapsed_steps >= self._max_episode_steps:
            info["TimeLimit.truncated"] = not done
            done = True
        return ob, rew, done, info

    def reset(self, **kwargs):
        self._elapsed_steps = 0
        return self.env.reset(**kwargs)

    @property
    def unwrapped(self):
        return self.env.unwrapped

    def __getattr__(self, attr):
        if attr.startswith("__") or attr == "env":
            raise AttributeError(attr)
        return getattr(self.env, attr)


def make(env_id=ENV_ID, fire=True, lives=3, hazard=97, max_episode_steps=400, height=H, width=W):
    """What `gym.make(env_id)` would return for the fake game."""
    assert "NoFrameskip" in env_id
    return TimeLimit(FakeAle(fire=fire, lives=lives, hazard=hazard, height=height, width=width), max_episode_steps)


def optimal_first_life_return(hazard, fire=True, noop_max=30):
    """Expected clipped return of the optimal policy from a real reset to the first life loss under wrap_deepmind:
    NoopReset's n ~ U{1..noop_max} noops and, with FIRE, FireReset's two 4-frame steps come first; every later agent
    step of 4 frames earns +1 until (and including) the step holding raw frame `hazard`."""
    pre = 8 if fire else 0
    steps = [-(-(hazard - n - pre) // 4) for n in range(1, noop_max + 1)]
    return float(np.mean(steps))
