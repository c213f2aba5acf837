"""Per-env host chain of an Atari game: the non-pixel part of the reference's wrap_deepmind, applied by ONE object.

The reference builds, for a `*NoFrameskip` id (/root/reference/torchrl/env/get_env.py:8-22, :90-105):
    FrameStack( ClipRewardEnv( ScaledFloatFrame( WarpFrame( FireResetEnv( MaxAndSkipEnv( NoopResetEnv(
        EpisodicLifeEnv( BaseWrapper( TimeLimitAugment( gym.make(env_id) ))))))))))
AtariHostEnv restates every layer below WarpFrame and the reward clipping; it hands out the max-pooled RAW RGB frame
(H, W, 3) uint8, and the per-frame arithmetic (WarpFrame, FrameStack, ScaledFloatFrame) runs on the device over the
whole batch (env/atari_host.py, csrc/atari_frames.cu).  Layers, innermost first:
  * TimeLimitAugment.step  base_wrapper.py:152-156  info['time_limit'] = done and _max_episode_steps == _elapsed_steps,
                                                    when gym.make returned a TimeLimit (get_env.py:92-93)
  * EpisodicLifeEnv        atari_wrapper.py:64-95   a lost life (lives > 0) ends the episode; reset only on a real
                                                    game over, otherwise one NOOP step
  * NoopResetEnv           atari_wrapper.py:13-38   1..30 NOOPs drawn from unwrapped.np_random.randint after reset
  * MaxAndSkipEnv          atari_wrapper.py:98-123  4 frames of one action, rewards summed, the max of the last two
                                                    frames from a PERSISTENT two-slot buffer: a game over at frame
                                                    i < 2 of a step leaves one or both slots as an older step wrote them
  * FireResetEnv           atari_wrapper.py:41-61   FIRE then action 2 after reset, when the game has a FIRE action
  * ClipRewardEnv          atari_wrapper.py:126-132 sign of the summed reward, when clip_rewards
BaseWrapper's train/eval flags change nothing in this chain.  Nothing here imports gym or cv2.
"""
import numpy as np


class AtariHostEnv:
    def __init__(self, env, clip_rewards=False, noop_max=30, skip=4):
        self.env = env
        self.clip_rewards = bool(clip_rewards)
        self.noop_max = int(noop_max)
        self.skip = int(skip)
        meanings = env.unwrapped.get_action_meanings()
        if meanings[0] != "NOOP":
            raise ValueError("an Atari game's action 0 must be NOOP (NoopResetEnv), got %r" % (meanings[0],))
        self.fire = "FIRE" in meanings
        if self.fire and (meanings[1] != "FIRE" or len(meanings) < 3):
            raise ValueError("FireResetEnv needs FIRE as action 1 and at least 3 actions, got %r" % (meanings,))
        self._time_limit = type(env).__name__.find("TimeLimit") >= 0
        self.observation_space = env.observation_space
        self.action_space = env.action_space
        shape = tuple(self.observation_space.shape)
        if len(shape) != 3 or shape[2] != 3:
            raise ValueError("an Atari game hands out (H, W, 3) RGB frames, got %r" % (shape,))
        self._obs_buffer = np.zeros((2,) + shape, dtype=np.uint8)
        self.lives = 0
        self.was_real_done = True
        self.training = True

    def train(self):
        self.training = True

    def eval(self):
        self.training = False

    def seed(self, s):
        return self.env.seed(s)

    def close(self):
        self.env.close()

    def render(self, *a, **k):
        return self.env.render(*a, **k)

    # ---- TimeLimitAugment over the raw env
    def _raw_step(self, action):
        ob, rew, done, info = self.env.step(action)
        if self._time_limit:
            info["time_limit"] = done and self.env._max_episode_steps == self.env._elapsed_steps
        return ob, rew, done, info

    # ---- EpisodicLifeEnv
    def _life_step(self, action):
        ob, rew, done, info = self._raw_step(action)
        self.was_real_done = done
        lives = self.env.unwrapped.ale.lives()
        if lives < self.lives and lives > 0:
            done = True
        self.lives = lives
        return ob, rew, done, info

    def _life_reset(self):
        if self.was_real_done:
            ob = self.env.reset()
        else:
            ob = self._raw_step(0)[0]
        self.lives = self.env.unwrapped.ale.lives()
        return ob

    # ---- NoopResetEnv
    def _noop_reset(self):
        self._life_reset()
        noops = self.env.unwrapped.np_random.randint(1, self.noop_max + 1)
        ob = None
        for _ in range(noops):
            ob, _, done, _ = self._life_step(0)
            if done:
                ob = self._life_reset()
        return ob

    # ---- MaxAndSkipEnv
    def _skip_step(self, action):
        total, done, info = 0.0, None, None
        for i in range(self.skip):
            ob, rew, done, info = self._life_step(action)
            if i == self.skip - 2:
                self._obs_buffer[0] = ob
            if i == self.skip - 1:
                self._obs_buffer[1] = ob
            total += rew
            if done:
                break
        return self._obs_buffer.max(axis=0), total, done, info

    # ---- FireResetEnv, then the public API
    def reset(self, **kwargs):
        """The frame the reference's reset hands to WarpFrame: NoopReset's raw frame, or FireReset's max-pooled one."""
        ob = self._noop_reset()
        if not self.fire:
            return ob
        ob, _, done, _ = self._skip_step(1)
        if done:
            self._noop_reset()
        ob, _, done, _ = self._skip_step(2)
        if done:
            self._noop_reset()
        return ob

    def step(self, action):
        ob, rew, done, info = self._skip_step(int(action))
        if self.clip_rewards:
            rew = np.sign(rew)
        return ob, rew, done, info


def get_atari_env(env_id, env_param, make=None):
    """One Atari chain (reference: get_single_env with a 3-D observation, get_env.py:90-105).  `make` defaults to
    gym.make; pass any callable `make(env_id) -> env` for a game that is not registered with gym."""
    if make is None:
        import gym
        make = gym.make
    return AtariHostEnv(make(env_id), clip_rewards=bool((env_param or {}).get("clip_rewards", False)))
