"""Atari games through the host chain (hostenv/atari.py), CPU side: the NumPy restatement of WarpFrame against OpenCV,
the host area tables against the restatement, the product's host chain + the restated WarpFrame / FrameStack /
ScaledFloatFrame against the reference's executed wrap_deepmind over the fake ALE game, and the env routing."""
import numpy as np
import pytest

from oracle import atari_frames as af
from oracle import fake_ale

SIZES = ((210, 160), (250, 160))


def _random_frames(rs, H, W, k):
    out = []
    for i in range(k):
        f = rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
        if i % 3 == 1:
            f = (f // 64 * 64).astype(np.uint8)
        elif i % 3 == 2:
            f = np.full((H, W, 3), rs.randint(0, 256, 3), np.uint8)
            f[rs.randint(0, H - 40):, rs.randint(0, W - 40):][:40, :40] = rs.randint(0, 256, 3)
        out.append(f)
    return np.stack(out)


@pytest.mark.parametrize("H,W", SIZES)
def test_oracle_warp_equals_opencv(H, W, golden_dir):
    cv2 = pytest.importorskip("cv2")
    z = np.load("%s/atari_frames.npz" % golden_dir)
    rgb = z["rgb_%d" % H]
    np.testing.assert_array_equal(af.warp(rgb), z["warp_%d" % H])
    fresh = _random_frames(np.random.RandomState(H), H, W, 9)
    for f in np.concatenate([rgb, fresh]):
        g = cv2.cvtColor(f, cv2.COLOR_RGB2GRAY)
        np.testing.assert_array_equal(af.gray(f), g)
        np.testing.assert_array_equal(af.resize_area(g), cv2.resize(g, (84, 84), interpolation=cv2.INTER_AREA))
    # the vectorised restatement equals itself frame by frame
    np.testing.assert_array_equal(af.warp(fresh), np.stack([af.warp(f) for f in fresh]))


@pytest.mark.parametrize("H,W", SIZES + ((84, 96), (97, 336)))
def test_host_area_tables_equal_the_oracle(H, W):
    from torchrl_b200.env.atari_host import area_tables
    tab_i, tab_w = area_tables(H, W)
    xt, yt = af.area_table(W), af.area_table(H)
    nx, ny = len(xt), len(yt)
    assert tab_i.dtype == np.int32 and tab_w.dtype == np.float32 and tab_i.size == 170 + nx + ny
    for ofs, src, w, tab in ((tab_i[:85], tab_i[170:170 + nx], tab_w[:nx], xt),
                             (tab_i[85:170], tab_i[170 + nx:], tab_w[nx:], yt)):
        np.testing.assert_array_equal(ofs, np.searchsorted([d for d, _, _ in tab], np.arange(85)))
        np.testing.assert_array_equal(src, [s for _, s, _ in tab])
        np.testing.assert_array_equal(w, np.array([a for _, _, a in tab], np.float32))


def test_lut_is_scaled_float_frames_expression():
    from torchrl_b200.env.atari_host import frame_lut
    x = np.arange(256, dtype=np.uint8)
    np.testing.assert_array_equal(frame_lut(True), np.array(x).astype(np.float32) / 255.0 - 0.5)
    np.testing.assert_array_equal(frame_lut(False), x.astype(np.float32))
    np.testing.assert_array_equal(af.lut(True), frame_lut(True))


def test_fake_game_rules():
    g = fake_ale.FakeAle(fire=False, lives=2, hazard=1000)
    g.seed(1)
    g.reset()
    right = g.up if g.cue == 0 else g.down
    assert [g.step(right)[1] for _ in range(4)] == [2, 2, 2, 2]
    assert g.moves == 4 and g.cue == g.next_cue
    rews = []
    for _ in range(6):
        wrong = g.down if g.cue == 0 else g.up          # the cue may change after every 4th move
        rews.append(g.step(wrong)[1])
    assert rews == [-1] * 6 and g.lives_left == 1 and g.moves == 0
    assert [g.step(0)[1] for _ in range(3)] == [0, 0, 0] and g.moves == 0
    assert fake_ale.optimal_first_life_return(97) == np.mean([-(-(97 - n - 8) // 4) for n in range(1, 31)])


# ---------------------------------------------------------------------------------------------------- host chain
FIRE_ID, PLAIN_ID = "FakeAleNoFrameskip-v4", "FakeAleNoFireNoFrameskip-v4"
VARIANTS = {FIRE_ID: dict(fire=True, lives=5, hazard=37, max_episode_steps=100),
            PLAIN_ID: dict(fire=False, lives=4, hazard=53, max_episode_steps=90)}


def make_fake(env_id):
    """Top-level (picklable) `make` hook of the fake game's ids."""
    return fake_ale.make(env_id, **VARIANTS[env_id])


class Replay:
    """The product's chain (hostenv VecEnv of AtariHostEnv) fed through the oracle's WarpFrame + FrameStack + LUT."""

    def __init__(self, venv, scale, C=4):
        self.venv, self.lut, self.C = venv, af.lut(scale), C
        self.stack = None

    def reset(self):
        w = af.warp(np.asarray(self.venv.reset()))
        self.stack = np.repeat(w[:, None], self.C, axis=1)
        return self.lut[self.stack]

    def step(self, acts):
        ob, r, d, info = self.venv.step(acts)
        w = af.warp(np.asarray(ob))
        self.stack = np.concatenate([self.stack[:, 1:], w[:, None]], axis=1)
        return self.lut[self.stack], np.array(r), np.array(d), np.array(info["time_limit"])

    def partial_reset(self, mask):
        ob = np.asarray(self.venv.partial_reset(mask))
        w = af.warp(ob[mask])
        self.stack[mask] = w[:, None]
        return self.lut[self.stack]


def _ref_vecenv(ref, N, env_id, env_param):
    import gym
    for k in VARIANTS:
        gym.register(k, lambda k=k: make_fake(k))
    from torchrl.env.get_env import get_single_env
    from torchrl.env.vecenv import VecEnv
    return VecEnv(N, get_single_env, [env_id, dict(env_param)])


@pytest.mark.reference
@pytest.mark.parametrize("env_id", [FIRE_ID, PLAIN_ID])
@pytest.mark.parametrize("scale,clip", [(True, True), (False, False)])
def test_host_chain_equals_reference_wrap_deepmind(env_id, scale, clip):
    from oracle import reference_loader
    from torchrl_b200.hostenv import VecEnv, get_atari_env
    ref_mod = reference_loader.load()
    param = {"frame_stack": True, "scale": scale, "clip_rewards": clip}
    N, T = 6, 120
    ref = _ref_vecenv(ref_mod, N, env_id, param)
    prod_venv = VecEnv(N, get_atari_env, [env_id, param, make_fake])
    mine = Replay(prod_venv, scale)
    games = [e.env.unwrapped for e in prod_venv.envs]
    rs = np.random.RandomState(5)
    seen = {"life": 0, "game_over": 0, "mid_skip": 0, "time_limit": 0, "partial": 0}
    for mode in ("train", "eval"):
        getattr(ref, mode)()
        getattr(prod_venv, mode)()
        ref.seed(11)
        prod_venv.seed(11)
        np.testing.assert_array_equal(np.asarray(ref.reset()), mine.reset())
        nA = len(games[0].meanings)
        for t in range(T):
            # mostly random play, with stretches of one move per env so that wrong moves cost lives mid-skip
            acts = rs.randint(0, nA, N) if t % 20 < 12 else np.full(N, games[0].up)
            before = [g.total_frames for g in games]
            o1, r1, d1, i1 = ref.step(acts)
            o2, r2, d2, tl2 = mine.step(acts)
            np.testing.assert_array_equal(np.asarray(o1), o2)
            np.testing.assert_array_equal(np.asarray(r1), r2)
            np.testing.assert_array_equal(np.asarray(d1), d2)
            np.testing.assert_array_equal(np.asarray(i1["time_limit"]).astype(bool), tl2)
            for n, g in enumerate(games):
                if d2[n, 0]:
                    over = g.game_over
                    seen["game_over"] += over
                    seen["life"] += not over and not tl2[n]
                    seen["mid_skip"] += over and g.total_frames - before[n] <= 2
                    seen["time_limit"] += tl2[n]
            if d2.any():
                mask = d2[:, 0]
                seen["partial"] += 1
                np.testing.assert_array_equal(np.asarray(ref.partial_reset(mask)), mine.partial_reset(mask))
    assert all(v > 0 for v in seen.values()), seen


def test_noframeskip_ids_are_routed_to_the_atari_host_env():
    import importlib
    import torch
    ge = importlib.import_module("torchrl_b200.env.get_env")
    assert ge.is_atari("PongNoFrameskip-v4") and ge.is_atari(FIRE_ID) and not ge.is_atari("Pong-v4")
    try:
        import gym  # noqa: F401
        has_gym = True
    except ImportError:
        has_gym = False
    if not has_gym:
        for fn in (lambda: ge.get_vec_env("PongNoFrameskip-v4", {}, 2, device="cuda"),
                   lambda: ge.get_subprocvec_env("BreakoutNoFrameskip-v4", {}, 2, 2, device="cuda")):
            with pytest.raises(NotImplementedError, match="gym.*ALE"):
                fn()
    for other in ("Pong-v4", "Acrobot-v0", "Pendulum-v0", "LunarLander-v2", "MountainCar-v1"):
        with pytest.raises(NotImplementedError):
            ge.get_vec_env(other, {}, 2, device="cuda")
    if not torch.cuda.is_available():
        # with a make= hook the id reaches the device env, which needs a GPU
        with pytest.raises((RuntimeError, AssertionError)):
            ge.get_vec_env(FIRE_ID, {}, 2, device="cuda", make=make_fake)
