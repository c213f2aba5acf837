"""Atari games stepped on the host, their frames processed on the device: the pixel env of a `*NoFrameskip` id.

Each host env runs the non-pixel part of the reference's wrap_deepmind (hostenv/atari.py) and hands out its
max-pooled raw RGB frame; the batch's WarpFrame (gray + INTER_AREA to 84x84, bit for bit with OpenCV) and FrameStack
run as one kernel launch (csrc/atari_frames.cu) into `obs`, the (N, C, 84, 84) uint8 stack the pixel collectors read.
ScaledFloatFrame becomes `to_float`, a 256-entry map applied where frames enter a network.

One step: one D2H copy of the actions and one stream sync; the host steps every env; one host copy of each frame
from the vec env's slot into pinned staging; one H2D copy of the frames, rewards and flags; one launch.
`partial_reset` uploads only the masked envs' fresh frames (packed, with their env ids) and refills only their stacks
(one launch, none when no env is masked).
"""
import math

import numpy as np
import torch

from .. import ops
from ..spaces import Box

F32, U8, I32 = torch.float32, torch.uint8, torch.int32
OUT = 84


def area_tables(H, W, out=OUT):
    """OpenCV's INTER_AREA tables (computeResizeAreaTab, scale = 1 / (out / size) as cv::resize derives it) of
    W -> out and H -> out in the kernel's CSR form: tab_i = [xofs (out+1) | yofs (out+1) | xsrc | ysrc] int32,
    tab_w = [xw | yw] float32."""
    def one(ssize):
        scale = 1.0 / (out / ssize)
        ofs, src, w = [0], [], []
        for d in range(out):
            f1 = d * scale
            f2 = f1 + scale
            cell = min(scale, ssize - f1)
            s1, s2 = math.ceil(f1), math.floor(f2)
            s2 = min(s2, ssize - 1)
            s1 = min(s1, s2)
            if s1 - f1 > 1e-3:
                src.append(s1 - 1)
                w.append((s1 - f1) / cell)
            for s in range(s1, s2):
                src.append(s)
                w.append(1.0 / cell)
            if f2 - s2 > 1e-3:
                src.append(s2)
                w.append(min(min(f2 - s2, 1.0), cell) / cell)
            ofs.append(len(src))
        return ofs, src, w
    xo, xs, xw = one(W)
    yo, ys, yw = one(H)
    return np.array(xo + yo + xs + ys, dtype=np.int32), np.array(xw + yw, dtype=np.float32)


def frame_lut(scale):
    """to_float's map: ScaledFloatFrame's own expression (atari_wrapper.py:180) with `scale`, else float(x)."""
    x = np.arange(256).astype(np.float32)
    return x / 255.0 - 0.5 if scale else x


def _pad16(n):
    return (n + 15) & ~15


class AtariHostVecEnv:
    pixel = True
    host_bridge = True
    lockstep = False
    obs_norm = False
    _obs_normalizer = None

    def __init__(self, host_env, env_param=None, device="cuda"):
        env_param = dict(env_param or {})
        self.host = host_env
        self.env_nums = N = int(host_env.env_nums)
        self.device = dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("AtariHostVecEnv feeds a CUDA pipeline (there is no CPU path); got %r" % (device,))
        H, W, three = (int(s) for s in host_env.observation_space.shape)
        if three != 3 or H < OUT or W < OUT or (3 * W) % 16:
            raise ValueError("Atari frames must be (H, W, 3) with H, W >= 84 and 3W % 16 == 0, got %r"
                             % (tuple(host_env.observation_space.shape),))
        self.frame_shape = (H, W, 3)
        self.frame_stack = C = 4 if env_param.get("frame_stack", True) else 1
        self.scale = bool(env_param.get("scale", False))
        self.observation_space = Box(0, 255, (C, OUT, OUT), dtype=np.uint8)
        self.action_space = host_env.action_space
        self._reward_scale = 1
        self.training = True
        self.dist = None
        F = H * W * 3
        # ---- staging: [env ids i32 N | frames u8 N*F | reward f32 N | done u8 N | time_limit u8 N], pinned + twin.
        # A step uploads [frames .. end); a partial reset packs its k frames first and uploads [0, frames + k*F).
        f0 = _pad16(4 * N)
        r0 = f0 + N * F
        cuts = (0, f0, r0, r0 + 4 * N, r0 + 5 * N, r0 + 6 * N)
        nbytes = _pad16(cuts[-1])
        self._pin = torch.empty(nbytes, dtype=U8, pin_memory=True)
        self._dev = torch.zeros(nbytes, dtype=U8, device=dev)
        pin_np = self._pin.numpy()
        self._h_idx = pin_np[cuts[0]:cuts[0] + 4 * N].view(np.int32)
        self._h_frames = pin_np[cuts[1]:cuts[2]].reshape(N, H, W, 3)
        self._h_rew = pin_np[cuts[2]:cuts[3]].view(np.float32)
        self._h_done = pin_np[cuts[3]:cuts[4]]
        self._h_tl = pin_np[cuts[4]:cuts[5]]
        self._idx = self._dev[cuts[0]:cuts[0] + 4 * N].view(I32)
        self._frames = self._dev[cuts[1]:cuts[2]].view(N, H, W, 3)
        self.reward = self._dev[cuts[2]:cuts[3]].view(F32)
        self.done = self._dev[cuts[3]:cuts[4]]
        self.time_limit = self._dev[cuts[4]:cuts[5]]
        self._f0, self._F, self._step_lo, self._step_hi = f0, F, f0, cuts[-1]
        self.obs = torch.zeros(N, C, OUT, OUT, dtype=U8, device=dev)
        self._no_fresh = torch.zeros(N, dtype=U8, device=dev)
        tab_i, tab_w = area_tables(H, W)
        self._tab_i = torch.from_numpy(tab_i).to(dev)
        self._tab_w = torch.from_numpy(tab_w).to(dev)
        self._lut = torch.from_numpy(frame_lut(self.scale)).to(dev)
        self._act_pin = torch.empty(N, dtype=F32, pin_memory=True)
        self._act_np = self._act_pin.numpy()
        self._h2d_done = None
        self.host_done = np.zeros(N, dtype=bool)                 # host copy of the last step's `done`
        self.h2d_bytes_per_step = self._step_hi - self._step_lo
        self.d2h_bytes_per_step = 4 * N

    # ------------------------------------------------------------------ reference API
    def train(self):
        self.training = True
        self.host.train()

    def eval(self):
        self.training = False
        self.host.eval()

    def close(self):
        self.host.close()

    def render(self, *a, **k):
        return None

    def seed(self, seed):
        self.host.seed(seed)

    def _wait_staging(self):
        """The pinned block may still be the source of an H2D copy in flight: wait before the host rewrites it."""
        if self._h2d_done is not None:
            self._h2d_done.synchronize()

    def _upload(self, lo, hi):
        self._dev[lo:hi].copy_(self._pin[lo:hi], non_blocking=True)
        if self._h2d_done is None:
            self._h2d_done = torch.cuda.Event()
        self._h2d_done.record(torch.cuda.current_stream(self.device))

    def reset(self, **kwargs):
        frames = self.host.reset(**kwargs)
        self._wait_staging()
        np.copyto(self._h_frames, frames, casting="no")
        self._upload(self._f0, self._f0 + self.env_nums * self._F)
        ops.atari_warp_stack(self._frames, self.obs, self._tab_i, self._tab_w)
        return self.obs

    def partial_reset(self, index_mask, **kwargs):
        """Masked host reset; the masked envs' stacks are refilled with their new first frame, the others kept."""
        if torch.is_tensor(index_mask):
            index_mask = index_mask.reshape(-1).bool().cpu().numpy()
        mask = np.asarray(index_mask).reshape(-1).astype(bool)
        idx = np.flatnonzero(mask)
        if idx.size == 0:
            return self.obs
        frames = self.host.partial_reset(mask, **kwargs)
        k = idx.size
        self._wait_staging()
        self._h_idx[:k] = idx
        np.take(frames, idx, axis=0, out=self._h_frames[:k])
        self._upload(0, self._f0 + k * self._F)
        ops.atari_warp_stack(self._frames[:k], self.obs, self._tab_i, self._tab_w, env_idx=self._idx[:k])
        return self.obs

    def launch_step(self, actions, *unused, **unused_kw):
        """actions (N,) on the device -> host step -> frames, rewards and flags on the device -> `obs` in place."""
        self._act_pin.copy_(actions.reshape(-1), non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        frames, rew, done, infos = self.host.step(self._act_np.astype(np.int64))
        self._wait_staging()
        np.copyto(self._h_frames, frames, casting="no")
        np.copyto(self._h_rew, np.asarray(rew).reshape(-1), casting="same_kind")
        done = np.asarray(done).reshape(-1).astype(bool)
        self._h_done[...] = done
        tl = infos.get("time_limit", None) if isinstance(infos, dict) else None
        self._h_tl[...] = 0 if tl is None else np.asarray(tl).reshape(-1).astype(bool)
        self.host_done = done
        self._upload(self._step_lo, self._step_hi)
        ops.atari_warp_stack(self._frames, self.obs, self._tab_i, self._tab_w, fresh=self._no_fresh)
        return self.obs

    def step(self, actions):
        """obs (N, C, 84, 84) uint8, reward (N, 1), done (N, 1) bool, {'time_limit': (N,) bool} -- device tensors."""
        act = torch.as_tensor(actions, device=self.device).reshape(-1).to(F32).contiguous()
        self.launch_step(act)
        return self.obs, self.reward.unsqueeze(-1), self.done.bool().unsqueeze(-1), \
            {"time_limit": self.time_limit.bool()}

    def to_float(self, obs_u8, out=None):
        """uint8 frames -> float32 through the 256-entry map (ScaledFloatFrame with `scale`, else float(x))."""
        return ops.u8_lut_f32(obs_u8, self._lut, out)

    def __deepcopy__(self, memo):
        raise TypeError("an AtariHostVecEnv owns live host envs and cannot be deep-copied: build a second env "
                        "for evaluation and pass it as eval_env")


def make_atari_host_env(env_id, env_param, env_nums, device, make=None, proc_nums=None):
    """The device pixel env over `env_nums` host Atari chains: in this process, or in `proc_nums` worker processes
    (then `make` must be picklable).  `make(env_id) -> env` defaults to gym.make."""
    from ..hostenv import SubProcVecEnv, VecEnv, get_atari_env
    if make is None:
        try:
            import gym  # noqa: F401
        except ImportError:
            raise NotImplementedError("%r is an Atari game: it needs gym with the Atari games (ALE and its ROMs) "
                                      "installed, or a make= hook" % (env_id,)) from None
    if device is None:
        device = "cuda"
    args = [env_id, env_param, make]
    if proc_nums:
        host = SubProcVecEnv(int(proc_nums), int(env_nums), get_atari_env, args)
    else:
        host = VecEnv(int(env_nums), get_atari_env, args)
    return AtariHostVecEnv(host, env_param, device=device)
