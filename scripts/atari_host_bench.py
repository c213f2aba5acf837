"""Cost of one step of host Atari envs (env/atari_host.py) over the fake ALE game (oracle/fake_ale.py), N in {16, 64,
256}:
  * the WarpFrame + FrameStack kernel: CUDA events over many launches on N resident frames, and the bytes it must move
    (the RGB frame read, the C-1 kept frames read and the C frames written per env) over that time against the H100
    SXM's 3.35 TB/s;
  * H2D bytes per step, from the shapes (the frames plus reward, done and time_limit);
  * host ms per step (synchronised) of this path -- action D2H, host chain, one copy into pinned staging, H2D, one
    launch -- and of the reference's layout: the same host chain, cv2 WarpFrame and a NumPy FrameStack per env on the
    host, then the full float32 stacks (ScaledFloatFrame) uploaded.
Prints the card and its power limit, then one JSON line.

    python scripts/atari_host_bench.py
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import fake_ale  # noqa: E402
from torchrl_b200 import ops  # noqa: E402
from torchrl_b200.env.atari_host import make_atari_host_env  # noqa: E402
from torchrl_b200.hostenv import VecEnv, get_atari_env  # noqa: E402
from scripts.pendulum_bench import HBM_BYTES_PER_S, card  # noqa: E402

ENV_ID = fake_ale.ENV_ID
PARAM = {"frame_stack": True, "scale": True, "clip_rewards": True}


def kernel_us(env, launches):
    acts = torch.zeros(env.env_nums, device="cuda")
    env.launch_step(acts)
    fr, st, ti, tw, nf = env._frames, env.obs, env._tab_i, env._tab_w, env._no_fresh
    for _ in range(10):
        ops.atari_warp_stack(fr, st, ti, tw, fresh=nf)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        ops.atari_warp_stack(fr, st, ti, tw, fresh=nf)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / launches


def host_ms(step, steps):
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def reference_layout_step(venv, stacks, dev_out, rs, cv2):
    """Host chain, cv2 WarpFrame + FrameStack per env, ScaledFloatFrame, full float32 stacks uploaded."""
    frames, _, _, _ = venv.step(rs.randint(0, 4, venv.env_nums))
    for n in range(venv.env_nums):
        g = cv2.resize(cv2.cvtColor(frames[n], cv2.COLOR_RGB2GRAY), (84, 84), interpolation=cv2.INTER_AREA)
        stacks[n, :-1] = stacks[n, 1:]
        stacks[n, -1] = g.astype(np.float32) / 255.0 - 0.5
    dev_out.copy_(torch.from_numpy(stacks), non_blocking=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    name, watts = card()
    print("card: %s, power limit: %s W" % (name, watts))
    try:
        import cv2
    except ImportError:
        cv2 = None
    rows = []
    for N in args.envs:
        env = make_atari_host_env(ENV_ID, PARAM, N, "cuda", make=fake_ale.make)
        env.seed(0)
        env.reset()
        H, W, _ = env.frame_shape
        C = env.frame_stack
        us = kernel_us(env, args.launches)
        moved = N * (H * W * 3 + (C - 1) * 84 * 84 + C * 84 * 84)
        rs = np.random.RandomState(0)
        acts = torch.zeros(N, device="cuda")

        def ours():
            acts.copy_(torch.from_numpy(rs.randint(0, 4, N).astype(np.float32)))
            env.launch_step(acts)
            if env.host_done.any():
                env.partial_reset(env.host_done)
        ms = host_ms(ours, args.steps)
        row = {"N": N, "kernel_us": us, "kernel_bytes": moved, "kernel_TBps": moved / us / 1e6,
               "share_of_hbm_peak": moved / us / 1e-6 / HBM_BYTES_PER_S, "h2d_bytes_per_step": env.h2d_bytes_per_step,
               "host_ms_per_step": ms}
        env.close()
        if cv2 is not None:
            venv = VecEnv(N, get_atari_env, [ENV_ID, PARAM, fake_ale.make])
            venv.seed(0)
            venv.reset()
            stacks = np.zeros((N, C, 84, 84), np.float32)
            dev_out = torch.empty(N, C, 84, 84, device="cuda")

            def ref():
                reference_layout_step(venv, stacks, dev_out, rs, cv2)
                d = venv._slots.done[:, 0]
                if d.any():
                    venv.partial_reset(d)
            row["reference_layout_host_ms_per_step"] = host_ms(ref, args.steps)
            row["reference_layout_h2d_bytes_per_step"] = stacks.nbytes
            venv.close()
        rows.append(row)
        print(row)
    print(json.dumps({"card": name, "power_limit_w": watts, "rows": rows}))


if __name__ == "__main__":
    main()
