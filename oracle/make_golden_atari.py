"""Write tests/golden/atari_frames.npz: OpenCV's WarpFrame outputs on adversarial RGB frames (TEST INFRASTRUCTURE ONLY).

    python oracle/make_golden_atari.py        # needs cv2

For each frame size (210x160, ALE's, and 250x160) the file holds `rgb_<H>` (K, H, W, 3) uint8 and, computed by the
installed OpenCV exactly as the reference's WarpFrame does (/root/reference/torchrl/env/atari_wrapper.py:124-131),
`warp_<H>` = cv2.resize(cv2.cvtColor(rgb, RGB2GRAY), (84, 84), INTER_AREA), plus `cv2_version`.
The frames: black, white, a one-pixel checkerboard, isolated bright pixels on the area cells' borders, horizontal and
vertical ramps, a flat field with a block, coarse quantised noise, a band of full-range noise, and pixels whose gray
values sit on rounding ties of the area weights.  The GPU tests compare the kernel with these arrays without needing OpenCV.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "atari_frames.npz")
SIZES = ((210, 160), (250, 160))


def frames(H, W, seed):
    rs = np.random.RandomState(seed)
    r, c = np.arange(H)[:, None], np.arange(W)[None, :]
    fs = [np.zeros((H, W, 3), np.uint8), np.full((H, W, 3), 255, np.uint8)]
    fs.append(np.repeat(((r + c) % 2 * 255).astype(np.uint8)[..., None], 3, axis=2))
    dots = np.zeros((H, W, 3), np.uint8)
    dots[::5, ::2] = 255                                      # on the 2.5-row / 1.905-column cell borders
    dots[1::7, 1::3] = (255, 0, 128)
    fs.append(dots)
    fs.append(np.stack([np.broadcast_to(c * 255 // (W - 1), (H, W)), np.broadcast_to(r * 255 // (H - 1), (H, W)),
                        np.broadcast_to((r + c) % 256, (H, W))], axis=2).astype(np.uint8))
    flat = np.full((H, W, 3), rs.randint(0, 256, 3), np.uint8)
    flat[50:91, 31:70] = rs.randint(0, 256, 3)
    fs.append(flat)
    fs.append(np.repeat(rs.randint(0, 4, (H, W // 4, 3)) * 64 + 63, 4, axis=1).astype(np.uint8))
    noise = np.zeros((H, W, 3), np.uint8)
    noise[H // 2 - 24:H // 2 + 24] = rs.randint(0, 256, (48, W, 3))     # a band keeps the file small
    fs.append(noise)
    ties = np.zeros((H, W, 3), np.uint8)
    ties[:, 1::2] = (1, 1, 1)                                 # gray 1 next to 0: sums land near .5
    ties[::2] += np.uint8(127)
    fs.append(ties)
    return np.stack(fs)


def main():
    import cv2
    out = {"cv2_version": np.array(cv2.__version__)}
    for k, (H, W) in enumerate(SIZES):
        rgb = frames(H, W, 100 + k)
        gray = [cv2.cvtColor(f, cv2.COLOR_RGB2GRAY) for f in rgb]
        out["rgb_%d" % H] = rgb
        out["warp_%d" % H] = np.stack([cv2.resize(g, (84, 84), interpolation=cv2.INTER_AREA) for g in gray])
    np.savez_compressed(OUT, **out)
    print("%s: %d bytes" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    sys.exit(main())
