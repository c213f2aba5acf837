"""NumPy restatement of the per-frame arithmetic of the reference's Atari chain (wrap_deepmind,
/root/reference/torchrl/env/get_env.py:8-22): WarpFrame's cv2.cvtColor(RGB2GRAY) and cv2.resize(INTER_AREA) to 84x84
(/root/reference/torchrl/env/atari_wrapper.py:112-131), FrameStack (:134-168) and ScaledFloatFrame (:171-180).

TEST INFRASTRUCTURE ONLY: the definition csrc/atari_frames.cu is checked against, itself checked against OpenCV.

* gray: OpenCV's 15-bit fixed-point RGB2GRAY for 8-bit images, (9798 R + 19235 G + 3735 B + 16384) >> 15.
* area_table: OpenCV's computeResizeAreaTab -- for each output index, the (output, source, weight) entries in OpenCV's
  order, computed in double from scale = 1 / (dsize / ssize) (as cv::resize derives it), weights stored as fp32, the
  1e-3 thresholds.
* resize_area: OpenCV's resizeArea for non-integer scales -- per source row buf[dx] += src[sx] * alpha over the x
  table; per output row sum = beta * buf for the first source row, then sum += beta * buf; round half to even and
  saturate.  Every operation is a separate fp32 rounding (NumPy does not fuse).
"""
import math

import numpy as np

OUT = 84


def gray(rgb):
    """(..., H, W, 3) uint8 -> (..., H, W) uint8."""
    x = rgb.astype(np.int64)
    return ((9798 * x[..., 0] + 19235 * x[..., 1] + 3735 * x[..., 2] + 16384) >> 15).astype(np.uint8)


def area_table(ssize, dsize=OUT):
    """[(d, s, alpha)] in OpenCV's order; alpha is np.float32."""
    scale = 1.0 / (dsize / ssize)
    tab = []
    for d in range(dsize):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, ssize - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, ssize - 1)
        s1 = min(s1, s2)
        if s1 - f1 > 1e-3:
            tab.append((d, s1 - 1, np.float32((s1 - f1) / cell)))
        for s in range(s1, s2):
            tab.append((d, s, np.float32(1.0 / cell)))
        if f2 - s2 > 1e-3:
            tab.append((d, s2, np.float32(min(min(f2 - s2, 1.0), cell) / cell)))
    return tab


def resize_area(g, out_h=OUT, out_w=OUT):
    """(..., H, W) uint8 -> (..., out_h, out_w) uint8, vectorised over the leading axes and the rows."""
    H, W = g.shape[-2:]
    src = g.astype(np.float32)
    buf = np.zeros(g.shape[:-1] + (out_w,), np.float32)
    for dx, sx, a in area_table(W, out_w):
        buf[..., dx] = buf[..., dx] + src[..., sx] * a
    out = np.zeros(g.shape[:-2] + (out_h, out_w), np.float32)
    seen = set()
    for dy, sy, b in area_table(H, out_h):
        t = b * buf[..., sy, :]
        out[..., dy, :] = t if dy not in seen else out[..., dy, :] + t
        seen.add(dy)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def warp(rgb):
    """WarpFrame.observation without the channel axis: (..., H, W, 3) -> (..., 84, 84)."""
    return resize_area(gray(rgb))


def stack_update(stack, frame, fresh):
    """FrameStack on one env's (C, 84, 84) stack: reset (fresh) fills every slot, step shifts and appends."""
    if fresh:
        stack[...] = frame
    else:
        stack[:-1] = stack[1:].copy()
        stack[-1] = frame
    return stack


def lut(scale):
    """The 256-entry map of the network input: ScaledFloatFrame's own expression, or float(x)."""
    if scale:
        return np.arange(256).astype(np.float32) / 255.0 - 0.5
    return np.arange(256).astype(np.float32)
