"""numpy / torch restatements of the video processors (reference diffsynth/processors): Pillow 12.2's ImageEnhance
Contrast and Sharpness in numpy fp32, and processors/RIFE.py's RIFESmoother on top of oracle/rife_oracle.py.

Pillow's arithmetic, as its C code evaluates it (float operands, no FMA on x86-64):
  - L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16; ImageStat's mean is the sum of L over the pixel count in double;
  - Image.blend(a, b, alpha): t = (float) a + alpha * (float)(b - a) with alpha a C float; inside 0 <= alpha <= 1 the
    byte is (int) t, outside it t is clipped to [0, 255] first;
  - ImageFilter.SMOOTH: a 3x3 kernel of weights 1/13 around and 5/13 at the centre (fp32), summed from 0 in row-major tap
    order, stored as 0 / 255 / (int)(ss + 0.5); the border rows and columns are copied.
"""
import numpy as np
import torch

from oracle import rife_oracle as R

f32 = np.float32
SMOOTH_W = np.array([1, 1, 1, 1, 5, 1, 1, 1, 1], np.float32) / f32(13)


def luma_sum(frame):
    """uint8 RGB [H, W, 3] -> the integer sum of Pillow's L"""
    a = frame.astype(np.int64)
    return int(((19595 * a[..., 0] + 38470 * a[..., 1] + 7471 * a[..., 2] + 0x8000) >> 16).sum())


def blend(d, x, rate):
    """Image.blend(d, x, rate) on uint8 arrays (d broadcastable to x)"""
    r = f32(rate)
    d = np.asarray(d).astype(np.int32)
    t = d.astype(np.float32) + r * (x.astype(np.int32) - d).astype(np.float32)
    if 0 <= r <= 1:
        return t.astype(np.int32).astype(np.uint8)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, t.astype(np.int32))).astype(np.uint8)


def contrast(frame, rate):
    """ImageEnhance.Contrast(Image.fromarray(frame)).enhance(rate) on uint8 RGB [H, W, 3]"""
    mean = int(luma_sum(frame) / (frame.shape[0] * frame.shape[1]) + 0.5)
    return blend(mean, frame, rate)


def smooth(frame):
    """Image.fromarray(frame).filter(ImageFilter.SMOOTH) on uint8 RGB [H, W, 3]"""
    H, W = frame.shape[:2]
    out = frame.copy()
    if H < 3 or W < 3:
        return out
    x = frame.astype(np.float32)
    ss = np.zeros((H - 2, W - 2, 3), np.float32)
    for k, (dy, dx) in enumerate((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)):
        ss = ss + x[1 + dy:H - 1 + dy, 1 + dx:W - 1 + dx] * SMOOTH_W[k]
    out[1:-1, 1:-1] = np.where(ss <= 0, 0, np.where(ss >= 255, 255, (ss + f32(0.5)).astype(np.int32)))
    return out


def sharpness(frame, rate):
    """ImageEnhance.Sharpness(Image.fromarray(frame)).enhance(rate) on uint8 RGB [H, W, 3]"""
    return blend(smooth(frame), frame, rate)


def average_u8(x, merged):
    """processors/RIFE.py with interpolate=False, after the first pass: x f32 BGR [F, 3, H, W] (frames / 255), merged
    [F - 2, 3, H, W] -> uint8 RGB [F, H, W, 3]; the inner frames (x + merged) / 2, decoded by clipping and truncating"""
    y = x.clone()
    y[1:-1] = (x[1:-1] + merged) / 2
    return R.to_uint8(y)


def rife_smooth(sd, frames, scale=1.0, batch_size=4, interpolate=True, rnd=R._ident):
    """processors/RIFE.py RIFESmoother(scale, batch_size, interpolate) on uint8 RGB [F, H, W, 3] (sides that are
    multiples of 32, where the reference does not resize) -> uint8 RGB [F, H, W, 3]"""
    x = R.to_tensor(frames)
    mid = R._batched(sd, torch.cat((x[:-2], x[2:]), 1), scale, batch_size, rnd)
    if not interpolate:
        return average_u8(x, mid)
    x[1:-1] = R._batched(sd, torch.cat((x[1:-1], mid), 1), scale, batch_size, rnd)
    return R.to_uint8(x)
