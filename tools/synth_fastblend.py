"""Synthetic video for the FastBlend tests, golden and benchmark: uint8 [n, H, W, 3] frames of smooth colour fields that
drift from frame to frame, with a per-frame flicker and pixel noise (what a deflickerer is for)."""
import hashlib

import numpy as np


def make_frames(n, H, W, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    out = []
    for t in range(n):
        base = np.stack([np.sin((x + 2.5 * t) / 7.0 + c) * np.cos((y - 1.5 * t) / 9.0 - c) for c in range(3)], -1)
        flick = rng.normal(0, 12, size=3)
        img = 128 + 90 * base + flick + rng.normal(0, 6, size=(H, W, 3))
        out.append(img.clip(0, 255).astype(np.uint8))
    return np.stack(out)


def nnf_inputs(H, W, B, seed):
    """one estimate_nnf batch: source guide, target guide (uint8, the next frames) and a non-integer f32 source style"""
    f = make_frames(B + 1, H, W, seed)
    ss = (f[:B].astype(np.float32) * np.float32(0.75) + np.float32(20.3)).astype(np.float32)
    return f[:B], f[1:], ss


def digest(a, dtype):
    """SHA-256 of the C-order bytes of `a` cast to `dtype` (exact for the golden's int32 fields and f32 frames): pins
    large arrays bit for bit without storing them"""
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a).astype(dtype, copy=False)).tobytes()).hexdigest()
