"""Contrast and sharpness editors (the reference's diffsynth/processors/PILEditor.py) on the kernels of
include/svi_b200_processors.h, byte for byte what Pillow's ImageEnhance.Contrast / Sharpness give.

Frames must be RGB and all of one size (one device layout); anything else raises ValueError, where the reference would
edit each frame on its own."""
import numpy as np
import torch

from .. import _native as nv
from .base import VideoProcessor, frames_like, frames_to_device


class _Editor(VideoProcessor):
    """An editor of every frame at one `rate` (the Image.blend factor); the frames of a PIL call go to `device`."""

    device_frames = True

    def __init__(self, rate=1.5):
        self.rate, self.device = rate, "cuda"

    @classmethod
    def from_model_manager(cls, model_manager, **kwargs):
        return cls(**kwargs)


class ContrastEditor(_Editor):
    """ImageEnhance.Contrast(frame).enhance(rate) on every frame: each frame blended with its mean grey."""

    def __call__(self, rendered_frames, **kwargs):
        rate = _rate(self.rate, "ContrastEditor")
        device = _device(rendered_frames, self.device)
        nv.require_cuda(device, "ContrastEditor")
        u8 = frames_to_device(rendered_frames, device, "ContrastEditor")
        F, H, W, _ = u8.shape
        sums = nv.luma_sum_u8(u8, torch.empty(F, dtype=torch.int64, device=u8.device))
        # ImageStat's mean: the histogram's sum over the pixel count in double, then int(mean + 0.5)
        grey = [float(int(s / (H * W) + 0.5)) for s in sums.tolist()]
        out = torch.empty_like(u8)
        nv.enhance_blend_u8(u8, torch.tensor(grey, dtype=torch.float32, device=u8.device), rate, out)
        return frames_like(out, rendered_frames)


class SharpnessEditor(_Editor):
    """ImageEnhance.Sharpness(frame).enhance(rate) on every frame: each frame blended with its ImageFilter.SMOOTH."""

    def __call__(self, rendered_frames, **kwargs):
        rate = _rate(self.rate, "SharpnessEditor")
        device = _device(rendered_frames, self.device)
        nv.require_cuda(device, "SharpnessEditor")
        u8 = frames_to_device(rendered_frames, device, "SharpnessEditor")
        return frames_like(nv.sharpen_u8(u8, rate, torch.empty_like(u8)), rendered_frames)


def _rate(rate, who):
    """Image.blend takes its alpha as a C float"""
    r = np.float32(rate)
    if not np.isfinite(r):
        raise ValueError(f"{who}: rate must be a finite number, got {rate!r}")
    return r


def _device(frames, default):
    """a frame tensor is edited where it lives; PIL frames go to the editor's device"""
    return frames.device if torch.is_tensor(frames) else default
