"""Video processors with the reference's in-memory interface (diffsynth/processors): PIL frames in, PIL frames out.

The processors of this package that run on the kernel library (`device_frames = True`) also take the frames as a
uint8 [F, H, W, 3] CUDA tensor and then return one, so that a chain of them keeps the frames on the device."""
import numpy as np
import torch
from PIL import Image


class VideoProcessor:
    """A video processor: called with a list of frames, returns a list of frames (diffsynth/processors/base.py)."""

    # True: __call__ also takes a uint8 [F, H, W, 3] CUDA tensor and returns the same kind it was given
    device_frames = False

    def __init__(self):
        pass

    def __call__(self):
        raise NotImplementedError


def frames_to_device(frames, device, who):
    """PIL RGB frames of one size, or a uint8 [F, H, W, 3] tensor -> a contiguous uint8 [F, H, W, 3] tensor on `device`
    (the tensor itself when it is already there).  Anything else raises ValueError naming `who`."""
    if torch.is_tensor(frames):
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[0] == 0:
            raise ValueError(f"{who}: a frame tensor must be uint8 [F, H, W, 3], got {frames.dtype} {tuple(frames.shape)}")
        return frames.to(device).contiguous()
    frames = list(frames)
    if not frames:
        raise ValueError(f"{who}: no frames")
    if any(not isinstance(f, Image.Image) or f.mode != "RGB" for f in frames):
        raise ValueError(f"{who}: frames must be PIL images of mode RGB")
    if any(f.size != frames[0].size for f in frames):
        raise ValueError(f"{who}: every frame must have the size of the first, {frames[0].size}")
    return torch.from_numpy(np.stack([np.asarray(f) for f in frames])).to(device)


def frames_like(u8, given):
    """uint8 [F, H, W, 3] on the device -> the kind of `given`: the tensor when a tensor was given, else PIL images"""
    if torch.is_tensor(given):
        return u8
    return [Image.fromarray(f) for f in u8.cpu().numpy()]
