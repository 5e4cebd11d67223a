"""RIFE as a video processor (the reference's diffsynth/processors/RIFE.py) on the RIFEEngine of diffsynth.extensions.RIFE.

Every inner frame is replaced with RIFE's view of it from its two neighbours: the first pass interpolates each pair
(i - 1, i + 1); then, with interpolate=True, a second pass interpolates between frame i and that result, and with
interpolate=False frame i becomes the fp32 average of itself and that result (svi_rife_average_u8).  The first and last
frames stay.  This is not extensions.RIFE.RIFESmoother: its options live on the instance.

Sizes follow extensions.RIFE: a frame size that `check_size` accepts runs at its own size, any other raises ValueError.
The reference instead resizes such frames to (side + 31) // 32 pixels (it never multiplies back by 32), which IFNet
cannot run on; that resize is deliberately not reproduced.
"""
import torch

from .. import _native as nv
from ..extensions.RIFE import RIFEInterpolater, _scale_list, check_size
from .base import VideoProcessor, frames_like, frames_to_device


class RIFESmoother(VideoProcessor):
    device_frames = True

    def __init__(self, model, device="cuda", scale=1.0, batch_size=4, interpolate=True):
        self.model, self.device = model, device
        self.scale, self.batch_size, self.interpolate = scale, batch_size, interpolate

    @staticmethod
    def from_model_manager(model_manager, **kwargs):
        # the reference reads model_manager.RIFE, which its ModelManager does not define
        return RIFESmoother(model_manager.fetch_model("rife"), device=model_manager.device, **kwargs)

    @torch.no_grad()
    def __call__(self, rendered_frames, **kwargs):
        """PIL frames or a uint8 [F, H, W, 3] CUDA tensor -> the same kind, F >= 3 frames of one size"""
        if int(self.batch_size) < 1:
            raise ValueError(f"RIFESmoother: batch_size must be >= 1, got {self.batch_size}")
        nv.require_cuda(self.device, "RIFESmoother")
        u8 = frames_to_device(rendered_frames, self.device, "RIFESmoother")
        F, H, W, _ = u8.shape
        if F < 3:
            raise ValueError(f"RIFESmoother: needs at least 3 frames, got {F}")
        check_size(H, W, _scale_list(self.scale))
        interp = RIFEInterpolater(self.model, device=self.device)
        eng = interp._engine()
        if u8 is rendered_frames:
            u8 = u8.clone()                    # the caller's tensor stays as it was
        frames = nv.rife_stage_frames(u8, torch.empty(F, H, W, 4, device=eng.device))
        mid = torch.empty(F - 2, H, W, 4, device=eng.device)
        interp._pairs(frames[:-2], frames[2:], self.scale, int(self.batch_size), merged=mid)
        if self.interpolate:
            interp._pairs(frames[1:-1], mid, self.scale, int(self.batch_size), rgb=u8[1:-1])
        else:
            nv.rife_average_u8(frames, mid, u8)
        return frames_like(u8, rendered_frames)
