"""FastBlend as a video processor (the reference's diffsynth/processors/FastBlend.py): the fast, balanced and accurate
deflicker modes through the runners of diffsynth.extensions.FastBlend.runners, on the native kernels."""
import torch

from ..extensions import FastBlend
from ..extensions.FastBlend import runners
from .base import VideoProcessor

_RUNNERS = {"fast": runners.FastModeRunner, "balanced": runners.BalancedModeRunner, "accurate": runners.AccurateModeRunner}


class FastBlendSmoother(VideoProcessor):
    """Deflickers rendered frames, guided by the original frames or, with original_frames=None, by the rendered frames
    themselves.  `inference_mode` is "fast", "balanced" or "accurate"; the other arguments are the reference's."""

    device_frames = True

    def __init__(self, inference_mode="fast", batch_size=8, window_size=60, minimum_patch_size=5, threads_per_block=8,
                 num_iter=5, gpu_id=0, guide_weight=10.0, initialize="identity", tracking_window_size=0):
        self.inference_mode = inference_mode
        self.batch_size = batch_size
        self.window_size = window_size
        self.ebsynth_config = {
            "minimum_patch_size": minimum_patch_size,
            "threads_per_block": threads_per_block,
            "num_iter": num_iter,
            "gpu_id": gpu_id,
            "guide_weight": guide_weight,
            "initialize": initialize,
            "tracking_window_size": tracking_window_size,
        }

    @property
    def device(self):
        return FastBlend._device(self.ebsynth_config["gpu_id"])

    @staticmethod
    def from_model_manager(model_manager, **kwargs):
        return FastBlendSmoother(**kwargs)

    def __call__(self, rendered_frames, original_frames=None, **kwargs):
        """PIL images (or uint8 [H, W, 3] arrays) -> PIL images, in frame order; a uint8 [F, H, W, 3] CUDA tensor ->
        a uint8 tensor on the device (original_frames may be either kind)"""
        if self.inference_mode not in _RUNNERS:
            raise ValueError("inference_mode must be fast, balanced or accurate")
        if not torch.is_tensor(rendered_frames):
            rendered_frames = list(rendered_frames)
        guide = rendered_frames if original_frames is None else original_frames
        if not torch.is_tensor(guide):
            guide = list(guide)
        return _RUNNERS[self.inference_mode]().run(guide, rendered_frames, self.batch_size, self.window_size,
                                                   self.ebsynth_config)
