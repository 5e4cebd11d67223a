"""Processor dispatch and chaining with the reference's names and spelling (diffsynth/processors/sequencial_processor.py):
`AutoVideoProcessor.from_model_manager(model_manager, processor_type, **config)` builds one processor by type name, and
`SequencialProcessor` runs a list of them in order.

SequencialProcessor hands the frames from one processor to the next as a uint8 CUDA tensor while both sides run on the
kernel library (`device_frames`), so PIL frames are staged to the device once and converted back once; a processor
from outside this package gets PIL frames, as in the reference.  Staging needs RGB frames of one size: a chain refuses
other frames with ValueError, even where its first processor alone would convert them."""
import importlib

import torch

from .base import VideoProcessor, frames_like, frames_to_device

# processor_type -> (module of this package, class); the module is imported when its type is first asked for
PROCESSOR_TYPES = {
    "FastBlend": ("FastBlend", "FastBlendSmoother"),
    "Contrast": ("PILEditor", "ContrastEditor"),
    "Sharpness": ("PILEditor", "SharpnessEditor"),
    "RIFE": ("RIFE", "RIFESmoother"),
}


class AutoVideoProcessor(VideoProcessor):
    @staticmethod
    def from_model_manager(model_manager, processor_type, **kwargs):
        """The processor of `processor_type` ("FastBlend", "Contrast", "Sharpness" or "RIFE"), built by its own
        from_model_manager with kwargs as its configuration"""
        if processor_type not in PROCESSOR_TYPES:
            raise ValueError(f"invalid processor_type: {processor_type}")
        module, name = PROCESSOR_TYPES[processor_type]
        cls = getattr(importlib.import_module(f"{__package__}.{module}"), name)
        return cls.from_model_manager(model_manager, **kwargs)


class SequencialProcessor(VideoProcessor):
    def __init__(self, processors=None):
        self.processors = list(processors) if processors is not None else []

    @staticmethod
    def from_model_manager(model_manager, configs):
        """configs: [{"processor_type": ..., "config": {...}}, ...], run in this order"""
        return SequencialProcessor([AutoVideoProcessor.from_model_manager(model_manager, c["processor_type"], **c["config"])
                                    for c in configs])

    def __call__(self, rendered_frames, **kwargs):
        """Run every processor in order, each called with the previous one's frames and these kwargs (e.g.
        original_frames).  Returns PIL frames for PIL frames, and a uint8 tensor on the input's device for a tensor."""
        frames = rendered_frames
        for processor in self.processors:
            on_device = getattr(processor, "device_frames", False)
            if on_device and not torch.is_tensor(frames):
                frames = frames_to_device(frames, processor.device, type(processor).__name__)
            elif not on_device and torch.is_tensor(frames):
                frames = frames_like(frames, None)
            frames = processor(frames, **kwargs)
        if torch.is_tensor(rendered_frames):
            return frames_to_device(frames, rendered_frames.device, "SequencialProcessor")
        return frames_like(frames, None) if torch.is_tensor(frames) else frames
