"""Pipeline base: size checks, PIL<->tensor conversion, CPU-generator noise (reference pipelines/base.py).

Residency policy on H100 (80 GB HBM3): every model stays resident on the device; the reference's
offload / onload choreography (base.py:111-137, vram_management/layers.py) has nothing to do here, so
``load_models_to_device`` only makes sure the named models live on ``self.device``.
"""
import numpy as np
import torch
from PIL import Image


class BasePipeline(torch.nn.Module):
    def __init__(self, device="cuda", torch_dtype=torch.float16, height_division_factor=64, width_division_factor=64):
        super().__init__()
        self.device = device
        self.torch_dtype = torch_dtype
        self.height_division_factor = height_division_factor
        self.width_division_factor = width_division_factor
        self.cpu_offload = False
        self.model_names = []

    def check_resize_height_width(self, height, width):
        """round up to the division factor (reference base.py:21-28)."""
        for name, f in (("height", self.height_division_factor), ("width", self.width_division_factor)):
            v = height if name == "height" else width
            if v % f != 0:
                v = (v + f - 1) // f * f
                print(f"The {name} cannot be evenly divided by {f}. We round it up to {v}.")
            if name == "height":
                height = v
            else:
                width = v
        return height, width

    def preprocess_image(self, image, use_aug=False):
        """PIL RGB -> f32 [1,3,H,W] in [-1,1] (reference base.py:44-48).  Augmentation is a training feature."""
        if use_aug:
            raise NotImplementedError("training-time augmentation is outside the inference hot path")
        return torch.from_numpy(np.array(image, dtype=np.float32) * (2 / 255) - 1).permute(2, 0, 1).unsqueeze(0)

    def preprocess_images(self, images):
        return [self.preprocess_image(im) for im in images]

    def vae_output_to_image(self, vae_output):
        im = vae_output[0].cpu().float().permute(1, 2, 0).numpy()
        return Image.fromarray(((im / 2 + 0.5).clip(0, 1) * 255).astype("uint8"))

    def vae_output_to_video(self, vae_output):
        v = vae_output.cpu().permute(1, 2, 0).numpy()
        return [Image.fromarray(((im / 2 + 0.5).clip(0, 1) * 255).astype("uint8")) for im in v]

    def enable_cpu_offload(self):
        self.cpu_offload = True

    def load_models_to_device(self, loadmodel_names=[]):
        for name in loadmodel_names:
            m = getattr(self, name, None)
            if isinstance(m, torch.nn.Module):
                p = next(m.parameters(), None)
                if p is not None and p.device != torch.device(self.device):
                    m.to(self.device)

    def generate_noise(self, shape, seed=None, device="cpu", dtype=torch.float16):
        """reference base.py:140-143 — CPU generator so that seeds reproduce across devices."""
        g = None if seed is None else torch.Generator(device).manual_seed(seed)
        return torch.randn(shape, generator=g, device=device, dtype=dtype)
