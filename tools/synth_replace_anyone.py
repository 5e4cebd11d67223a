"""Seeded weights and inputs of the UniAnimate-DiT Replace-Anyone fixtures and tests
(tests/golden/make_golden_replace_anyone.py, tests/test_replace_anyone_*.py).

The DiT, the pose stems and the conditioning are those of tools/synth_unianimate.py (a one-layer 5120-wide DiT, since the
reference hard-codes the pose stem's width); this adds the learn-in and inpaint stems, the video and its segmentation,
and the latents that stand in for the VAE encoding of the masked video.
"""
import torch

from tools.synth_unianimate import CFG_5120, _conv_sd  # noqa: F401  (re-exported for the fixtures)

# the fixture's call: 9 frames (3 latent frames) at 64x48, two steps
REPLACE = dict(H=48, W=64, num_frames=9, steps=2, seed=42, ctx_len=16)


def learn_in_sd(seed):
    """Weights of the 4-conv learn-in stem (learn_in_embedding, wan_video.py:1353-1361): keys 0/2/4/6."""
    return _conv_sd([(16, 4, 3, 3, 3)] + [(16, 16, 3, 3, 3)] * 3, seed)


def inpaint_sd(seed):
    """Weights of the 3-conv inpaint stem (inpaint_embedding, wan_video.py:1363-1369): keys 0/2/4."""
    return _conv_sd([(16, 16, 3, 3, 3)] * 3, seed)


def video(T, H, W, seed):
    """[3, T, H, W] f32 in [-1, 1]."""
    return torch.rand(3, T, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def segmentation(T, H, W, seed, dtype=torch.uint8):
    """[1, T, H, W]: about half the pixels 0 (kept), the rest 1 .. 255 (replaced), including 1 and 255."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randint(1, 256, (1, T, H, W), generator=g)
    v[torch.rand(1, T, H, W, generator=g) < 0.5] = 0
    v.view(-1)[:2] = torch.tensor([1, 255])
    return v.to(dtype)


def masked_latents(frames, h, w, seed):
    """[1, 16, frames, h, w] f32: what the fixture's stubbed VAE encoder returns for the masked video."""
    return torch.randn(1, 16, frames, h, w, generator=torch.Generator().manual_seed(seed))
