"""Seeded weights and inputs of the UniAnimate-DiT fixtures and tests (tests/golden/make_golden_unianimate.py,
tests/test_unianimate_*.py).

The reference hard-codes the pose stem's width to 5120 (pipelines/wan_video.py:541), so the fixture's DiT is a
one-layer model of that width (``CFG_5120``) with a small FFN; the native tests use any width through the checkpoint.
"""
import numpy as np
import torch

CFG_5120 = dict(has_image_input=True, patch_size=(1, 2, 2), in_dim=36, dim=5120, ffn_dim=256, freq_dim=64, text_dim=96,
                out_dim=16, num_heads=40, num_layers=1, eps=1e-6)

# the fixture's long-video call: 9 latent frames in windows of 5 overlapping by 2 -> starts 0, 3 and 4 (the third window
# [6, 7, 8, 0, 1] realigned to [4 .. 8])
LONG = dict(H=48, W=64, num_frames=33, context_size=5, context_overlap=2, steps=2, cfg_scale=5.0, seed=42, ctx_len=16)


def _conv_sd(shapes, seed):
    """Keys '0.weight', '0.bias', '2.weight', ... (an nn.Sequential with SiLU between the convs), drawn in that order:
    weights ~ N(0, 1.5^2 / fan_in) rounded to bf16, biases ~ N(0, 0.01)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, shape in enumerate(shapes):
        sd[f"{2 * i}.weight"] = (torch.randn(shape, generator=g) * (1.5 / np.prod(shape[1:]) ** 0.5)).to(torch.bfloat16).float()
        sd[f"{2 * i}.bias"] = torch.randn(shape[0], generator=g) * 0.1
    return sd


def pose_stem_sd(dim, seed):
    """Weights of the 7-conv pose stem (dwpose_embedding, svi_video_dance.py:256-268) with output width `dim`."""
    return _conv_sd([(16, 3, 3, 3, 3)] + [(16, 16, 3, 3, 3)] * 5 + [(dim, 16, 1, 2, 2)], seed)


def ref_stem_sd(seed):
    """Weights of the 6-conv reference-pose stem (randomref_embedding_pose, wan_video.py:544-558)."""
    return _conv_sd([(16, 3, 3, 3)] + [(16, 16, 3, 3)] * 4 + [(20, 16, 3, 3)], seed)


def pose_video(T, H, W, seed):
    """[3, T, H, W] in 0..255 (float)."""
    return torch.randint(0, 256, (3, T, H, W), generator=torch.Generator().manual_seed(seed)).float()


def ref_pose(H, W, seed):
    """[H, W, 3] in 0..255 (float)."""
    return torch.randint(0, 256, (H, W, 3), generator=torch.Generator().manual_seed(seed)).float()


def conditioning(cfg, frames, h, w, ctx_len, seed):
    """Fixed prompt embeddings (positive, negative), CLIP feature and image condition y [1, 20, frames, h, w]."""
    g = torch.Generator().manual_seed(seed)
    pos = torch.randn(1, ctx_len, cfg["text_dim"], generator=g)
    neg = torch.randn(1, ctx_len, cfg["text_dim"], generator=g)
    clip = torch.randn(1, 257, 1280, generator=g)
    y = torch.randn(1, 20, frames, h, w, generator=g) * 0.5
    return pos, neg, clip, y


def dummy_image(H, W):
    from PIL import Image
    return Image.fromarray(np.zeros((H, W, 3), dtype=np.uint8))
