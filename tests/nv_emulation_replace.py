"""Torch stand-in for the Replace-Anyone staging kernel of diffsynth._native (include/svi_b200_replace.h) — TEST
INFRASTRUCTURE ONLY.  `install(monkeypatch)` adds it to the UniAnimate, DiT, VAE and conv stand-ins, so the Replace-Anyone
pipeline runs end to end on the CPU."""
import torch

import nv_emulation_unianimate


def replace_mask_stage(video, seg, masked, ring):
    keep = (~(seg / 255. > 0)).float()
    m = video * keep
    if masked is not None:
        masked.copy_(m)
    ring[..., :3] = m.permute(1, 2, 3, 0).to(ring.dtype)
    ring[..., 3] = keep.to(ring.dtype)
    return masked, ring


def install(monkeypatch=None):
    from diffsynth import _native as nv
    nv_emulation_unianimate.install(monkeypatch)
    put = (lambda n, v: monkeypatch.setattr(nv, n, v)) if monkeypatch is not None else (lambda n, v: setattr(nv, n, v))
    put("replace_mask_stage", replace_mask_stage)
