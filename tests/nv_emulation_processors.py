"""Torch stand-ins for the video processors' entry points (include/svi_b200_processors.h) — TEST INFRASTRUCTURE ONLY.

Each function restates its kernel with oracle/processors_oracle.py on whatever device the tensors live, reading and
writing the processors' buffers as the kernel does.  `install(monkeypatch)` installs these together with the RIFE and
FastBlend stand-ins (tests/nv_emulation_rife.py, tests/nv_emulation_fastblend_modes.py), so a whole processor chain runs
on the CPU.
"""
import numpy as np
import torch

import nv_emulation_fastblend_modes as emu_fb
import nv_emulation_rife as emu_rife
from oracle import processors_oracle as P


def luma_sum_u8(rgb, sums):
    sums.copy_(torch.tensor([P.luma_sum(f) for f in rgb.cpu().numpy()], dtype=torch.int64))
    return sums


def enhance_blend_u8(rgb, degenerate, rate, out):
    d = degenerate.cpu().numpy().astype(np.int32)
    out.copy_(torch.from_numpy(np.stack([P.blend(d[i], f, rate) for i, f in enumerate(rgb.cpu().numpy())])))
    return out


def sharpen_u8(rgb, rate, out):
    assert out.data_ptr() != rgb.data_ptr()
    out.copy_(torch.from_numpy(np.stack([P.sharpness(f, rate) for f in rgb.cpu().numpy()])))
    return out


def rife_average_u8(frames, merged, out):
    x = frames[..., :3].permute(0, 3, 1, 2).cpu()               # B, G, R: rife_oracle.to_tensor's order
    out[1:-1] = torch.from_numpy(P.average_u8(x, merged[..., :3].permute(0, 3, 1, 2).cpu())[1:-1])
    return out


_NAMES = ("luma_sum_u8", "enhance_blend_u8", "sharpen_u8", "rife_average_u8")


def install(monkeypatch):
    from diffsynth import _native as nv
    emu_fb.install(monkeypatch)
    emu_rife.install(monkeypatch)
    for name in _NAMES:
        monkeypatch.setattr(nv, name, globals()[name])
