"""Torch stand-ins for the FastBlend modes' entry points (include/svi_b200_fastblend_modes.h) — TEST INFRASTRUCTURE ONLY.

Each function restates its kernel with the oracles' functions (oracle/fastblend_oracle.py, oracle/fastblend_modes_oracle.py)
on whatever device the tensors live, reading and writing the engine's buffers as the kernel does.  `install(monkeypatch)`
installs these together with tests/nv_emulation_fastblend.py's stand-ins, so the whole engine runs on the CPU.
"""
import numpy as np
import torch

import nv_emulation_fastblend as emu
from oracle import fastblend_modes_oracle as M
from oracle import fastblend_oracle as O


def fastblend_candidate(nnf_in, nnf_out, mode, dir=0, draw=0, radius=0, shift=0, pairwise=False):
    assert nnf_out.data_ptr() != nnf_in.data_ptr()
    if mode == 1:
        nnf_out.copy_(O.neighbour_nnf(nnf_in, dir))
    elif mode == 2:
        nnf_out.copy_(O.random_nnf(nnf_in, draw, radius))
    else:
        nnf_out.copy_(M.track_nnf(nnf_in, shift, pairwise))
    return nnf_out


def fastblend_select(src_guide, src_style, tgt_guide, tgt_style, cand, nnf_in, err_in, nnf_out, err_out, patch_size,
                     guide_weight, pairwise=False):
    assert nnf_out.data_ptr() not in (cand.data_ptr(), None if nnf_in is None else nnf_in.data_ptr())
    sg, ss, tg = src_guide[..., :3], src_style[..., :3], tgt_guide[..., :3]
    if pairwise:
        gw = torch.tensor(np.float32(guide_weight), device=sg.device)
        e = M.guide_error(sg, tg, cand, patch_size) * gw + M.pairwise_style_error(ss, cand, patch_size)
    else:
        ts = tgt_style[..., :3].expand_as(ss).contiguous()
        e = O.error(sg, tg, ss, ts, cand, patch_size, guide_weight)
    if nnf_in is None:
        nnf_out.copy_(cand)
        err_out.copy_(e)
    else:
        better = e < err_in
        nnf_out.copy_(torch.where(better.unsqueeze(-1), cand, nnf_in))
        err_out.copy_(torch.where(better, e, err_in))


def fastblend_batch_mean(src, out):
    out.copy_(M.batch_mean(src))
    out[..., 3] = 0
    return out


def fastblend_running_mean(frame, s, result, divisor, out, frame_u8=False):
    f = frame.to(torch.uint8) if frame_u8 else frame
    out.copy_(f.double() * s + (result / torch.full_like(result, np.float32(divisor))).double())
    out[..., 3] = 0
    return out


def fastblend_to_u8(a, out, a_u8=False):
    out.copy_(a[..., :3].clamp(0, 255).to(torch.uint8))
    return out


_NAMES = ("fastblend_candidate", "fastblend_select", "fastblend_batch_mean", "fastblend_running_mean", "fastblend_to_u8")


def install(monkeypatch):
    from diffsynth import _native as nv
    emu.install(monkeypatch)
    for name in _NAMES:
        monkeypatch.setattr(nv, name, globals()[name])
