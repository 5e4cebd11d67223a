"""Torch stand-ins for the FastBlend entry points (include/svi_b200_fastblend.h) — TEST INFRASTRUCTURE ONLY.

Each function restates what its kernel computes with the oracle's functions (oracle/fastblend_oracle.py), on whatever
device the tensors live, reading and writing the engine's buffers as the kernel does (channel-padded frames, the
double-buffered field and error, the table dtypes).  `install(monkeypatch)` swaps them into diffsynth._native, lifts the
CUDA requirement and places the engine on the CPU, as tests/nv_emulation.py does for the other engines.
"""
import torch

from oracle import fastblend_oracle as O


def fastblend_stage_frames(rgb, out):
    out.zero_()
    out[..., :3] = rgb.float()
    return out


def fastblend_downsample(src, k, out):
    out.zero_()
    out[..., :3] = O.box_down(src[..., :3].contiguous(), k)
    return out


def fastblend_nnf_identity(nnf):
    B, H, W, _ = nnf.shape
    nnf.copy_(O.identity_nnf(B, H, W, nnf.device))
    return nnf


def fastblend_nnf_upscale(src, out):
    B, h, w, _ = src.shape
    out.copy_(O.upscale_nnf(src, 2 * h, 2 * w))
    return out


def fastblend_remap(style, nnf, patch_size, out):
    out.zero_()
    out[..., :3] = O.remap(style[..., :3], nnf, patch_size)
    return out


def fastblend_step(src_guide, src_style, tgt_guide, tgt_style, nnf_in, err_in, nnf_out, err_out, patch_size, mode,
                   guide_weight, dir=0, draw=0, radius=0):
    assert nnf_out.data_ptr() != nnf_in.data_ptr() and (err_in is None or err_in.data_ptr() != err_out.data_ptr())
    cand = nnf_in if mode == 0 else O.neighbour_nnf(nnf_in, dir) if mode == 1 else O.random_nnf(nnf_in, draw, radius)
    e = O.error(src_guide[..., :3], tgt_guide[..., :3], src_style[..., :3], tgt_style[..., :3], cand, patch_size,
                guide_weight)
    if mode == 0:
        nnf_out.copy_(cand)
        err_out.copy_(e)
    else:
        better = e < err_in
        nnf_out.copy_(torch.where(better.unsqueeze(-1), cand, nnf_in))
        err_out.copy_(torch.where(better, e, err_in))


def _typed(t, u8):
    return t[..., :3].to(torch.uint8) if u8 else t[..., :3]


def fastblend_table(op, out, a, sa=0.0, b=None, sb=0.0, c=None, sc=0.0, a_u8=False, b_u8=False, c_u8=False):
    A, B = _typed(a, a_u8), _typed(b, b_u8)
    if op == 0:
        v = A * torch.tensor(O.np.float32(sa)) + B / torch.full_like(B, O.np.float32(sb))
    elif op == 1:
        v = (A.to(torch.float32) + B) / torch.full_like(B, 2.0)
    else:
        v = O.promoted_add(O.scaled(A, sa), O.scaled(B, sb))
        if c is not None:
            v = O.promoted_add(v, O.scaled(_typed(c, c_u8), sc))
    if out.dtype == torch.uint8:
        out.copy_(v.clamp(0, 255).to(torch.uint8))
    else:
        assert v.dtype == out.dtype, (v.dtype, out.dtype)
        out.zero_()
        out[..., :3] = v
    return out


_NAMES = ("fastblend_stage_frames", "fastblend_downsample", "fastblend_nnf_identity", "fastblend_nnf_upscale",
          "fastblend_remap", "fastblend_step", "fastblend_table")


def install(monkeypatch):
    from diffsynth import _native as nv
    from diffsynth.extensions import FastBlend as FB
    for name in _NAMES:
        monkeypatch.setattr(nv, name, globals()[name])
    monkeypatch.setattr(nv, "require_cuda", lambda device, what: None)
    monkeypatch.setattr(FB, "_device", lambda gpu_id: torch.device("cpu"))
