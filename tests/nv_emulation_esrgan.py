"""Torch stand-ins for the ESRGAN entry points (include/svi_b200_esrgan.h) — TEST INFRASTRUCTURE ONLY.

Each function restates what its kernel computes, on whatever device the tensors live.  The convolution runs in fp64 from
the packed weight (so the host-side packing is checked, not assumed) and reads the launch as its descriptor states it:
the input pitch in_ld and channel count C_in of x's view, the bf16 destination's pitch and channel offset, and bf_up2.
`install(monkeypatch)` swaps them into diffsynth._native and lifts the CUDA requirement, as tests/nv_emulation.py does
for the other engines.
"""
import torch
import torch.nn.functional as F


def esrgan_stage_frames(rgb, out):
    out.zero_()
    out[..., :3] = (rgb.float() / 255).to(out.dtype)
    return out


def _pixels(t):
    """a channel-window view of a [N, H, W, pitch] buffer, widened to the end of the pixel"""
    ld = t.stride(2)
    return torch.as_strided(t, (*t.shape[:3], ld - t.storage_offset() % ld), t.stride())


def esrgan_conv2d(x, w, C_out, bias, tile_w, slope=0.0, residual=None, res_scale=1.0, residual2=None, res2_scale=1.0,
                  out=None, out_bf16=None, bf_up2=False, out_u8=None):
    N, H, W, C_in = x.shape
    cpad = (C_in + 63) // 64 * 64
    xin = _pixels(x)[..., :C_in].double().permute(0, 3, 1, 2)
    xin = F.pad(xin, (1, 1, 1, 1, 0, cpad - C_in))
    wk = w[:C_out, :9 * cpad].double().reshape(C_out, 3, 3, cpad).permute(0, 3, 1, 2)
    v = F.conv2d(xin, wk).permute(0, 2, 3, 1) + bias[:C_out].double()
    if slope:
        v = torch.where(v > 0, v, v * slope)
    if residual is not None:
        v = v * res_scale + residual[..., :C_out].double()
    if residual2 is not None:
        v = v * res2_scale + residual2[..., :C_out].double()
    if out is not None:
        out[..., :C_out] = v.to(out.dtype)
    if out_bf16 is not None:
        up = v.repeat_interleave(2, 1).repeat_interleave(2, 2) if bf_up2 else v
        _pixels(out_bf16)[..., :C_out] = up.to(out_bf16.dtype)
    if out_u8 is not None:
        out_u8.copy_((v[..., :3].float() * 255).clamp(0, 255).to(torch.uint8))


_NAMES = ("esrgan_stage_frames", "esrgan_conv2d")


def install(monkeypatch):
    from diffsynth import _native as nv
    for name in _NAMES:
        monkeypatch.setattr(nv, name, globals()[name])
    monkeypatch.setattr(nv, "require_cuda", lambda device, what: None)
