"""Torch stand-ins for the RIFE entry points (include/svi_b200_rife.h) — TEST INFRASTRUCTURE ONLY.

Each function restates what its kernel computes, on whatever device the tensors live: the convolution in fp64 from the
packed weight (so the host-side packing is checked, not assumed), the resizes with the kernels' ATen source-index
formula, the warp with F.grid_sample.  `install(monkeypatch)` swaps them into diffsynth._native and lifts the CUDA
requirement, as tests/nv_emulation.py does for the other engines.
"""
import torch
import torch.nn.functional as F


def rife_stage_frames(rgb, out):
    v = rgb.reshape(-1, 3).float() / 255
    o = out.view(-1, 4)
    o[:, :3] = v[:, [2, 1, 0]]
    o[:, 3] = 0
    return out


def _taps(n_out, scale, n_in, device):
    d = torch.arange(n_out, device=device, dtype=torch.float32)
    r = (torch.tensor(scale, dtype=torch.float32) * (d + 0.5) - 0.5).clamp_min(0)
    i0 = r.long()
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = r - i0.float()
    return i0, i1, 1 - l1, l1


def resize(x, h, w, scale):
    """bilinear resize of channels-last [n, H, W, C] with the kernels' source-index formula"""
    y0, y1, a0, a1 = _taps(h, scale, x.shape[1], x.device)
    x0, x1, b0, b1 = _taps(w, scale, x.shape[2], x.device)
    r0, r1 = x[:, y0], x[:, y1]
    b0, b1 = b0.view(1, 1, -1, 1), b1.view(1, 1, -1, 1)
    top = b0 * r0[:, :, x0] + b1 * r0[:, :, x1]
    bot = b0 * r1[:, :, x0] + b1 * r1[:, :, x1]
    return a0.view(1, -1, 1, 1) * top + a1.view(1, -1, 1, 1) * bot


def _state(img0, img1, state):
    if state is not None:
        return state
    P, H, W, _ = img0.shape
    s = torch.zeros(P, H, W, 12, device=img0.device)
    s[..., 0:3], s[..., 3:6] = img0[..., :3], img1[..., :3]
    return s


def rife_block_input(img0, img1, state, h, w, src_scale, flow_mul, out):
    v = resize(_state(img0, img1, state), h, w, float(src_scale))
    fl = v[..., 8:12] * float(flow_mul)
    d0 = torch.cat([v[..., 0:3], v[..., 3:6], v[..., 6:7], fl], -1)
    d1 = torch.cat([v[..., 3:6], v[..., 0:3], -v[..., 6:7], fl[..., 2:4], fl[..., 0:2]], -1)
    x = torch.cat([d0, d1], 0)                                                   # [2P, h, w, 11]
    n = x.shape[0]
    s2d = x.reshape(n, h // 2, 2, w // 2, 2, 11).permute(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 44)
    out.zero_()
    out[..., :44] = s2d.to(out.dtype)
    return out


def rife_conv2d(x, w, kh, kw, pad, C_out, phase_cols, bias, tile_w, prelu=None, residual=None, out=None, out_bf16=None,
                bf_s2d=False):
    N, H, W, C_in = x.shape
    cpad = (C_in + 63) // 64 * 64
    wk = w[:C_out, :kh * kw * cpad].double().reshape(C_out, kh, kw, cpad).permute(0, 3, 1, 2)
    xin = F.pad(x.double().permute(0, 3, 1, 2), (pad, kw - 1 - pad, pad, kh - 1 - pad))
    xin = F.pad(xin, (0, 0, 0, 0, 0, cpad - C_in))
    v = F.conv2d(xin, wk).permute(0, 2, 3, 1) + bias[:C_out].double()          # [N, H, W, C_out]
    if prelu is not None:
        a = prelu[:C_out].double()
        v = torch.where(v > 0, v, v * a)
    phases = C_out // phase_cols
    if phases == 4:
        v = v.reshape(N, H, W, 2, 2, phase_cols).permute(0, 1, 3, 2, 4, 5).reshape(N, 2 * H, 2 * W, phase_cols)
    if residual is not None:
        v = v + residual[..., :phase_cols].double()
    if out is not None:
        out[..., :phase_cols] = v.to(out.dtype)
    if out_bf16 is not None:
        if bf_s2d:
            n, Hd, Wd, c = v.shape
            v = v.reshape(n, Hd // 2, 2, Wd // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, Hd // 2, Wd // 2, 4 * c)
        out_bf16[..., :v.shape[-1]] = v.to(out_bf16.dtype)


def _warp(img, flow):
    P, H, W, _ = flow.shape
    gx = torch.linspace(-1.0, 1.0, W, device=img.device).view(1, 1, W).expand(P, H, W)
    gy = torch.linspace(-1.0, 1.0, H, device=img.device).view(1, H, 1).expand(P, H, W)
    g = torch.stack([gx + flow[..., 0] / ((W - 1.0) / 2.0), gy + flow[..., 1] / ((H - 1.0) / 2.0)], -1)
    out = F.grid_sample(img[..., :3].permute(0, 3, 1, 2), g, mode="bilinear", padding_mode="border", align_corners=True)
    return out.permute(0, 2, 3, 1)


def rife_update_warp(heads, src_scale, flow_mul, img0, img1, state, first, merged=None, clip=False, rgb=None):
    P, H, W, _ = img0.shape
    up = resize(heads[..., :5], H, W, float(src_scale))
    f0, f1 = up[:P, ..., :4] * float(flow_mul), up[P:, ..., :4] * float(flow_mul)
    m0, m1 = up[:P, ..., 4], up[P:, ..., 4]
    flow = torch.zeros(P, H, W, 4, device=img0.device) if first else state[..., 8:12].clone()
    mask = torch.zeros(P, H, W, device=img0.device) if first else state[..., 6].clone()
    flow = flow + (f0 + torch.cat([f1[..., 2:4], f1[..., 0:2]], -1)) / 2
    mask = mask + (m0 + (-m1)) / 2
    w0, w1 = _warp(img0, flow[..., 0:2]), _warp(img1, flow[..., 2:4])
    state[..., 0:3], state[..., 3:6], state[..., 6], state[..., 7], state[..., 8:12] = w0, w1, mask, 0, flow
    sg = torch.sigmoid(mask)[..., None]
    m = w0 * sg + w1 * (1 - sg)
    if merged is not None:
        merged[..., :3] = m.clamp(0, 1) if clip else m
        merged[..., 3:4] = sg
    if rgb is not None:
        rgb.copy_((m[..., [2, 1, 0]] * 255).clamp(0, 255).to(torch.uint8))


_NAMES = ("rife_stage_frames", "rife_block_input", "rife_conv2d", "rife_update_warp")


def install(monkeypatch):
    from diffsynth import _native as nv
    for name in _NAMES:
        monkeypatch.setattr(nv, name, globals()[name])
    monkeypatch.setattr(nv, "require_cuda", lambda device, what: None)
