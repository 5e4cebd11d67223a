"""Torch stand-ins for the kernels the wav2vec2 engine calls — TEST INFRASTRUCTURE ONLY.

Extends tests/nv_emulation.py (whose DiT / VAE stand-ins are reused as they are) with the encoder kernels the audio
engine uses and the four wav2vec2 exports (include/svi_b200.h), restated with torch on whatever device the tensors live on
and rounded to bf16 exactly where the kernel stores bf16.  `install(monkeypatch)` swaps them into diffsynth._native.
"""
import torch
import torch.nn.functional as F

import nv_emulation as base


def layernorm_f32(x, gamma, beta, eps, out):
    out.copy_(F.layer_norm(x, (x.shape[1],), gamma, beta, eps))
    return out


def attention_small(q, k, v, out, num_heads, head_dim, scale, bias_table=None, bucket=None, key_mask=None):
    assert bias_table is None and bucket is None and key_mask is None
    qf, kf, vf = (t.float().reshape(t.shape[0], num_heads, head_dim).transpose(0, 1) for t in (q, k, v))
    o = torch.softmax(qf @ kf.transpose(-1, -2) * scale, dim=-1) @ vf           # fp32 throughout (SIMT kernel)
    out.copy_(o.transpose(0, 1).reshape(q.shape[0], num_heads * head_dim).to(out.dtype))
    return out


def col_stats_workspace_bytes(T, C):
    return 16


def col_stats(x, mean, var, workspace):
    xd = x.double()
    m = xd.mean(dim=0)
    mean.copy_(m.float())
    var.copy_(((xd * xd).mean(dim=0) - m * m).clamp_min(0).float())


def col_norm_act(x, mean, var, eps, gamma, beta, act, out):
    v = (x - mean) * torch.rsqrt(var + eps)
    if gamma is not None:
        v = v * gamma
    if beta is not None:
        v = v + beta
    out.copy_(base._act(v, act).to(out.dtype))
    return out


def conv1d_gather(src, out, kernel, stride, pad_left=0, pad_right=0, col0=0, C=None, split=False):
    T_in = src.shape[0]
    C = src.shape[1] - col0 if C is None else C
    T_out = out.shape[0]
    kpad = out.shape[1] // (2 if split else 1)
    x = F.pad(src[:, col0:col0 + C].float(), (0, 0, pad_left, pad_right))
    idx = torch.arange(T_out).unsqueeze(1) * stride + torch.arange(kernel).unsqueeze(0)       # [T_out, k] padded rows
    cols = x[idx].reshape(T_out, kernel * C)
    out.zero_()
    hi = cols.to(torch.bfloat16)
    out[:, :kernel * C] = hi
    if split:
        out[:, kpad:kpad + kernel * C] = (cols - hi.float()).to(torch.bfloat16)
    assert T_in + pad_left + pad_right - kernel >= (T_out - 1) * stride
    return out


def interp_layernorm(x, T_out, gamma, beta, eps, out):
    y = F.interpolate(x.t().unsqueeze(0), size=T_out, mode="linear", align_corners=True)[0].t()
    out.copy_(F.layer_norm(y, (y.shape[1],), gamma, beta, eps).to(out.dtype))
    return out


_NAMES = ("layernorm_f32", "attention_small", "col_stats_workspace_bytes", "col_stats", "col_norm_act", "conv1d_gather",
          "interp_layernorm")


def install(monkeypatch):
    from diffsynth import _native as nv
    base.install(monkeypatch)
    for name in _NAMES:
        monkeypatch.setattr(nv, name, globals()[name])
