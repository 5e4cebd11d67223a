"""Torch stand-ins for the cross-attention scorers' entry points (include/svi_b200_reward.h) — TEST INFRASTRUCTURE ONLY.

Each function restates what its kernel computes, rounding to bf16 where the kernel stores bf16.  `install(monkeypatch)`
adds them to the quality stand-ins of tests/nv_emulation_quality.py, so the ImageReward and MPS engines run end to end
on the CPU.
"""
import torch
import torch.nn.functional as F

import nv_emulation_quality


def reward_attn(q, k, v, out, batch, num_heads, scale, kv_heads=None, kv_shared=False, key_mask=None):
    kv_heads = num_heads if kv_heads is None else kv_heads
    Lq = q.shape[0] // batch
    Lk = k.shape[0] if kv_shared else k.shape[0] // batch
    Q = q[:, :num_heads * 64].double().reshape(batch, Lq, num_heads, 64).transpose(1, 2)
    kb = 1 if kv_shared else batch
    K, V = (t[:, :kv_heads * 64].double().reshape(kb, Lk, kv_heads, 64).transpose(1, 2) for t in (k, v))
    s = (Q @ K.transpose(-1, -2)) * scale
    if key_mask is not None:
        keep = key_mask.reshape(-1, Lk).bool()[:, None, None, :]
        s = s.masked_fill(~keep, float("-inf"))
    o = (s.softmax(-1) @ V).transpose(1, 2).reshape(batch * Lq, num_heads * 64)
    out[:, :num_heads * 64] = o.to(out.dtype)
    return out


def reward_layernorm(x, gamma, beta, eps, y, yb):
    v = F.layer_norm(x, (x.shape[1],), gamma, beta, eps)
    y.copy_(v)
    yb.copy_(v.to(yb.dtype))
    return y, yb


def reward_embed(patch, cls, pos, out):
    n, D = pos.shape[0] - 1, pos.shape[1]
    B = patch.shape[0] // n
    out.copy_((torch.cat([cls.view(1, 1, D).expand(B, 1, D), patch.view(B, n, D)], 1) + pos).reshape(-1, D))
    return out


def reward_swiglu(x, out):
    a, g = x.chunk(2, -1)
    out.copy_((F.silu(g) * a).to(out.dtype))
    return out


def reward_rope(x, L, cos, sin):
    M, W = x.shape
    t = x.float().reshape(M, W // 64, 2, 32)
    c, s = cos[torch.arange(M) % L][:, None], sin[torch.arange(M) % L][:, None]
    t1, t2 = t[:, :, 0], t[:, :, 1]
    x.copy_(torch.stack([t1 * c + (-t2) * s, t2 * c + t1 * s], 2).reshape(M, W).to(x.dtype))
    return x


def reward_cond_mask(text, cond, threshold, ratio, keep):
    sim = (text.double() @ cond.double().T).max(-1).values.float()
    ratio.copy_(sim / sim.max())
    keep.copy_(ratio > threshold)
    return ratio, keep


def reward_head(x, n_seq, w, bias, out):
    L = x.shape[0] // n_seq
    out.copy_(x[::L].double() @ w.double() + bias)
    return out


NAMES = ("reward_attn", "reward_layernorm", "reward_embed", "reward_swiglu", "reward_rope", "reward_cond_mask",
         "reward_head")


def install(monkeypatch=None):
    from diffsynth import _native as nv
    nv_emulation_quality.install(monkeypatch)
    put = (lambda n, v: monkeypatch.setattr(nv, n, v)) if monkeypatch is not None else (lambda n, v: setattr(nv, n, v))
    for name in NAMES:
        put(name, globals()[name])
