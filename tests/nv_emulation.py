"""Torch stand-ins for the DiT kernels of diffsynth._native — TEST INFRASTRUCTURE ONLY.

The product has no CPU path: every engine starts with `_native.require_cuda`, and every wrapper refuses CPU tensors.
To test the HOST logic of the engines on the CPU-only build box (operation order, buffer aliasing, fused-weight layouts,
the sequence-parallel row bookkeeping under a 2-process gloo group), `install(monkeypatch)` swaps the wrappers of the
module for the functions below, which restate what each kernel computes (include/svi_b200.h) with torch on whatever
device the tensors live on, rounding to bf16 exactly where the kernel stores bf16.  Nothing under
stable-video-infinity_b200/ imports this file.
"""
import torch
import torch.nn.functional as F


def _act(v, act):
    if act == 1:
        # in fp64: torch's fp32 0.5 x (1 + tanh(u)) cancels for x < -2 (a bf16 ulp off in a quarter of those elements, 0 below
        # about -5.5), while the kernels' x * sigmoid(2u) keeps ~1e-6 relative accuracy
        return F.gelu(v.double(), approximate="tanh").to(v.dtype)
    if act == 2:
        return F.silu(v)
    if act == 3:
        return F.gelu(v)
    if act == 4:
        return F.relu(v)
    return v


def gemm(a, w, out, bias=None, act=0, gate=None, residual=None, sumsq=None, sumsq_group_cols=0, ln=None, emit=None):
    v = (a.double() @ w.double().T).float()      # fp64 accumulation, rounded once: independent of the row count / blocking
    if ln is not None:                             # LayerNorm folded into the GEMM: r (acc - mu u), then + c (= bias)
        stats, u, dim, eps = ln
        mean = stats[:, 0:1] / dim
        r = torch.rsqrt((stats[:, 1:2] / dim - mean * mean).clamp_min(0) + eps)
        v = r * (v - mean * u)
    if bias is not None:
        v = v + bias
    v = _act(v, act)
    if sumsq is not None and sumsq.dim() == 3:     # [M, groups, parts]: one STORED partial per 128-column segment
        assert sumsq.shape[2] * 128 == sumsq_group_cols
        for g in range(sumsq.shape[1]):
            for part in range(sumsq.shape[2]):
                c0 = g * sumsq_group_cols + part * 128
                cols = v[:, c0:c0 + 128]
                sumsq[:, g, part] = (cols * cols).sum(dim=1)
    elif sumsq is not None:                        # atomicAdd of the row sum of squares per column group
        for g in range(sumsq.shape[1]):
            cols = v[:, g * sumsq_group_cols:(g + 1) * sumsq_group_cols]
            if cols.numel():
                sumsq[:, g] += (cols * cols).sum(dim=1)
    if gate is not None:
        v = v * gate
    if residual is not None:
        v = v + residual
    if emit is not None:                           # next GEMM's folded operand + row statistics of the final value
        a_next, g_next, row_stats = emit
        a_next.copy_((v * g_next).to(a_next.dtype))
        row_stats[:, 0] += v.sum(dim=1)
        row_stats[:, 1] += (v * v).sum(dim=1)
    out.copy_(v.to(out.dtype))
    return out


def ln_fold_prepare(mods, layers, g_out, rows):
    D = mods.shape[1]
    m = mods[:6 * layers].reshape(layers, 2, 3, D)
    g = 1.0 + m[:, :, 1]
    t = m[:, :, 0]
    g_out.copy_(g)
    gh, th = g.to(torch.bfloat16), t.to(torch.bfloat16)
    rows.copy_(torch.stack([gh, (g - gh.float()).to(torch.bfloat16), th, (t - th.float()).to(torch.bfloat16)], dim=2))


def ln_fold_combine(o4, bias, u, c):
    u.copy_(o4[0] + o4[1])
    c.copy_(o4[2] + o4[3] + (0 if bias is None else bias))


def attention(q, k, v, out, num_heads, scale=None, accumulate=False, workspace=None):
    H, hd = num_heads, q.shape[1] // num_heads
    scale = hd ** -0.5 if scale is None else scale
    qf, kf, vf = (t.float().reshape(t.shape[0], H, hd).transpose(0, 1) for t in (q, k, v))
    s = (qf @ kf.transpose(-1, -2)) * scale
    p = torch.exp(s - s.amax(dim=-1, keepdim=True))
    o = (p.to(torch.bfloat16).float() @ vf) / p.sum(dim=-1, keepdim=True)      # P is consumed as bf16, the row sum in fp32
    o = o.transpose(0, 1).reshape(q.shape[0], H * hd)
    if accumulate:
        o = o + out.float()
    out.copy_(o.to(out.dtype))
    return out


def attention_workspace_bytes(Lq, Lk, num_heads):
    return 0


def _group_sum(ss, g):
    """row sums of squares of group g: [M, groups] or partials [M, groups, parts] added in index order"""
    return ss[:, g] if ss.dim() == 2 else ss[:, g].sum(dim=1)


def attention_qscale(q, k, v, out, num_heads, q_sumsq, q_dim, q_eps, scale=None, accumulate=False, workspace=None):
    hd = q.shape[1] // num_heads
    scale = hd ** -0.5 if scale is None else scale
    rs = torch.rsqrt(_group_sum(q_sumsq, 0) / q_dim + q_eps).unsqueeze(1)
    return attention((q.float() * rs), k, v, out, num_heads, scale, accumulate)     # the factor rides in fp32, q stays bf16


def _split(v, out):
    K = v.shape[1]
    hi = v.to(torch.bfloat16)
    out[:, :K] = hi
    out[:, K:] = (v - hi.float()).to(torch.bfloat16)
    return out


def split_f32_to_bf16x2(src, dst, act=0):
    return _split(_act(src.float(), act), dst)


def layernorm_modulate_split(x, out, eps, gamma=None, beta=None, scale=None, shift=None):
    y = F.layer_norm(x, (x.shape[1],), gamma, beta, eps)
    if scale is not None:
        y = y * (1 + scale)
    if shift is not None:
        y = y + shift
    return _split(y, out)


def qk_norm_rope(qk, sumsq, eps, wq, wk, rope_cos, rope_sin, row_offset=0):
    D = qk.shape[1] // 2
    rmsnorm_rope(qk[:, :D], sumsq, 0, eps, wq, rope_cos, rope_sin, row_offset)
    rmsnorm_rope(qk[:, D:], sumsq, 1, eps, wk, rope_cos, rope_sin, row_offset)
    return qk


def zero_(t):
    return t.zero_()


def layernorm_modulate(x, out, eps, gamma=None, beta=None, scale=None, shift=None):
    y = F.layer_norm(x, (x.shape[1],), gamma, beta, eps)
    if scale is not None:
        y = y * (1 + scale)
    if shift is not None:
        y = y + shift
    out.copy_(y.to(out.dtype))
    return out


def rmsnorm_rope(t, sumsq, sumsq_col, eps, weight, rope_cos=None, rope_sin=None, row_offset=0):
    M, D = t.shape
    rs = torch.rsqrt(_group_sum(sumsq, sumsq_col) / D + eps).unsqueeze(1)
    v = t.float() * rs * weight
    if rope_cos is not None:
        rows = torch.arange(M) + row_offset
        cos = rope_cos[rows].repeat(1, D // 128)                # [M, D/2]: pair p of head h uses table column p
        sin = rope_sin[rows].repeat(1, D // 128)
        re, im = v[:, 0::2], v[:, 1::2]
        v = torch.stack([re * cos - im * sin, re * sin + im * cos], dim=-1).reshape(M, D)
    t.copy_(v.to(t.dtype))
    return t


def patchify_gather(x, y, tokens, split=False):
    src = x if y is None else torch.cat([x, y], dim=0)
    C, Fr, H, W = src.shape
    p = src.reshape(C, Fr, H // 2, 2, W // 2, 2).permute(1, 2, 4, 0, 3, 5).reshape(Fr * (H // 2) * (W // 2), C * 4)
    tokens.zero_()
    hi = p.to(tokens.dtype)
    tokens[:, :C * 4] = hi
    if split:
        kp = tokens.shape[1] // 2
        tokens[:, kp:kp + C * 4] = (p - hi.float()).to(tokens.dtype)
    return tokens


def unpatchify(head_out, out):
    C, Fr, H, W = out.shape
    v = head_out[:, :4 * C].reshape(Fr, H // 2, W // 2, 2, 2, C).permute(5, 0, 1, 3, 2, 4).reshape(C, Fr, H, W)
    out.copy_(v)
    return out


def cfg_euler_step(latents, v_cond, v_uncond, cfg, sigma, sigma_next):
    v = v_cond if v_uncond is None else v_uncond + cfg * (v_cond - v_uncond)
    latents.add_(v * (sigma_next - sigma))
    return latents


def cast_f32_to_bf16(src, dst, act=0):
    dst.copy_(_act(src, act).to(dst.dtype))
    return dst


def cast_bf16_to_f32(src, dst):
    dst.copy_(src.float())
    return dst


def add_rows(table, t, out):
    out.copy_(table + t.repeat(table.shape[0] // t.shape[0], 1))
    return out


def axpby(a, alpha, b, beta, out):
    out.copy_(alpha * a + beta * b)
    return out


# ---------------------------------------------------------------------------------------------- VAE kernels
def vae_norm_act(x, n_pix, C, ldx, gamma, silu, out, Cpad):
    v = torch.as_strided(x, (n_pix, C), (ldx, 1)).float()
    if gamma is not None:
        v = v / v.norm(dim=1, keepdim=True).clamp_min(1e-12) * (C ** 0.5) * gamma
    if silu:
        v = F.silu(v)
    o = out.reshape(-1, Cpad)[:n_pix]            # `out` is contiguous and may have more rows than n_pix (padded work buffers)
    o[:, :C] = v.to(o.dtype)
    o[:, C:] = 0
    return out


def vae_upsample2x(x, H, W, C, out):
    out.copy_(x.repeat_interleave(2, 0).repeat_interleave(2, 1).to(out.dtype))
    return out


def vae_space_to_depth(x, H, W, C, out):
    # y[h, w, (dy*2 + dx)*C + c] = x[2h+dy, 2w+dx, c]
    out.copy_(x.view(H // 2, 2, W // 2, 2, C).permute(0, 2, 1, 3, 4).reshape(H // 2, W // 2, 4 * C).to(out.dtype))
    return out


def vae_space_to_depth_act(x, H, W, C, act, out):
    return vae_space_to_depth(_act(x.float(), act), H, W, C, out)


def vae_from_planar(x, C, n_pix, scale, shift, out, ldo, out_is_bf16, ldc=None):
    v = x.reshape(C, n_pix).t().float()
    if scale is not None:
        v = v * scale
    if shift is not None:
        v = v + shift
    o = out.view(n_pix, ldo)
    o[:, :C] = v.to(o.dtype)
    o[:, C:] = 0
    return out


def vae_to_planar(x, ldx, C, n_pix, pre_shift, scale, clamp, out, ldc=None):
    v = x[:, :C].float()
    if pre_shift is not None:
        v = v + pre_shift
    if scale is not None:
        v = v * scale
    if clamp:
        v = v.clamp(-1, 1)
    out.view(C, n_pix).copy_(v.t())
    return out


def softmax_rows(s, N, scale, p):
    p.zero_()
    p[:, :N] = torch.softmax(s[:, :N].float() * scale, dim=1).to(p.dtype)
    return p


def _mem(ptr, n, dtype):
    """n elements of `dtype` at the raw (host) address `ptr` as a tensor sharing that memory: the conv descriptor carries
    pointers, exactly as the C ABI receives them."""
    import ctypes
    size = {torch.float32: 4, torch.bfloat16: 2}[dtype]
    buf = (ctypes.c_char * (n * size)).from_address(ptr)
    return torch.frombuffer(buf, dtype=dtype)


def conv3d_causal(d):
    """svi_conv3d_causal on host memory (include/svi_b200.h): implicit GEMM over the frame ring with the (output frame, k_t) ->
    slot table, zero fill outside the ring frame (TMA out-of-bounds), bias / residual / channel->frame split, and the fused
    producer of the next conv's input (RMS norm + SiLU -> bf16 ring)."""
    kt, kh, kw, H, W, T = d.kt, d.kh, d.kw, d.H, d.W, d.T
    Ci, Co = d.C_in, d.C_out
    cpad = (Ci + 63) // 64 * 64
    ring = _mem(d.x_ring, d.ring_slots * d.in_H * d.in_W * Ci, torch.bfloat16).view(d.ring_slots, d.in_H, d.in_W, Ci)
    wp = _mem(d.w_packed, d.w_rows * d.w_ld, torch.bfloat16).view(d.w_rows, d.w_ld)[:Co, :kt * kh * kw * cpad]
    w = wp.float().view(Co, kt, kh, kw, cpad)[..., :Ci].permute(0, 4, 1, 2, 3).contiguous()       # [Co, Ci, kt, kh, kw]
    bias = _mem(d.bias, Co, torch.float32) if d.bias else None
    gamma = _mem(d.next_gamma, Co, torch.float32) if d.next_gamma else None
    write_f32 = d.write_f32 if d.next_ring else 1
    for t in range(T):
        # input window: rows h + b - pad_h, columns w + c - pad_w; zero where that leaves the ring frame
        x = torch.zeros(kt, H + kh - 1, W + kw - 1, Ci)
        for a in range(kt):
            fr = ring[d.slot[t * 3 + a]].float()
            for i in range(H + kh - 1):
                si = i - d.pad_h
                if 0 <= si < d.in_H:
                    j0, j1 = max(0, d.pad_w), min(W + kw - 1, d.in_W + d.pad_w)
                    x[a, i, j0:j1] = fr[si, j0 - d.pad_w:j1 - d.pad_w]
        # fp64 accumulation, rounded once: the value of a pixel must not depend on how the CPU library blocks a frame of this size
        # (a band of rows vs the whole frame under spatial sharding), as it does not on the GPU
        v = F.conv3d(x.double().permute(3, 0, 1, 2).unsqueeze(0), w.double())[0, :, 0].permute(1, 2, 0).float()   # [H, W, Co]
        if bias is not None:
            v = v + bias
        if d.residual:
            res = _mem(d.residual + 4 * t * d.res_frame_stride, H * W * d.res_ld, torch.float32).view(H, W, d.res_ld)
            v = v + res[..., :Co]
        if write_f32:
            if d.n_split > 0:
                o0 = _mem(d.out + 4 * t * d.out_frame_stride, H * W * d.out_ld, torch.float32).view(H, W, d.out_ld)
                o1 = _mem(d.out + 4 * (d.split_offset + t * d.out_frame_stride), H * W * d.out_ld, torch.float32).view(H, W, d.out_ld)
                o0[..., :d.n_split] = v[..., :d.n_split]
                o1[..., :Co - d.n_split] = v[..., d.n_split:]
            else:
                o = _mem(d.out + 4 * t * d.out_frame_stride, H * W * d.out_ld, torch.float32).view(H, W, d.out_ld)
                o[..., :Co] = v
        if d.next_ring:
            y = v
            if gamma is not None:
                y = y / y.norm(dim=2, keepdim=True).clamp_min(1e-12) * (Co ** 0.5) * gamma
            if d.next_silu:
                y = F.silu(y)
            nr = _mem(d.next_ring + 2 * d.next_slot[t] * d.next_frame_stride, H * W * d.next_ld, torch.bfloat16).view(H, W, d.next_ld)
            nr[..., :Co] = y.to(torch.bfloat16)
    return 0


_NAMES = ("gemm", "attention", "attention_workspace_bytes", "attention_qscale", "layernorm_modulate", "layernorm_modulate_split",
          "rmsnorm_rope", "qk_norm_rope", "patchify_gather", "unpatchify", "cfg_euler_step", "cast_f32_to_bf16",
          "cast_bf16_to_f32", "split_f32_to_bf16x2", "zero_", "add_rows", "axpby", "ln_fold_prepare", "ln_fold_combine",
          "vae_norm_act", "vae_upsample2x", "vae_space_to_depth", "vae_space_to_depth_act", "vae_from_planar", "vae_to_planar", "softmax_rows", "conv3d_causal")


def install(monkeypatch=None):
    """Replace the wrappers of diffsynth._native by the functions above and lift the CUDA requirement.  With pytest's
    monkeypatch the change is undone after the test; without (spawned worker processes) it stays for the process."""
    from diffsynth import _native as nv
    put = (lambda n, v: monkeypatch.setattr(nv, n, v)) if monkeypatch is not None else (lambda n, v: setattr(nv, n, v))
    for name in _NAMES:
        put(name, globals()[name])
    put("require_cuda", lambda device, what: None)
    put("load", lambda: None)
