"""Kernel-level GPU checks with verbose diagnostics (development tool; the pytest -m gpu suite is the gate).

usage: python tools/gpu_check.py <section> [...]   sections: every sec_<name> below, e.g. gemm gemm_edges attn attn_online
       attn_sp_one_gpu conv conv_tiles ew perf_gemm perf_attn
Each section prints one line per case: name, max abs err, reference scale, verdict.  A "negative control" case passes when
a wrong but plausible reference fails the bar, i.e. when the bar is sharp enough to tell the two apart.
"""
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "stable-video-infinity_b200"))
from diffsynth import _native as nv  # noqa: E402

dev = "cuda"
RESULTS = []   # (name, ok) of every report() call — tests/test_kernels_gpu.py asserts on it


def _bar(got, ref, tol, min_inside):
    """(ok, max err, max |ref|, fraction inside the elementwise tolerance, err) of report()'s bar"""
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    mx = err.max().item()
    scale = ref.abs().max().item()
    rms = ref.pow(2).mean().sqrt().item()
    inside = (err <= 1e-3 * rms + 1e-2 * ref.abs()).float().mean().item()
    ok = math.isfinite(mx) and mx <= tol * max(scale, 1e-6) and (min_inside is None or inside >= min_inside)
    return ok, mx, scale, inside, err


def negative(name, got, wrong, tol, min_inside=None):
    """Negative control of report(): a wrong but plausible reference must FAIL the same bar (recorded as a case)."""
    ok_wrong, mx, _, inside, _ = _bar(got, wrong, tol, min_inside)
    print(f"[{'BAD' if ok_wrong else 'OK '}] negative control {name}: the wrong reference "
          f"{'passes' if ok_wrong else 'fails'} the bar (max_err={mx:.4e} inside={inside:.4f})", flush=True)
    RESULTS.append((f"negative control {name}", not ok_wrong))


def report(name, got, ref, tol, min_inside=None):
    """Max-norm criterion (err <= tol * max|ref|) and, when min_inside is given, the elementwise criterion of the north
    star as well: the fraction of elements with err <= 1e-3 * rms(ref) + 1e-2 * |ref| must reach min_inside (atol is taken
    relative to the reference's rms so that the bar means the same for unit-scale and for 1/sqrt(L)-scale outputs)."""
    got = got.float()
    ref = ref.float()
    ok, mx, scale, inside, err = _bar(got, ref, tol, min_inside)
    bad = (err > tol * max(scale, 1e-6)).float().mean().item()
    print(f"[{'OK ' if ok else 'BAD'}] {name}: max_err={mx:.4e} ref_max={scale:.4e} frac_bad={bad:.4f} "
          f"inside(rtol 1e-2, atol 1e-3 rms)={inside:.4f}", flush=True)
    RESULTS.append((name, ok))
    if not ok:
        # locate the error pattern to help debugging descriptor/layout mistakes
        idx = (err > tol * max(scale, 1e-6)).nonzero()
        if idx.numel():
            rows = idx[:, 0].unique()
            cols = idx[:, 1].unique() if idx.shape[1] > 1 else idx[:, 0]
            print(f"      bad rows: n={rows.numel()} first={rows[:8].tolist()} | bad cols: n={cols.numel()} first={cols[:16].tolist()}")
            r0, c0 = idx[0, 0].item(), (idx[0, 1].item() if idx.shape[1] > 1 else 0)
            print(f"      sample got={got[r0, c0:c0+4].tolist()} ref={ref[r0, c0:c0+4].tolist()}")
    return ok


def time_ms(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s = torch.cuda.Event(enable_timing=True)
    e = torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def sec_gemm():
    g = torch.Generator(device="cpu").manual_seed(0)
    for (M, N, K) in [(128, 256, 64), (128, 256, 256), (256, 512, 128), (100, 64, 64), (1, 1536, 256),
                      (3200, 1536, 1536), (333, 4608, 1536), (512, 1536, 4096), (777, 8960, 1536), (640, 1536, 8960),
                      (130, 264, 72)]:
        a = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
        w = (torch.randn(N, K, generator=g) * 0.5).to(dev, torch.bfloat16)
        out = torch.full((M, N), float("nan"), device=dev, dtype=torch.float32)
        nv.gemm(a, w, out)
        torch.cuda.synchronize()
        ref = a.float() @ w.float().t()
        report(f"gemm f32out M={M} N={N} K={K}", out, ref, 2e-3)


def sec_gemm_epi():
    g = torch.Generator(device="cpu").manual_seed(1)
    M, N, K = 300, 1536, 512
    a = (torch.randn(M, K, generator=g) * 0.3).to(dev, torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.1).to(dev, torch.bfloat16)
    bias = torch.randn(N, generator=g).to(dev)
    gate = torch.randn(N, generator=g).to(dev)
    res = torch.randn(M, N, generator=g).to(dev)
    acc = a.float() @ w.float().t()
    # bf16 out + bias + gelu
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    nv.gemm(a, w, out, bias=bias, act=nv.ACT_GELU_TANH)
    report("epi bias+gelu_tanh bf16", out, torch.nn.functional.gelu(acc + bias, approximate="tanh"), 1e-2)
    nv.gemm(a, w, out, bias=bias, act=nv.ACT_SILU)
    report("epi bias+silu bf16", out, torch.nn.functional.silu(acc + bias), 1e-2)
    nv.gemm(a, w, out, bias=bias, act=nv.ACT_GELU_ERF)
    report("epi bias+gelu_erf bf16", out, torch.nn.functional.gelu(acc + bias), 1e-2)
    # f32 out, gate, residual in place
    x = res.clone()
    nv.gemm(a, w, x, bias=bias, gate=gate, residual=x)
    report("epi bias+gate+residual(in place) f32", x, res + gate * (acc + bias), 2e-3)
    # sumsq with 3 groups of 512 columns, 2 accumulated; output into a column-slice view (ld > N)
    big = torch.zeros(M, 2 * N, device=dev, dtype=torch.bfloat16)
    ss = torch.zeros(M, 2, device=dev, dtype=torch.float32)
    nv.gemm(a, w, big[:, N:], bias=bias, sumsq=ss, sumsq_group_cols=512)
    v = acc + bias
    report("epi strided bf16 out", big[:, N:], v, 1e-2)
    report("epi strided untouched half", big[:, :N], torch.zeros_like(v), 1e-6)
    ref_ss = torch.stack([(v[:, :512] ** 2).sum(1), (v[:, 512:1024] ** 2).sum(1)], dim=1)
    report("epi sumsq", ss, ref_ss, 2e-3)


def sec_ln_fold():
    """LayerNorm folded into the GEMM: producer (a_next = bf16(v * g), row statistics) and consumer
    (r (acc - mu u) + c) against the explicit LayerNorm -> modulate -> Linear in fp32."""
    g = torch.Generator(device="cpu").manual_seed(21)
    for (M, d, N) in [(300, 1536, 4608), (1000, 256, 512), (777, 1536, 1536), (100, 256, 512)]:     # M <= 128: one row tile
        x0 = (torch.randn(M, d, generator=g) * 1.5 + 0.2).to(dev)
        a = (torch.randn(M, 512, generator=g) * 0.3).to(dev, torch.bfloat16)
        wo = (torch.randn(d, 512, generator=g) * 0.05).to(dev, torch.bfloat16)
        bo, gate = torch.randn(d, generator=g).to(dev) * 0.1, torch.randn(d, generator=g).to(dev)
        gmod = (1 + 0.1 * torch.randn(d, generator=g)).to(dev)
        tmod = (0.1 * torch.randn(d, generator=g)).to(dev)
        # producer: x = x0 + gate * (a wo^T + bo), emits bf16(x * gmod) and (sum x, sum x^2)
        x = x0.clone()
        a_next = torch.full((M, d), float("nan"), device=dev, dtype=torch.bfloat16)
        stats = torch.zeros(M, 2, device=dev)
        nv.gemm(a, wo, x, bias=bo, gate=gate, residual=x, emit=(a_next, gmod, stats))
        x_ref = x0 + gate * (a.float() @ wo.float().t() + bo)
        report(f"fold producer out M={M} d={d}", x, x_ref, 2e-3)
        report(f"fold producer a_next M={M} d={d}", a_next, x_ref * gmod, 6e-3)
        report(f"fold producer row stats M={M} d={d}", stats, torch.stack([x_ref.sum(1), (x_ref ** 2).sum(1)], 1), 2e-3)
        # consumer: (LN(x) * gmod + tmod) w^T + b  ==  r (acc - mu u) + c with u = w gmod, c = w tmod + b
        w = (torch.randn(N, d, generator=g) / d ** 0.5).to(dev, torch.bfloat16)
        b = torch.randn(N, generator=g).to(dev) * 0.1
        u = w.float() @ gmod
        cvec = w.float() @ tmod + b
        out = torch.full((M, N), float("nan"), device=dev, dtype=torch.bfloat16)
        ss = torch.zeros(M, 1, device=dev)
        nv.gemm(a_next, w, out, bias=cvec, sumsq=ss, sumsq_group_cols=N, ln=(stats, u, d, 1e-6))
        h = torch.nn.functional.layer_norm(x_ref, (d,), eps=1e-6) * gmod + tmod
        ref = h @ w.float().t() + b
        # (both forms feed a bf16 A operand: ~95.5 % of the elements inside the rms-relative tolerance either way)
        report(f"fold consumer M={M} d={d} N={N}", out, ref, 1.5e-2, min_inside=0.94)
        report(f"fold consumer sumsq M={M}", ss, (ref ** 2).sum(1, keepdim=True), 1e-2)
        # the unfused path on the same numbers, for scale: LN kernel -> bf16 -> GEMM
        hb = torch.empty(M, d, device=dev, dtype=torch.bfloat16)
        nv.layernorm_modulate(x, hb, 1e-6, scale=gmod - 1, shift=tmod)
        out2 = torch.empty_like(out)
        nv.gemm(hb, w, out2, bias=b)
        report(f"(unfused LN -> GEMM on the same inputs) M={M} d={d} N={N}", out2, ref, 1.5e-2, min_inside=0.94)
        e_fold, e_plain = (out.float() - ref).abs().mean().item(), (out2.float() - ref).abs().mean().item()
        ok = e_fold <= 1.1 * e_plain
        print(f"[{'OK ' if ok else 'BAD'}] fold mean |err| {e_fold:.3e} vs unfused {e_plain:.3e}", flush=True)
        RESULTS.append((f"fold error not above the unfused path M={M}", ok))


def attn_ref(q, k, v, H, scale):
    Lq, Lk = q.shape[0], k.shape[0]
    qh = q.float().view(Lq, H, 128).transpose(0, 1)
    kh = k.float().view(Lk, H, 128).transpose(0, 1)
    vh = v.float().view(Lk, H, 128).transpose(0, 1)
    s = (qh @ kh.transpose(1, 2)) * scale
    p = torch.softmax(s, dim=-1)
    return (p @ vh).transpose(0, 1).reshape(Lq, H * 128)


def attn_ref_no_rescale(q, k, v, H, scale, hd=128, tile=128, first_tile=0):
    """A WRONG online softmax for negative controls: K/V tiles in the kernel's visiting order (starting at first_tile,
    wrapping), the running max updated per tile, but the accumulated O and row sum never rescaled by exp(m_old - m_new)."""
    Lq, Lk = q.shape[0], k.shape[0]
    qh = q.float().view(Lq, H, hd).transpose(0, 1)
    kh = k.float().view(Lk, H, hd).transpose(0, 1)
    vh = v.float().view(Lk, H, hd).transpose(0, 1)
    n = (Lk + tile - 1) // tile
    m = torch.full((H, Lq, 1), float("-inf"), device=q.device)
    l = torch.zeros(H, Lq, 1, device=q.device)
    o = torch.zeros(H, Lq, hd, device=q.device)
    for j in range(n):
        t = (j + first_tile) % n
        s = (qh @ kh[:, t * tile:(t + 1) * tile].transpose(1, 2)) * scale
        m = torch.maximum(m, s.amax(-1, keepdim=True))
        p = torch.exp(s - m)
        l = l + p.sum(-1, keepdim=True)
        o = o + p @ vh[:, t * tile:(t + 1) * tile]
    return (o / l).transpose(0, 1).reshape(Lq, H * hd)


def sec_attn():
    g = torch.Generator(device="cpu").manual_seed(2)
    scale = 128 ** -0.5
    for (Lq, Lk, H, amp) in [(256, 128, 1, 1.0), (256, 256, 1, 1.0), (256, 512, 2, 1.0), (128, 128, 1, 1.0),
                             (300, 333, 2, 1.0), (1000, 1000, 3, 3.0), (257, 77, 1, 1.0), (3200, 3200, 2, 2.0),
                             # 300 units on 132 SMs: the 36 units of the third wave are cut into K/V slices and merged
                             (3200, 3200, 12, 1.0), (3000, 4100, 13, 2.0)]:
        q = (torch.randn(Lq, H * 128, generator=g) * amp).to(dev, torch.bfloat16)
        k = (torch.randn(Lk, H * 128, generator=g) * amp).to(dev, torch.bfloat16)
        v = torch.randn(Lk, H * 128, generator=g).to(dev, torch.bfloat16)
        ref = attn_ref(q, k, v, H, scale)
        for ws in (None, torch.empty(nv.attention_workspace_bytes(Lq, Lk, H) // 4 + 1, device=dev)):
            out = torch.full((Lq, H * 128), float("nan"), device=dev, dtype=torch.bfloat16)
            nv.attention(q, k, v, out, H, scale, workspace=ws)
            torch.cuda.synchronize()
            report(f"attn Lq={Lq} Lk={Lk} H={H} amp={amp} workspace={'yes' if ws is not None else 'no'}", out, ref, 2e-2)


def attn_ref_chunked(q, k, v, H, scale, chunk=4096):
    """fp32 reference on the GPU, query rows in chunks (a [chunk, Lk] score matrix per head at a time)."""
    Lq, Lk = q.shape[0], k.shape[0]
    out = torch.empty(Lq, H * 128, device=q.device, dtype=torch.float32)
    for h in range(H):
        kh = k[:, h * 128:(h + 1) * 128].float()
        vh = v[:, h * 128:(h + 1) * 128].float()
        for r0 in range(0, Lq, chunk):
            sc = (q[r0:r0 + chunk, h * 128:(h + 1) * 128].float() @ kh.t()) * scale
            out[r0:r0 + chunk, h * 128:(h + 1) * 128] = torch.softmax(sc, dim=-1) @ vh
    return out


def sec_attn_bench():
    """Self-attention at the BENCHMARK shape (L = 32760 = 255*128 + 120, 12 heads): 3072 (head, Q-tile) units on 132 SMs =
    23 whole waves + a sliced last wave merged by attn_merge_kernel, ragged last K/V and Q tiles.  amp 3 makes the softmax
    peaked (score std 9), so the outputs are O(1) and the elementwise tolerance bites."""
    g = torch.Generator(device="cpu").manual_seed(12)
    scale = 128 ** -0.5
    L, H = 32760, 12
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for amp in (1.0, 3.0):
            q = (torch.randn(L, H * 128, generator=g) * amp).to(dev, torch.bfloat16)
            k = (torch.randn(L, H * 128, generator=g) * amp).to(dev, torch.bfloat16)
            v = torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16)
            ref = attn_ref_chunked(q, k, v, H, scale)
            for ws in (torch.empty(nv.attention_workspace_bytes(L, L, H) // 4 + 1, device=dev), None):
                out = torch.full((L, H * 128), float("nan"), device=dev, dtype=torch.bfloat16)
                nv.attention(q, k, v, out, H, scale, workspace=ws)
                torch.cuda.synchronize()
                # amp 1: every output is an average over ~32760 comparably weighted values (|out| ~ 1/sqrt(L)): the bf16 P
                # operand leaves an absolute noise floor of ~1e-3 rms that the near-zero outputs feel;
                # amp 3 (peaked softmax, O(1) outputs): the relative leg decides
                report(f"attn bench shape L={L} H={H} amp={amp} workspace={'yes' if ws is not None else 'no'}", out, ref, 2e-2,
                       min_inside=0.94 if amp == 1.0 else 0.99)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def sec_abi3():
    """Entry points added with ABI 3: split-precision staging, q|k norm in one launch, attention with a per-row Q scale."""
    g = torch.Generator(device="cpu").manual_seed(13)
    # two-term bf16 split: hi + lo reproduces the f32 value to ~2^-17
    for (M, K, act, fn) in [(5, 256, nv.ACT_NONE, lambda t: t), (300, 1536, nv.ACT_SILU, torch.nn.functional.silu),
                            (257, 1280, nv.ACT_GELU_ERF, torch.nn.functional.gelu),
                            (512, 96, nv.ACT_GELU_TANH, lambda t: torch.nn.functional.gelu(t, approximate="tanh"))]:
        x = (torch.randn(M, K, generator=g) * 3).to(dev)
        d2 = torch.full((M, 2 * K), float("nan"), device=dev, dtype=torch.bfloat16)
        nv.split_f32_to_bf16x2(x, d2, act=act)
        report(f"split_f32_to_bf16x2 M={M} K={K} act={act}", d2[:, :K].float() + d2[:, K:].float(), fn(x), 2e-5)
        report(f"split hi part is the bf16 rounding act={act}", d2[:, :K], fn(x).to(torch.bfloat16), 4e-3)
    # LayerNorm + modulate, split output
    for (M, D) in [(77, 1536), (9, 5120), (33, 256)]:
        x = (torch.randn(M, D, generator=g) * 2 + 0.3).to(dev)
        sc, sh = torch.randn(D, generator=g).to(dev) * 0.1, torch.randn(D, generator=g).to(dev) * 0.1
        o2 = torch.full((M, 2 * D), float("nan"), device=dev, dtype=torch.bfloat16)
        nv.layernorm_modulate_split(x, o2, 1e-6, scale=sc, shift=sh)
        ref = torch.nn.functional.layer_norm(x, (D,), eps=1e-6) * (1 + sc) + sh
        report(f"layernorm_modulate_split M={M} D={D}", o2[:, :D].float() + o2[:, D:].float(), ref, 2e-5)
    # patchify, split output
    C0, C1, F, Hh, Ww = 16, 20, 3, 8, 12
    x = torch.randn(C0, F, Hh, Ww, generator=g).to(dev)
    y = torch.randn(C1, F, Hh, Ww, generator=g).to(dev)
    L = F * (Hh // 2) * (Ww // 2)
    kp = 4 * (C0 + C1)
    tok = torch.full((L, 2 * kp), float("nan"), device=dev, dtype=torch.bfloat16)
    nv.patchify_gather(x, y, tok, split=True)
    xy = torch.cat([x, y], 0)
    ref = xy.view(C0 + C1, F, Hh // 2, 2, Ww // 2, 2).permute(1, 2, 4, 0, 3, 5).reshape(L, kp)
    report("patchify_gather split", tok[:, :kp].float() + tok[:, kp:].float(), ref, 2e-5)
    # q | k norm + rope in one launch == two single launches
    M, H = 333, 3
    D = H * 128
    t = torch.randn(M, 3 * D, generator=g).to(dev, torch.bfloat16)
    tf = t.float()
    ss = torch.stack([(tf[:, :D] ** 2).sum(1), (tf[:, D:2 * D] ** 2).sum(1)], 1).contiguous()
    wq = (torch.randn(D, generator=g) * 0.2 + 1).to(dev)
    wk = (torch.randn(D, generator=g) * 0.2 + 1).to(dev)
    ang = torch.rand(M + 7, 64, generator=g, dtype=torch.float64) * 6.28
    cos, sin = ang.cos().float().to(dev), ang.sin().float().to(dev)
    a, b = t.clone(), t.clone()
    nv.qk_norm_rope(a[:, :2 * D], ss, 1e-6, wq, wk, cos, sin, row_offset=7)
    nv.rmsnorm_rope(b[:, :D], ss, 0, 1e-6, wq, cos, sin, row_offset=7)
    nv.rmsnorm_rope(b[:, D:2 * D], ss, 1, 1e-6, wk, cos, sin, row_offset=7)
    report("qk_norm_rope == rmsnorm_rope(q), rmsnorm_rope(k)", a, b, 1e-6)
    # attention with the Q RMS factor in the softmax scale == attention on the normalised q
    scale = 128 ** -0.5
    for (Lq, Lk, Hh_) in [(700, 512, 2), (3200, 257, 12), (130, 77, 1)]:
        Dq = Hh_ * 128
        q = (torch.randn(Lq, Dq, generator=g) * 2.5).to(dev, torch.bfloat16)
        k = torch.randn(Lk, Dq, generator=g).to(dev, torch.bfloat16)
        v = torch.randn(Lk, Dq, generator=g).to(dev, torch.bfloat16)
        ssq = (q.float() ** 2).sum(1, keepdim=True).contiguous()
        qn = q.float() * torch.rsqrt(ssq / Dq + 1e-6)
        out = torch.full((Lq, Dq), float("nan"), device=dev, dtype=torch.bfloat16)
        nv.attention_qscale(q, k, v, out, Hh_, ssq, Dq, 1e-6, scale)
        ref = attn_ref(qn, k, v, Hh_, scale)
        report(f"attention_qscale Lq={Lq} Lk={Lk} H={Hh_}", out, ref, 2e-2, min_inside=0.95)     # diffuse scores: see attn_bench
        # the folded factor must give what attention() gives on the explicitly normalised (bf16-rounded) q, to P-rounding noise
        out2 = torch.empty_like(out)
        nv.attention(qn.to(torch.bfloat16), k, v, out2, Hh_, scale)
        report(f"attention_qscale vs attention(normalised q) Lq={Lq} Lk={Lk} H={Hh_}", out, out2, 2e-2)
        nv.attention_qscale(q, k, v, out, Hh_, ssq, Dq, 1e-6, scale, accumulate=True)
        report(f"attention_qscale accumulate Lq={Lq} Lk={Lk} H={Hh_}", out, ref.bfloat16().float() + ref, 3e-2)
    # reproducible row sums of squares: the GEMM epilogue STORES one partial per 128-column segment ([M, groups, parts]), with one
    # and with several 128-row tiles; consumers add the partials in index order
    for Mg in (100, 700):
        Kk, gc, Ng = 256, 512, 3
        a_ = torch.randn(Mg, Kk, generator=g).to(dev, torch.bfloat16)
        w_ = (torch.randn(Ng * gc, Kk, generator=g) / 16).to(dev, torch.bfloat16)
        b_ = torch.randn(Ng * gc, generator=g).to(dev) * 0.1
        o_ = torch.empty(Mg, Ng * gc, device=dev, dtype=torch.bfloat16)
        parts = torch.full((Mg, 2, gc // 128), float("nan"), device=dev)          # 2 of the 3 groups; garbage in: nothing is accumulated
        nv.gemm(a_, w_, o_, bias=b_, sumsq=parts, sumsq_group_cols=gc)
        vref = a_.float() @ w_.float().t() + b_
        want = torch.stack([(vref[:, :gc] ** 2).sum(1), (vref[:, gc:2 * gc] ** 2).sum(1)], 1)
        report(f"gemm sumsq partials M={Mg}: sum of the {gc // 128} partials per group", parts.sum(2), want, 2e-3)
        first = parts.clone()
        nv.gemm(a_, w_, o_, bias=b_, sumsq=parts, sumsq_group_cols=gc)
        report(f"gemm sumsq partials M={Mg}: second run bit-identical", parts, first, 0.0)
    # consumers on partials == consumers on the summed value
    P = D // 128
    ssp = (tf[:, :2 * D].reshape(t.shape[0], 2, P, 128) ** 2).sum(3).contiguous()
    a2 = t.clone()
    nv.qk_norm_rope(a2[:, :2 * D], ssp, 1e-6, wq, wk, cos, sin, row_offset=7)
    report("qk_norm_rope on partial sums == on sums", a2, a, 1e-2)
    a3 = t.clone()
    nv.rmsnorm_rope(a3[:, D:2 * D], ssp, 1, 1e-6, wk, cos, sin, row_offset=7)
    report("rmsnorm_rope on partial sums (group 1) == on sums", a3[:, D:2 * D], a[:, D:2 * D], 1e-2)
    # D % 256 == 0: the kernel's warp-cooperative reduction of the partials (a warp's 256 columns lie in one row and group)
    for Hw in (2, 12, 40):
        Dw = Hw * 128
        tw_ = torch.randn(301, 3 * Dw, generator=g).to(dev, torch.bfloat16)
        sw = (tw_.float()[:, :2 * Dw].reshape(301, 2, Hw, 128) ** 2).sum(3).contiguous()
        wqw = (torch.randn(Dw, generator=g) * 0.2 + 1).to(dev)
        wkw = (torch.randn(Dw, generator=g) * 0.2 + 1).to(dev)
        angw = torch.rand(301 + 5, 64, generator=g, dtype=torch.float64) * 6.28
        cw, sn_ = angw.cos().float().to(dev), angw.sin().float().to(dev)
        x1, x2, x3 = tw_.clone(), tw_.clone(), tw_.clone()
        nv.qk_norm_rope(x1[:, :2 * Dw], sw, 1e-6, wqw, wkw, cw, sn_, row_offset=5)
        nv.qk_norm_rope(x2[:, :2 * Dw], sw.sum(2).contiguous(), 1e-6, wqw, wkw, cw, sn_, row_offset=5)
        report(f"qk_norm_rope D={Dw}: partial sums (warp reduction) == sums", x1, x2, 1e-2)
        nv.rmsnorm_rope(x3[:, Dw:2 * Dw], sw, 1, 1e-6, wkw, cw, sn_, row_offset=5)
        report(f"rmsnorm_rope D={Dw}: group 1 of the partials == qk_norm_rope's k", x3[:, Dw:2 * Dw], x1[:, Dw:2 * Dw], 0.0)
        x4 = tw_.clone()
        nv.qk_norm_rope(x4[:, :2 * Dw], sw, 1e-6, wqw, wkw, cw, sn_, row_offset=5)
        report(f"qk_norm_rope D={Dw}: second run bit-identical", x4, x1, 0.0)
    Lq, Lk, Hh_ = 700, 512, 2
    Dq = Hh_ * 128
    q = (torch.randn(Lq, Dq, generator=g) * 2.5).to(dev, torch.bfloat16)
    k = torch.randn(Lk, Dq, generator=g).to(dev, torch.bfloat16)
    v = torch.randn(Lk, Dq, generator=g).to(dev, torch.bfloat16)
    qp = (q.float().view(Lq, 1, Hh_, 128) ** 2).sum(3).contiguous()
    o_a = torch.empty(Lq, Dq, device=dev, dtype=torch.bfloat16)
    o_b = torch.empty_like(o_a)
    nv.attention_qscale(q, k, v, o_a, Hh_, qp, Dq, 1e-6, scale)
    nv.attention_qscale(q, k, v, o_b, Hh_, qp.sum(2).contiguous(), Dq, 1e-6, scale)
    report("attention_qscale on partial sums == on sums", o_a, o_b, 1e-2)
    # clip-boundary conversion: planar f32 video -> uint8 frames, bit-identical to the reference's numpy formula
    vid = (torch.rand(3, 5, 24, 40, generator=g) * 2.4 - 1.2).to(dev)
    u8 = torch.empty(5, 24, 40, 3, device=dev, dtype=torch.uint8)
    nv.frames_to_uint8(vid, u8)
    want = ((vid.float().permute(1, 2, 3, 0) + 1) * 127.5).clip(0, 255).cpu().numpy().astype("uint8")
    report("frames_to_uint8 == tensor2video arithmetic", u8.cpu().float().reshape(-1, 3), torch.from_numpy(want).float().reshape(-1, 3), 1e-9)
    # periodic add_rows + zero_
    tb = torch.randn(12, 256, generator=g).to(dev)
    tt = torch.randn(6, 256, generator=g).to(dev)
    oo = torch.empty_like(tb)
    nv.add_rows(tb, tt, oo)
    report("add_rows periodic", oo, tb + tt.repeat(2, 1), 1e-6)
    z = torch.randn(1000, 3, generator=g).to(dev)
    nv.zero_(z)
    report("zero_", z + 1, torch.ones_like(z), 1e-7)


def sec_attn_cross():
    g = torch.Generator(device="cpu").manual_seed(3)
    scale = 128 ** -0.5
    H, Lq = 2, 700
    # fused qkv layout: q,k,v are column slices of one [L, 3*H*128] buffer
    qkv = torch.randn(Lq, 3 * H * 128, generator=g).to(dev, torch.bfloat16)
    d = H * 128
    out = torch.empty(Lq, d, device=dev, dtype=torch.bfloat16)
    nv.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], out, H, scale)
    report("attn strided qkv slices", out, attn_ref(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], H, scale), 2e-2)
    # cross attention: Lk=512 then accumulate Lk=257
    q = torch.randn(Lq, d, generator=g).to(dev, torch.bfloat16)
    k1 = torch.randn(512, d, generator=g).to(dev, torch.bfloat16)
    v1 = torch.randn(512, d, generator=g).to(dev, torch.bfloat16)
    k2 = torch.randn(257, d, generator=g).to(dev, torch.bfloat16)
    v2 = torch.randn(257, d, generator=g).to(dev, torch.bfloat16)
    nv.attention(q, k1, v1, out, H, scale)
    r1 = attn_ref(q, k1, v1, H, scale)
    report("cross Lk=512", out, r1, 2e-2)
    nv.attention(q, k2, v2, out, H, scale, accumulate=True)
    report("cross accumulate Lk=257", out, r1.bfloat16().float() + attn_ref(q, k2, v2, H, scale), 3e-2)


def sec_ew():
    g = torch.Generator(device="cpu").manual_seed(4)
    for (M, D) in [(77, 1536), (5, 5120), (300, 256), (33, 1280)]:
        x = (torch.randn(M, D, generator=g) * 2 + 0.3).to(dev)
        scale = torch.randn(D, generator=g).to(dev) * 0.1
        shift = torch.randn(D, generator=g).to(dev) * 0.1
        gamma = torch.randn(D, generator=g).to(dev)
        beta = torch.randn(D, generator=g).to(dev)
        out = torch.empty(M, D, device=dev, dtype=torch.bfloat16)
        nv.layernorm_modulate(x, out, 1e-6, scale=scale, shift=shift)
        ref = torch.nn.functional.layer_norm(x, (D,), eps=1e-6) * (1 + scale) + shift
        report(f"ln_modulate M={M} D={D}", out, ref, 1e-2)
        nv.layernorm_modulate(x, out, 1e-6, gamma=gamma, beta=beta)
        ref = torch.nn.functional.layer_norm(x, (D,), gamma, beta, eps=1e-6)
        report(f"ln_affine M={M} D={D}", out, ref, 1e-2)
    # rmsnorm + rope
    M, H = 200, 3
    D = H * 128
    t = torch.randn(M, 3 * D, generator=g).to(dev, torch.bfloat16)
    w = (torch.randn(D, generator=g) * 0.2 + 1).to(dev)
    tf = t.float()
    ss = torch.stack([(tf[:, :D] ** 2).sum(1), (tf[:, D:2 * D] ** 2).sum(1)], 1).contiguous()
    ang = torch.rand(M + 10, 64, generator=g, dtype=torch.float64) * 6.28
    cos, sin = ang.cos().float().to(dev), ang.sin().float().to(dev)
    ref_in = tf[:, D:2 * D]
    ref = ref_in * torch.rsqrt(ss[:, 1:2] / D + 1e-6) * w
    refc = torch.view_as_complex(ref.double().reshape(M, H, 64, 2))
    fr = torch.polar(torch.ones(M, 64, dtype=torch.float64), ang[3:3 + M]).to(dev)
    ref_r = torch.view_as_real(refc * fr[:, None, :]).reshape(M, D).float()
    t2 = t.clone()
    nv.rmsnorm_rope(t2[:, D:2 * D], ss, 1, 1e-6, w, cos, sin, row_offset=3)
    report("rmsnorm+rope (strided k slice)", t2[:, D:2 * D], ref_r, 1e-2)
    report("rmsnorm+rope left q slice untouched", t2[:, :D], tf[:, :D], 1e-6)
    t3 = t.clone()
    nv.rmsnorm_rope(t3[:, :D], ss, 0, 1e-6, w)
    report("rmsnorm only", t3[:, :D], tf[:, :D] * torch.rsqrt(ss[:, 0:1] / D + 1e-6) * w, 1e-2)
    # patchify / unpatchify
    C0, C1, F, Hh, Ww = 16, 20, 3, 8, 12
    x = torch.randn(C0, F, Hh, Ww, generator=g).to(dev)
    y = torch.randn(C1, F, Hh, Ww, generator=g).to(dev)
    L = F * (Hh // 2) * (Ww // 2)
    tok = torch.empty(L, 4 * (C0 + C1), device=dev, dtype=torch.bfloat16)
    nv.patchify_gather(x, y, tok)
    xy = torch.cat([x, y], 0)
    ref = xy.view(C0 + C1, F, Hh // 2, 2, Ww // 2, 2).permute(1, 2, 4, 0, 3, 5).reshape(L, (C0 + C1) * 4)
    report("patchify_gather", tok, ref, 1e-2)
    ho = torch.randn(L, 64, generator=g).to(dev)
    out = torch.empty(16, F, Hh, Ww, device=dev)
    nv.unpatchify(ho, out)
    ref = ho.view(F, Hh // 2, Ww // 2, 2, 2, 16).permute(5, 0, 1, 3, 2, 4).reshape(16, F, Hh, Ww)
    report("unpatchify", out.reshape(16, -1), ref.reshape(16, -1), 1e-6)
    # cfg euler
    lat = torch.randn(1000, 7, generator=g).to(dev)
    vc = torch.randn(1000, 7, generator=g).to(dev)
    vu = torch.randn(1000, 7, generator=g).to(dev)
    l2 = lat.clone()
    nv.cfg_euler_step(l2, vc, vu, 5.0, 0.9, 0.8)
    report("cfg_euler", l2, lat + (vu + 5.0 * (vc - vu)) * (0.8 - 0.9), 1e-5)
    tb = torch.randn(6, 1536, generator=g).to(dev)
    tt = torch.randn(6, 1536, generator=g).to(dev)
    oo = torch.empty_like(tb)
    nv.add_rows(tb, tt, oo)
    report("add_rows", oo, tb + tt, 1e-6)
    nv.add_rows(tb[:2].contiguous(), tt[:1].contiguous(), oo[:2])
    report("add_rows bcast", oo[:2], tb[:2] + tt[:1], 1e-6)


def _gemm_bound_report(name, got, a, w, K, bias=None, act=0, gate=None, residual=None, c=2.0, drop_tail=True):
    """Per-element bar of a GEMM against its fp64 reference: |err| <= c K 2^-24 (|A| |W|^T)[m, n] (accumulation), plus a few
    fp32 roundings of the epilogue terms, plus half a bf16 ulp of the value for bf16 outputs.  Negative control: the reference
    without the last 8 columns of K (a K tail read as zero) must fail it."""
    def ref_of(kk):
        v = a[:, :kk].double() @ w[:, :kk].double().t()
        if bias is not None:
            v = v + bias.double()
        if act == nv.ACT_RELU:
            v = v.clamp_min(0)
        if gate is not None:
            v = v * gate.double()
        if residual is not None:
            v = v + residual.double()
        return v
    ref = ref_of(K)
    P = a.double().abs() @ w.double().abs().t()
    g_abs = gate.double().abs() if gate is not None else 1.0
    epi = (bias.double().abs() if bias is not None else 0.0) * g_abs + (residual.double().abs() if residual is not None else 0.0)
    bound = 2.0 ** -24 * (c * K * P * g_abs + 4 * (epi + ref.abs()))
    gotd = got.double()
    if got.dtype == torch.bfloat16:
        _, e = torch.frexp(torch.maximum(gotd.abs(), ref.abs()))
        bound = bound + torch.ldexp(torch.full_like(bound, 0.5), e - 8)      # half a bf16 ulp
    err = (gotd - ref).abs()
    inside = err <= bound
    ok = bool(inside.all())
    worst = (err / bound.clamp_min(1e-300)).max().item()
    print(f"[{'OK ' if ok else 'BAD'}] {name}: max_err={err.max().item():.3e} worst err/bound={worst:.3f} (c={c})", flush=True)
    RESULTS.append((name, ok))
    if not ok:
        r, cc = (~inside).nonzero()[0].tolist()
        print(f"      first outside [{r},{cc}] got={gotd[r, cc].item()} ref={ref[r, cc].item()} bound={bound[r, cc].item():.3e}")
    if drop_tail and K > 8:
        caught = not bool(((gotd - ref_of(K - 8)).abs() <= bound).all())
        print(f"[{'OK ' if caught else 'BAD'}] negative control {name}: reference without the last 8 K columns fails: {caught}", flush=True)
        RESULTS.append((f"negative control {name}", caught))
    return ref


def sec_gemm_edges():
    """GEMM edges under a per-element fp64 bound: ReLU epilogue, A and W as column slices of NaN-padded wider buffers
    (lda / ldw > K, K % 64 != 0: the tensor-map extent must zero-fill, not read the neighbours), bf16 out with gate + f32
    residual, N = 8 / 264, M = 1, 32-column atomic sumsq groups, and more than 2 x 132 tiles so every CTA loops.
    Measured on an H100 80GB HBM3 at a 400 W power limit: f32 outputs use at most 9 % of the c = 2 bound (K = 8; under 2 %
    for K >= 72); bf16 outputs up to 99.8 %, which is the half-ulp rounding term."""
    g = torch.Generator(device="cpu").manual_seed(31)

    def operands(M, N, K, pad=0):
        a_big = torch.full((M, K + pad), float("nan"), dtype=torch.bfloat16, device=dev)
        w_big = torch.full((N, K + pad), float("nan"), dtype=torch.bfloat16, device=dev)
        a_big[:, :K] = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
        w_big[:, :K] = (torch.randn(N, K, generator=g) * 0.5).to(dev, torch.bfloat16)
        return a_big[:, :K], w_big[:, :K]

    for (M, N, K, pad) in [(300, 264, 8, 56), (130, 264, 72, 8), (257, 520, 200, 24), (1, 8, 72, 40), (1, 264, 200, 0),
                           (129, 8, 8, 8)]:
        a, w = operands(M, N, K, pad)
        out = torch.full((M, N), float("nan"), device=dev)
        nv.gemm(a, w, out)
        _gemm_bound_report(f"gemm_edges f32 M={M} N={N} K={K} lda=ldw={K + pad}", out, a, w, K)
    # ReLU epilogue (AudioProjModel), f32 and bf16 out
    M, N, K = 300, 264, 200
    a, w = operands(M, N, K, 24)
    bias = torch.randn(N, generator=g).to(dev)
    for dt in (torch.float32, torch.bfloat16):
        out = torch.full((M, N), float("nan"), device=dev, dtype=dt)
        nv.gemm(a, w, out, bias=bias, act=nv.ACT_RELU)
        _gemm_bound_report(f"gemm_edges bias+relu {dt}", out, a, w, K, bias=bias, act=nv.ACT_RELU)
        negative(f"gemm_edges relu {dt}: reference without the ReLU", out, a.float() @ w.float().t() + bias, 2e-3)
    # bf16 out with gate + f32 residual, into a column slice of a wider buffer
    gate = torch.randn(N, generator=g).to(dev)
    res = torch.randn(M, N, generator=g).to(dev)
    big = torch.full((M, N + 40), float("nan"), device=dev, dtype=torch.bfloat16)
    nv.gemm(a, w, big[:, :N], bias=bias, gate=gate, residual=res)
    _gemm_bound_report("gemm_edges bf16 out bias+gate+residual", big[:, :N], a, w, K, bias=bias, gate=gate, residual=res)
    RESULTS.append(("gemm_edges bf16 out: columns beyond N untouched", bool(torch.isnan(big[:, N:].float()).all())))
    # 32-column atomic sumsq groups (7 of the 8 groups accumulated)
    N2 = 256
    a2, w2 = operands(M, N2, K, 8)
    b2 = torch.randn(N2, generator=g).to(dev)
    ss = torch.zeros(M, 7, device=dev)
    out = torch.full((M, N2), float("nan"), device=dev)
    nv.gemm(a2, w2, out, bias=b2, sumsq=ss, sumsq_group_cols=32)
    v = _gemm_bound_report("gemm_edges f32 with 32-column sumsq groups", out, a2, w2, K, bias=b2)
    want = (v[:, :224] ** 2).reshape(M, 7, 32).sum(2)
    P = (a2.double().abs() @ w2.double().abs().t() + b2.double().abs())[:, :224]
    ss_bound = (2 * v[:, :224].abs() * 2.0 ** -24 * (2 * K * P + 4 * v[:, :224].abs())).reshape(M, 7, 32).sum(2) \
        + 2.0 ** -24 * 64 * want
    err = (ss.double() - want).abs()
    ok = bool((err <= ss_bound).all())
    print(f"[{'OK ' if ok else 'BAD'}] gemm_edges sumsq 32-column groups: worst err/bound={(err / ss_bound).max().item():.3f}", flush=True)
    RESULTS.append(("gemm_edges sumsq 32-column groups", ok))
    wrong_ss = (v[:, :256] ** 2).reshape(M, 8, 32).sum(2)[:, 1:]          # groups shifted by one
    RESULTS.append(("negative control gemm_edges sumsq: shifted groups fail", not bool(((ss.double() - wrong_ss).abs() <= ss_bound).all())))
    # more than 2 x 132 output tiles: every persistent CTA takes several
    a3, w3 = operands(2048, 4608, 136, 8)
    out = torch.full((2048, 4608), float("nan"), device=dev, dtype=torch.bfloat16)
    nv.gemm(a3, w3, out)
    _gemm_bound_report("gemm_edges bf16 M=2048 N=4608 K=136 (every CTA loops)", out, a3, w3, 136)


def attn_online_inputs(g, Lq, Lk, H, amp, ramp=0.0, dominant=None):
    """bf16 q, k, v of the online-softmax stresses: every score gains ramp * key / (Lk - 1) (with scale 1/sqrt(128), so the
    row max rises in every K/V tile), and key `dominant`, when given, gains +35 on every score"""
    q = torch.randn(Lq, H * 128, generator=g) * amp
    k = torch.randn(Lk, H * 128, generator=g) * amp
    v = torch.randn(Lk, H * 128, generator=g)
    q.view(Lq, H, 128)[:, :, 0] = 4.0                   # a common direction: scores rise with k[:, 0]
    k.view(Lk, H, 128)[:, :, 0] += ramp * torch.arange(Lk).float().unsqueeze(1) / max(Lk - 1, 1)
    if dominant is not None:
        k.view(Lk, H, 128)[dominant, :, 0] = 100.0     # +35 on every score of that key
    return tuple(t.to(dev, torch.bfloat16) for t in (q, k, v))


def sec_attn_online():
    """Online softmax under stress (bar: report()'s elementwise min_inside against the fp32 reference): key amplitude
    growing along the sequence so the row max rises in every K/V tile, one dominant key in the last tile or in a middle slice
    of a sliced plan, Lk = 1 / 129, Lq = 1, score std 10-20, with and without workspace.  Negative control: the same online
    softmax without the exp(m_old - m_new) rescale."""
    g = torch.Generator(device="cpu").manual_seed(32)
    scale = 128 ** -0.5

    def make(Lq, Lk, H, amp, ramp=0.0, dominant=None):
        return attn_online_inputs(g, Lq, Lk, H, amp, ramp, dominant)

    cases = [("ramp", 1000, 1000, 2, 3.5, 120.0, None), ("ramp sliced", 3200, 4100, 12, 3.5, 120.0, None),
             ("dominant key in the last tile", 700, 1000, 2, 3.2, 0.0, 999),
             ("dominant key in a middle slice", 3200, 4100, 12, 3.2, 0.0, 2053),
             ("Lk=1", 300, 1, 2, 3.5, 0.0, None), ("Lk=129", 300, 129, 3, 3.5, 50.0, 128), ("Lq=1", 1, 1000, 2, 3.5, 120.0, None),
             ("std 20", 513, 777, 2, 4.5, 0.0, None)]
    for name, Lq, Lk, H, amp, ramp, dom in cases:
        q, k, v = make(Lq, Lk, H, amp, ramp, dom)
        ref = attn_ref(q, k, v, H, scale)
        wrong = attn_ref_no_rescale(q, k, v, H, scale)
        s_std = (q.float()[:, :128] @ k.float()[:, :128].t() * scale).std().item()
        for ws in (None, torch.empty(nv.attention_workspace_bytes(Lq, Lk, H) // 4 + 1, device=dev)):
            out = torch.full((Lq, H * 128), float("nan"), device=dev, dtype=torch.bfloat16)
            nv.attention(q, k, v, out, H, scale, workspace=ws)
            torch.cuda.synchronize()
            tag = f"attn_online {name} Lq={Lq} Lk={Lk} H={H} score std {s_std:.1f} workspace={'yes' if ws is not None else 'no'}"
            report(tag, out, ref, 2e-2, min_inside=0.99)
            if Lk > 128:
                negative(tag + " (no rescale)", out, wrong, 2e-2, min_inside=0.99)


def _attn_sp_cases(shapes):
    """svi_attn_fwd_sp on one GPU: every flag already holds the epoch (set and synchronised before the launch), so the
    producer never waits; what runs is the K/V stream that starts on the local chunk and wraps, the ragged last tile visited
    mid-stream, sliced units offset by kv_first_tile and the merge of the slices."""
    g = torch.Generator(device="cpu").manual_seed(33)
    scale = 128 ** -0.5
    epoch = 5
    for (L, chunk, H, amp) in shapes:
        q = (torch.randn(L, H * 128, generator=g) * amp).to(dev, torch.bfloat16)
        k = (torch.randn(L, H * 128, generator=g) * amp).to(dev, torch.bfloat16)
        v = torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16)
        ref = attn_ref_chunked(q, k, v, H, scale) if L > 8192 else attn_ref(q, k, v, H, scale)
        n_chunks = (L + chunk - 1) // chunk
        flags = torch.full((n_chunks,), epoch, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()                          # the flags hold the epoch before any launch reads them
        for c in range(n_chunks):
            r0, r1 = c * chunk, min(L, (c + 1) * chunk)
            ql = q[r0:r1]
            plain = torch.empty(r1 - r0, H * 128, device=dev, dtype=torch.bfloat16)
            nv.attention(ql, k, v, plain, H, scale)
            first_tile = (c * chunk + 127) // 128
            for ws in (None, torch.empty(nv.attention_workspace_bytes(r1 - r0, L, H) // 4 + 1, device=dev)):
                out = torch.full((r1 - r0, H * 128), float("nan"), device=dev, dtype=torch.bfloat16)
                nv.attention_sp(ql, k, v, out, H, flags, epoch, chunk, c, scale, workspace=ws)
                torch.cuda.synchronize()
                tag = f"attn_sp one GPU L={L} chunk={chunk} H={H} self_chunk={c} workspace={'yes' if ws is not None else 'no'}"
                report(tag, out, ref[r0:r1], 2e-2, min_inside=0.95)
                report(tag + " vs attention()", out, plain, 2e-2)
            if c == n_chunks - 1:
                negative(f"attn_sp L={L} self_chunk={c} (no rescale)", out,
                         attn_ref_no_rescale(ql, k, v, H, scale, first_tile=first_tile), 2e-2, min_inside=0.95)


def sec_attn_sp_one_gpu():
    # L = 1260 in two 630-row chunks (chunk boundaries inside a K/V tile, ragged 108-row last tile); L = 4100 in two chunks:
    # 34 units on 132 SMs, so the workspace plan slices every unit and the slices start at j_begin + kv_first_tile
    _attn_sp_cases([(1260, 630, 2, 2.0), (4100, 2050, 2, 2.0), (1260, 420, 3, 2.0)])


def sec_attn_sp_one_gpu_long():
    # the benchmark shape on 4 ranks: L = 32760 in 8190-row chunks, 12 heads
    _attn_sp_cases([(32760, 8190, 12, 2.0)])


def sec_attn_small_long():
    """svi_attn_small at the wav2vec2 length (61 s at 50 Hz: ~3050 tokens, 12 heads x 64) against fp32, and a key mask.
    A launch whose keys are all masked writes 0 (header: svi_attn_small)."""
    g = torch.Generator(device="cpu").manual_seed(34)
    L, H, hd = 3050, 12, 64
    scale = hd ** -0.5
    q, k, v = ((torch.randn(L, H * hd, generator=g) * a).to(dev, torch.bfloat16) for a in (2.0, 2.0, 1.0))

    def ref_of(mask=None):
        qh, kh, vh = (t.float().view(L, H, hd).transpose(0, 1) for t in (q, k, v))
        s = qh @ kh.transpose(1, 2) * scale
        if mask is not None:
            s = s.masked_fill(mask.view(1, 1, L) == 0, float("-inf"))
        return (torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(L, H * hd)

    out = torch.full((L, H * hd), float("nan"), device=dev, dtype=torch.bfloat16)
    nv.attention_small(q, k, v, out, H, hd, scale)
    report(f"attn_small L={L} H={H} hd={hd}", out, ref_of(), 1e-2, min_inside=0.999)
    negative("attn_small (no rescale, 32-key tiles)", out, attn_ref_no_rescale(q, k, v, H, scale, hd=hd, tile=32), 1e-2, 0.999)
    mask = (torch.rand(L, generator=g) > 0.3).to(torch.int32).to(dev)
    out.fill_(float("nan"))
    nv.attention_small(q, k, v, out, H, hd, scale, key_mask=mask)
    report(f"attn_small L={L} key mask (30 % masked)", out, ref_of(mask), 1e-2, min_inside=0.999)
    negative("attn_small key mask ignored", out, ref_of(), 1e-2, 0.999)
    out.fill_(float("nan"))
    nv.attention_small(q, k, v, out, H, hd, scale, key_mask=torch.zeros(L, dtype=torch.int32, device=dev))
    ok = bool((out.float() == 0).all())
    print(f"[{'OK ' if ok else 'BAD'}] attn_small every key masked: all outputs 0", flush=True)
    RESULTS.append(("attn_small every key masked -> 0", ok))


def sec_perf_gemm():
    g = torch.Generator(device="cpu").manual_seed(5)
    L = 32760
    for (M, N, K, name) in [(L, 4608, 1536, "qkv"), (L, 1536, 1536, "o"), (L, 8960, 1536, "ffn1"),
                            (L, 1536, 8960, "ffn2"), (8192, 8192, 8192, "square8k")]:
        a = torch.randn(M, K, generator=g).to(dev, torch.bfloat16)
        w = (torch.randn(N, K, generator=g) * 0.02).to(dev, torch.bfloat16)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        ms = time_ms(lambda: nv.gemm(a, w, out))
        tf = 2.0 * M * N * K / ms / 1e9
        ms_t = time_ms(lambda: torch.matmul(a, w.t()))
        print(f"[PERF] gemm {name} M={M} N={N} K={K}: {ms:.3f} ms = {tf:.1f} TFLOP/s | cuBLAS {ms_t:.3f} ms = {2.0*M*N*K/ms_t/1e9:.1f}", flush=True)


def sec_perf_gemm_epi():
    """The DiT's GEMMs with the epilogues they carry in the block (the bare GEMM is perf_gemm)."""
    g = torch.Generator(device="cpu").manual_seed(7)
    L, d, f = 32760, 1536, 8960
    h = torch.randn(L, d, generator=g).to(dev, torch.bfloat16)
    hf = torch.randn(L, f, generator=g).to(dev, torch.bfloat16)
    x = torch.randn(L, d, generator=g).to(dev)
    gate = torch.randn(d, generator=g).to(dev)
    mk = lambda n, k: (torch.randn(n, k, generator=g) * 0.02).to(dev, torch.bfloat16)
    w_qkv, w_o, w_f0, w_f2 = mk(3 * d, d), mk(d, d), mk(f, d), mk(d, f)
    b3, b1, bf_ = torch.randn(3 * d, generator=g).to(dev), torch.randn(d, generator=g).to(dev), torch.randn(f, generator=g).to(dev)
    qkv = torch.empty(L, 3 * d, device=dev, dtype=torch.bfloat16)
    ffn = torch.empty(L, f, device=dev, dtype=torch.bfloat16)
    ss = torch.zeros(L, 2, device=dev)
    cases = [
        ("qkv  bias+sumsq -> bf16", lambda: nv.gemm(h, w_qkv, qkv, bias=b3, sumsq=ss, sumsq_group_cols=d), 2.0 * L * 3 * d * d),
        ("o    bias+gate+residual (in place f32)", lambda: nv.gemm(h, w_o, x, bias=b1, gate=gate, residual=x), 2.0 * L * d * d),
        ("ffn0 bias+gelu_tanh -> bf16", lambda: nv.gemm(h, w_f0, ffn, bias=bf_, act=nv.ACT_GELU_TANH), 2.0 * L * f * d),
        ("ffn2 bias+gate+residual (in place f32)", lambda: nv.gemm(hf, w_f2, x, bias=b1, gate=gate, residual=x), 2.0 * L * f * d),
    ]
    for name, fn, fl in cases:
        ms = time_ms(fn)
        print(f"[PERF] gemm {name}: {ms:.3f} ms = {fl / ms / 1e9:.1f} TFLOP/s", flush=True)


def sec_perf_ln_fold():
    """The LayerNorm fold's cost per GEMM at the bench shape: consumer (ffn.0 with GELU, qkv with the row sums) and producer
    (o-projection class emitting the next operand + row statistics) against the same GEMMs without the fold and the
    LayerNorm kernel they replace."""
    g = torch.Generator(device="cpu").manual_seed(7)
    L, d, f = 32760, 1536, 8960
    h = torch.randn(L, d, generator=g).to(dev, torch.bfloat16)
    x = torch.randn(L, d, generator=g).to(dev)
    gate = torch.randn(d, generator=g).to(dev)
    mk = lambda n, k: (torch.randn(n, k, generator=g) * 0.02).to(dev, torch.bfloat16)
    w_qkv, w_o, w_f0 = mk(3 * d, d), mk(d, d), mk(f, d)
    b3, b1, bf_ = torch.randn(3 * d, generator=g).to(dev), torch.randn(d, generator=g).to(dev), torch.randn(f, generator=g).to(dev)
    u3, u0 = torch.randn(3 * d, generator=g).to(dev), torch.randn(f, generator=g).to(dev)
    stats = torch.stack([torch.randn(L, generator=g) * 10, torch.rand(L, generator=g) * d + d], 1).to(dev).contiguous()
    qkv = torch.empty(L, 3 * d, device=dev, dtype=torch.bfloat16)
    ffn = torch.empty(L, f, device=dev, dtype=torch.bfloat16)
    a_next = torch.empty(L, d, device=dev, dtype=torch.bfloat16)
    rs = torch.zeros(L, 2, device=dev)
    ss = torch.zeros(L, 2, device=dev)
    cases = [
        ("ffn0 bias+gelu", lambda: nv.gemm(h, w_f0, ffn, bias=bf_, act=nv.ACT_GELU_TANH), 2.0 * L * f * d),
        ("ffn0 bias+gelu + LN consumer", lambda: nv.gemm(h, w_f0, ffn, bias=bf_, act=nv.ACT_GELU_TANH, ln=(stats, u0, d, 1e-6)), 2.0 * L * f * d),
        ("qkv bias+sumsq", lambda: nv.gemm(h, w_qkv, qkv, bias=b3, sumsq=ss, sumsq_group_cols=d), 2.0 * L * 3 * d * d),
        ("qkv bias+sumsq + LN consumer", lambda: nv.gemm(h, w_qkv, qkv, bias=b3, sumsq=ss, sumsq_group_cols=d, ln=(stats, u3, d, 1e-6)), 2.0 * L * 3 * d * d),
        ("o gate+residual", lambda: nv.gemm(h, w_o, x, bias=b1, gate=gate, residual=x), 2.0 * L * d * d),
        ("o gate+residual + emit", lambda: nv.gemm(h, w_o, x, bias=b1, gate=gate, residual=x, emit=(a_next, gate, rs)), 2.0 * L * d * d),
        ("layernorm_modulate (the launch a folded pair replaces)", lambda: nv.layernorm_modulate(x, a_next, 1e-6, scale=gate, shift=b1), 0.0),
    ]
    for name, fn, fl in cases:
        ms = time_ms(fn)
        print(f"[PERF] {name}: {ms * 1e3:.1f} us" + (f" = {fl / ms / 1e9:.1f} TFLOP/s" if fl else ""), flush=True)


def sec_perf_ew():
    """Row kernels at the bench shape, algorithmic bytes / time (HBM roofline: MEASURED_PEAKS.json hbm_gbps)."""
    g = torch.Generator(device="cpu").manual_seed(8)
    L, d = 32760, 1536
    x = torch.randn(L, d, generator=g).to(dev)
    sc, sh = torch.randn(d, generator=g).to(dev) * 0.1, torch.randn(d, generator=g).to(dev) * 0.1
    h = torch.empty(L, d, device=dev, dtype=torch.bfloat16)
    flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)

    def timed(fn, nbytes, name, cold):
        ts = []
        for _ in range(6):
            if cold:
                flush.zero_()      # evict x / h from L2 and leave 256 MB of dirty lines, as the preceding GEMM does
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ms = sorted(ts)[len(ts) // 2]
        print(f"[PERF] {name} ({'after a 256 MB write' if cold else 'back to back'}): {ms * 1e3:.1f} us = {nbytes / ms / 1e6:.0f} GB/s", flush=True)

    for cold in (False, True):
        timed(lambda: nv.layernorm_modulate(x, h, 1e-6, scale=sc, shift=sh), L * d * 6, "layernorm_modulate L=32760 d=1536", cold)
    qkv = torch.randn(L, 3 * d, generator=g).to(dev, torch.bfloat16)
    ss = torch.rand(L, 2, generator=g).to(dev) * d
    w = torch.randn(d, generator=g).to(dev)
    f, hh, ww = 21, 30, 52
    cos = torch.randn(L, 64, generator=g).to(dev)
    sin = torch.randn(L, 64, generator=g).to(dev)
    for cold in (False, True):
        timed(lambda: nv.rmsnorm_rope(qkv[:, :d], ss, 0, 1e-6, w, cos, sin, 0), L * d * 4, "rmsnorm_rope (q slice of qkv)", cold)
    ssp = (torch.rand(L, 2, d // 128, generator=g) * 128).to(dev)
    w2 = torch.randn(d, generator=g).to(dev)
    for cold in (False, True):
        timed(lambda: nv.qk_norm_rope(qkv[:, :2 * d], ss, 1e-6, w, w2, cos, sin, 0), L * d * 8, "qk_norm_rope, one sum per row and group", cold)
        timed(lambda: nv.qk_norm_rope(qkv[:, :2 * d], ssp, 1e-6, w, w2, cos, sin, 0), L * d * 8, "qk_norm_rope, 12 partial sums per row and group", cold)


def sec_perf_attn_quick():
    """Self-attention at the bench shape only (with the launch-plan workspace), for A/B runs of kernel variants
    (SVI_B200_LIB selects the library)."""
    g = torch.Generator(device="cpu").manual_seed(6)
    scale = 128 ** -0.5
    L, H = 32760, 12
    q, k, v = (torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16) for _ in range(3))
    out = torch.empty(L, H * 128, device=dev, dtype=torch.bfloat16)
    ws = torch.empty(nv.attention_workspace_bytes(L, L, H) // 4 + 1, device=dev)
    ms = time_ms(lambda: nv.attention(q, k, v, out, H, scale, workspace=ws), iters=8, warm=3)
    fl = 4.0 * L * L * H * 128
    print(f"[PERF] attn L={L} H={H} + workspace lib={os.path.basename(nv.lib_path())}: {ms:.3f} ms = {fl/ms/1e9:.1f} TFLOP/s", flush=True)


def sec_perf_attn():
    g = torch.Generator(device="cpu").manual_seed(6)
    scale = 128 ** -0.5
    for (L, H) in [(8192, 12), (32760, 12)]:
        q = torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16)
        k = torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16)
        v = torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16)
        out = torch.empty(L, H * 128, device=dev, dtype=torch.bfloat16)
        ms = time_ms(lambda: nv.attention(q, k, v, out, H, scale), iters=5, warm=2)
        fl = 4.0 * L * L * H * 128
        print(f"[PERF] attn L={L} H={H}: {ms:.3f} ms = {fl/ms/1e9:.1f} TFLOP/s", flush=True)
        ws = torch.empty(nv.attention_workspace_bytes(L, L, H) // 4 + 1, device=dev)
        ms = time_ms(lambda: nv.attention(q, k, v, out, H, scale, workspace=ws), iters=5, warm=2)
        print(f"[PERF] attn L={L} H={H} + workspace (sliced last wave): {ms:.3f} ms = {fl/ms/1e9:.1f} TFLOP/s", flush=True)
        try:
            from flash_attn import flash_attn_func
            q4, k4, v4 = (t.view(1, L, H, 128) for t in (q, k, v))
            ms2 = time_ms(lambda: flash_attn_func(q4, k4, v4), iters=5, warm=2)
            print(f"[PERF]   flash_attn2 (library, mma.sync) {ms2:.3f} ms = {fl/ms2/1e9:.1f} TFLOP/s", flush=True)
        except Exception as ex:  # noqa: BLE001
            print("[PERF]   flash_attn2 unavailable:", repr(ex)[:100])
    # cross attention shape
    L, H = 32760, 12
    q = torch.randn(L, H * 128, generator=g).to(dev, torch.bfloat16)
    k = torch.randn(512, H * 128, generator=g).to(dev, torch.bfloat16)
    v = torch.randn(512, H * 128, generator=g).to(dev, torch.bfloat16)
    out = torch.empty(L, H * 128, device=dev, dtype=torch.bfloat16)
    ms = time_ms(lambda: nv.attention(q, k, v, out, H, scale))
    print(f"[PERF] cross attn L={L} Lk=512: {ms:.3f} ms = {4.0*L*512*H*128/ms/1e9:.1f} TFLOP/s", flush=True)


def _conv_runner():
    """run(...) = one svi_conv3d_causal case against torch conv3d on a hand-built frame ring."""
    import torch.nn.functional as F
    g = torch.Generator(device="cpu").manual_seed(7)

    def run(Cin, Cout, kt, kh, kw, T, H, W, pad, n_split=0, residual=False, fuse=None, variant=1, tag="", tile_w=None):
        """tile_w: None = 8 for W <= 8 else 16; "pick" = the VAE's _pick_tile_w(H, W); an int; or a list of widths run on
        the same descriptor and inputs, whose outputs must be bit-identical (the per-pixel K loop does not depend on the
        tile shape).  Returns the widths run."""
        S = T + 2
        xs = (torch.randn(S, H, W, Cin, generator=g) * 0.5)
        ring = torch.zeros(S + 1, H, W, Cin, dtype=torch.bfloat16, device=dev)
        ring[:S] = xs.to(dev, torch.bfloat16)
        w = torch.randn(Cout, Cin, kt, kh, kw, generator=g) / math.sqrt(Cin * kt * kh * kw)
        b = torch.randn(Cout, generator=g) * 0.1
        cpad = (Cin + 63) // 64 * 64
        rows = (Cout + 15) // 16 * 16
        wp = torch.zeros(rows, kt, kh, kw, cpad)
        wp[:Cout, :, :, :, :Cin] = w.permute(0, 2, 3, 4, 1)
        wp = wp.reshape(rows, -1).to(dev, torch.bfloat16).contiguous()
        bias = torch.zeros(rows, device=dev)
        bias[:Cout] = b.to(dev)
        d = nv.ConvDesc()
        d.x_ring, d.ring_slots, d.in_H, d.in_W, d.C_in = ring.data_ptr(), S + 1, H, W, Cin
        d.w_packed, d.w_rows, d.w_ld = wp.data_ptr(), rows, wp.shape[1]
        d.kt, d.kh, d.kw, d.pad_h, d.pad_w = kt, kh, kw, pad, pad
        d.H, d.W, d.T = H, W, T
        for t in range(T):
            for a in range(kt):
                d.slot[t * 3 + a] = t + a + (3 - kt)   # frames t..t+2 of the ring are (t-2, t-1, t) of the stream
        d.C_out, d.tile_w = Cout, 8 if W <= 8 else 16
        d.variant = variant
        res = torch.randn(T, H, W, Cout, generator=g).to(dev) if residual else None
        if n_split:
            out = torch.full((2 * T, H, W, n_split), float("nan"), device=dev)
            d.out, d.out_frame_stride, d.out_ld = out.data_ptr(), 2 * out.stride(0), n_split
            d.n_split, d.split_offset = n_split, out.stride(0)
        else:
            out = torch.full((T, H, W, Cout), float("nan"), device=dev)
            d.out, d.out_frame_stride, d.out_ld = out.data_ptr(), out.stride(0), Cout
        d.bias = bias.data_ptr()
        if residual:
            d.residual, d.res_frame_stride, d.res_ld = res.data_ptr(), res.stride(0), Cout
        if fuse is not None:      # epilogue also produces the next conv's input: RMS norm + SiLU -> bf16 ring
            ncp = (Cout + 63) // 64 * 64
            nring = torch.zeros(T + 2, H, W, ncp, dtype=torch.bfloat16, device=dev)
            gamma = (torch.randn(Cout, generator=g) * 0.2 + 1).to(dev)
            d.next_ring, d.next_frame_stride, d.next_ld = nring.data_ptr(), nring.stride(0), ncp
            for t in range(T):
                d.next_slot[t] = (t + 1) % (T + 2)
            d.next_gamma, d.next_silu, d.write_f32 = gamma.data_ptr(), 1, 1 if fuse == "both" else 0
        xin = ring[:S].float().permute(3, 0, 1, 2).unsqueeze(0)        # [1,C,S,H,W]
        xin = xin[:, :, 3 - kt:] if kt < 3 else xin
        ref = F.conv3d(F.pad(xin, (pad, pad, pad, pad, 0, 0)) if kh == 3 else xin, w.to(dev).bfloat16().float(), b.to(dev))
        if kh == 2:   # 2x2 'valid' conv needs bottom/right zero pad to keep the output size (s2d down-sampling form)
            ref = F.conv3d(F.pad(xin, (0, 1, 0, 1, 0, 0)), w.to(dev).bfloat16().float(), b.to(dev))
        ref = ref[0].permute(1, 2, 3, 0)[:T]                           # [T,H,W,Cout]
        if residual:
            ref = ref + res
        want = F.silu(F.normalize(ref, dim=-1) * Cout ** 0.5 * gamma) if fuse is not None else None
        if n_split:
            ref = torch.stack([ref[..., :n_split], ref[..., n_split:]], dim=1).reshape(2 * T, H, W, n_split)
        if tile_w is None:
            widths = [8 if W <= 8 else 16]
        elif tile_w == "pick":
            from diffsynth.models.wan_video_vae import _pick_tile_w
            widths = [_pick_tile_w(H, W)]
        else:
            widths = [tile_w] if isinstance(tile_w, int) else list(tile_w)
        first = None
        for tw in widths:
            d.tile_w = tw
            out.fill_(float("nan"))
            if fuse is not None:
                nring.zero_()
            nv.conv3d_causal(d)
            torch.cuda.synchronize()
            wtag = f"{tag} tile_w={tw}" if tile_w is not None else tag
            if fuse is not None:
                got = torch.stack([nring[(t + 1) % (T + 2)] for t in range(T)])
                report(f"conv{wtag} fused next-input ({fuse}) Cin={Cin} Cout={Cout} T={T} {H}x{W} res={residual}",
                       got[..., :Cout].reshape(-1, Cout), want.reshape(-1, Cout), 2e-2)
                report(f"conv{wtag} fused next-input: padding channels and unused slots stay zero",
                       torch.cat([got[..., Cout:].reshape(-1), nring[0].reshape(-1)]).unsqueeze(0) + 1,
                       torch.ones(1, got[..., Cout:].numel() + nring[0].numel(), device=dev), 1e-7)
            if fuse is None or fuse == "both":
                report(f"conv{wtag} Cin={Cin} Cout={Cout} k=({kt},{kh},{kw}) T={T} {H}x{W} split={n_split} res={residual}",
                       out.reshape(-1, out.shape[-1]), ref.reshape(-1, ref.shape[-1]), 2e-2)
            outs = (out.clone(), nring.clone() if fuse is not None else None)
            if first is None:
                first = outs
                if tile_w is not None:     # negative control: the reference shifted by one pixel along W fails the bar
                    if fuse is None or fuse == "both":
                        negative(f"conv{wtag} reference shifted by one pixel", out.reshape(-1, out.shape[-1]),
                                 torch.roll(ref, 1, dims=-2).reshape(-1, ref.shape[-1]), 2e-2)
                    else:
                        negative(f"conv{wtag} fused next-input shifted by one pixel", got[..., :Cout].reshape(-1, Cout),
                                 torch.roll(want, 1, dims=-2).reshape(-1, Cout), 2e-2)
            else:
                same = torch.equal(outs[0].nan_to_num(7.0), first[0].nan_to_num(7.0)) and \
                    (fuse is None or torch.equal(outs[1], first[1]))
                print(f"[{'OK ' if same else 'BAD'}] conv{tag} tile_w={tw} bit-identical to tile_w={widths[0]}", flush=True)
                RESULTS.append((f"conv{tag} {H}x{W} tile_w={tw} bit-identical to tile_w={widths[0]}", same))
        return widths

    return run


def sec_conv():
    """svi_conv3d_causal against torch conv3d on hand-built frame rings."""
    run = _conv_runner()
    run(64, 96, 3, 3, 3, 2, 16, 16, 1)
    run(96, 96, 3, 3, 3, 1, 12, 20, 1, residual=True)
    run(384, 384, 3, 3, 3, 1, 8, 8, 1)
    run(192, 96, 1, 3, 3, 4, 20, 24, 1)
    run(384, 768, 3, 1, 1, 2, 6, 10, 0, n_split=384)
    run(192, 384, 1, 1, 1, 1, 9, 7, 0)
    run(384, 96, 1, 2, 2, 2, 10, 14, 0)
    run(64, 4, 3, 3, 3, 1, 4, 6, 1)
    run(96, 384, 3, 3, 3, 4, 30, 52, 1)
    run(96, 96, 3, 3, 3, 2, 20, 24, 1, fuse="only")
    run(192, 192, 3, 3, 3, 4, 12, 20, 1, residual=True, fuse="both")
    run(192, 96, 3, 3, 3, 1, 9, 7, 1, residual=True, fuse="both")
    # rows longer than one 128-pixel tile, ragged last tile, partial last channel chunk (96 = 64 + 32), two N tiles (384),
    # 2-D conv (k_t = 1); variant = 2 is accepted where k_w = 3 and pad_w = 1 and runs the same kernel
    run(64, 96, 3, 3, 3, 2, 6, 150, 1, variant=2)
    run(96, 96, 3, 3, 3, 1, 5, 200, 1, residual=True)
    run(96, 96, 3, 3, 3, 2, 4, 264, 1, fuse="only")
    run(192, 192, 3, 3, 3, 4, 3, 136, 1, residual=True, fuse="both")
    run(96, 384, 3, 3, 3, 1, 7, 130, 1)
    run(192, 96, 1, 3, 3, 3, 6, 257, 1)
    run(384, 384, 3, 3, 3, 1, 2, 40, 1, residual=True)
    run(96, 4, 3, 3, 3, 2, 5, 200, 1)          # decoder head: 3 (+1) output channels on an N = 16 tile
    run(16, 48, 3, 3, 3, 1, 4, 140, 1, fuse="both")


def sec_conv_tiles():
    """Every tile width of svi_conv3d_causal (BW x BH = 8x16, 16x8, 32x4, 64x2, 128x1) on H and W that are not multiples of
    the tile, with kt = 3 and 1, residual, the channel->frame split and the fused next input; the production geometries where
    the VAE picks 32, 64 or 128; and each descriptor at all five widths with bit-identical outputs (measured so on an H100
    80GB HBM3 at a 400 W power limit: fp32 output and fused bf16 next input identical for all six descriptors)."""
    from diffsynth.models.wan_video_vae import _pick_tile_w
    run = _conv_runner()
    every = (8, 16, 32, 64, 128)
    run(64, 96, 3, 3, 3, 2, 13, 150, 1, tile_w=every)
    run(96, 96, 1, 3, 3, 1, 11, 70, 1, residual=True, tile_w=every)
    run(384, 768, 3, 1, 1, 2, 6, 75, 0, n_split=384, tile_w=every)
    run(96, 96, 3, 3, 3, 2, 9, 100, 1, fuse="only", tile_w=every)
    run(192, 192, 3, 3, 3, 2, 7, 90, 1, residual=True, fuse="both", tile_w=every)
    run(16, 48, 3, 3, 3, 1, 5, 19, 1, fuse="both", tile_w=every)
    # where the VAE's tile choice is 32 (720p at 90x160 and 180x320), 64 (45-row band of a 320-wide stage) and 128 (45-row
    # band of a 640-wide stage, 720p on 8 ranks)
    for (H, W, want) in [(90, 160, 32), (180, 320, 32), (45, 320, 64), (45, 640, 128)]:
        got = _pick_tile_w(H, W)
        RESULTS.append((f"_pick_tile_w({H}, {W}) == {want}", got == want))
        run(16, 32, 3, 3, 3, 1, H, W, 1, residual=True, tile_w="pick")
    run(32, 16, 3, 3, 3, 2, 45, 640, 1, fuse="both", tile_w="pick")


def sec_perf_conv():
    """The convolution kernel at the VAE layer shapes that carry the FLOPs (480p decode), T = 4 frames per launch:
    mode 'mid' = first conv of a ResidualBlock (bf16 normalised output only), 'end' = second conv (+ fp32 residual, fp32 out and
    the next block's normalised input)."""
    g = torch.Generator(device="cpu").manual_seed(3)
    shapes = [(96, 96, 3, 480, 832), (192, 192, 3, 240, 416), (384, 384, 3, 120, 208), (384, 384, 3, 60, 104),
              (192, 96, 1, 480, 832), (96, 96, 3, 60, 832)]
    for Cin, Cout, kt, H, W in shapes:
        T, S = 4, 6
        ring = (torch.randn(S + 1, H, W, Cin, generator=g) * 0.5).to(dev, torch.bfloat16)
        cpad = (Cin + 63) // 64 * 64
        wp = (torch.randn(Cout, kt * 9 * cpad, generator=g) / math.sqrt(Cin * kt * 9)).to(dev, torch.bfloat16)
        bias = torch.zeros(Cout, device=dev)
        out = torch.empty(T, H, W, Cout, device=dev)
        res = torch.randn(T, H, W, Cout, device=dev)
        ncp = (Cout + 63) // 64 * 64
        nring = torch.zeros(T + 2, H, W, ncp, dtype=torch.bfloat16, device=dev)
        gamma = torch.ones(Cout, device=dev)
        fl = 2.0 * T * H * W * Cout * Cin * kt * 9
        for mode in ("mid", "end"):
            line = f"[PERF] conv {Cin}->{Cout} k=({kt},3,3) T={T} {H}x{W} {mode}:"
            d = nv.ConvDesc()
            d.x_ring, d.ring_slots, d.in_H, d.in_W, d.C_in = ring.data_ptr(), S + 1, H, W, Cin
            d.w_packed, d.w_rows, d.w_ld = wp.data_ptr(), Cout, wp.shape[1]
            d.kt, d.kh, d.kw, d.pad_h, d.pad_w = kt, 3, 3, 1, 1
            d.H, d.W, d.T = H, W, T
            for t in range(T):
                for a in range(kt):
                    d.slot[t * 3 + a] = t + a + (3 - kt)
            d.C_out = Cout
            from diffsynth.models.wan_video_vae import _pick_tile_w
            d.tile_w = _pick_tile_w(H, W)
            d.bias = bias.data_ptr()
            d.out_ld = Cout
            if Cout <= 256:
                d.next_ring, d.next_frame_stride, d.next_ld = nring.data_ptr(), nring.stride(0), ncp
            for t in range(T):
                d.next_slot[t] = t
            d.next_gamma, d.next_silu = gamma.data_ptr(), 1
            if mode == "end":
                d.out, d.out_frame_stride = out.data_ptr(), out.stride(0)
                d.residual, d.res_frame_stride, d.res_ld = res.data_ptr(), res.stride(0), Cout
                d.write_f32 = 1
            elif Cout <= 256:
                d.write_f32 = 0
            else:
                d.out, d.out_frame_stride, d.write_f32 = out.data_ptr(), out.stride(0), 1
            ms = time_ms(lambda: nv.conv3d_causal(d), iters=5, warm=2)
            line += f"  {ms * 1e3:.0f} us = {fl / ms / 1e9:.0f} TF/s"
            print(line, flush=True)
        del ring, wp, out, res, nring
        torch.cuda.empty_cache()


if __name__ == "__main__":
    print("device:", torch.cuda.get_device_name(0), "SMs:", nv.sm_count(), flush=True)
    for sec in sys.argv[1:]:
        print(f"=== {sec} ===", flush=True)
        t0 = time.time()
        globals()["sec_" + sec]()
        torch.cuda.synchronize()
        print(f"=== {sec} done in {time.time()-t0:.1f}s ===", flush=True)
