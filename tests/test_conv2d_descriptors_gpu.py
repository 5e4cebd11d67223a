"""svi_rife_conv2d and svi_esrgan_conv2d against an fp64 reference built from their descriptors alone.

The two 2-D instantiations of the conv mainloop (IFNet's and RRDBNet's) have their own epilogues.  The reference reads what
a descriptor points at, through its own pointers and pitches, builds the explicit im2col (images as ring slots, kt = 1) and
runs the header's epilogue.  Every launch is held to three bars:
  1. every output within a per-element fp64 bound: 2^-24 (2 K |A||W|^T) times the epilogue's Lipschitz factors (PReLU /
     LeakyReLU slope, residual scales) plus a few fp32 roundings of each term; a bf16 output within one bf16 ulp of
     bf16(v64) plus that floor, at most 1 % of it one ulp away; a uint8 output within 1 of trunc(clip(v64 * 255));
  2. every output bit-identical to svi_gemm_bf16 on the same im2col followed by the header's epilogue steps as separate
     torch fp32 ops (the epilogues contain no fused multiply-add), mapped to the destination (sub-pixel phase, space-to-
     depth channel, nearest x2, channel offset) and rounded to bf16 by round-to-nearest-even or truncated to uint8;
  3. nothing outside the described writes changes: pitch columns, image gaps, the channels of a shared in-place buffer
     outside the written window (the read window included), and the bytes past the last frame.
Explicit cases run at all five tile widths, bit-identical to tile_w = 8, and carry negative controls (a plausible wrong
reference that must fail its bar).  The engine tests record every launch of RIFEEngine.run and ESRGANEngine.run and check
each one.  test_conv2d_rejects_malformed_descriptors runs the host validation in a process that sees no GPU.
"""
import json
import os
import subprocess
import sys
import textwrap

import pytest
import torch

from diffsynth import _native as nv
from test_conv_descriptors_gpu import _bits, _region, _truncate_bf16, _view, im2col
from test_kernel_conformance_gpu import _bf16_inside

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = "cuda"
TILES = (8, 16, 32, 64, 128)
MAX_FLIP = 0.01
U = 2.0 ** -24                  # unit roundoff of fp32
U8_FILL = 0xA5                  # what a uint8 destination holds before the launch (there is no uint8 NaN)


def _ceil(a, b):
    return (a + b - 1) // b * b


def _locate(ptr, n, dtype, owners):
    """(flat tensor, element offset of ptr in it): the owning allocation when one of `owners` holds ptr (_region), which a
    uint8 pointer must have"""
    if dtype != torch.uint8:
        return _region(ptr, n, dtype, owners)
    for o in owners:
        base = o.data_ptr()
        if o.dtype == torch.uint8 and o.is_contiguous() and base <= ptr < base + o.numel():
            assert ptr - base + n <= o.numel()
            return o.view(-1), ptr - base
    raise AssertionError("a uint8 destination outside the buffers the test knows")


def _same_bits(a, b):
    return torch.equal(a, b) if a.dtype == torch.uint8 else torch.equal(_bits(a), _bits(b))


class _Target:
    """One output: flat buffer, element offset, and the index tensors [N, HW, cols] of each copy of the GEMM result"""

    def __init__(self, kind, ptr, idxs, owners, prefill=True):
        dtype = {"f32": torch.float32, "bf16": torch.bfloat16, "u8": torch.uint8}[kind]
        self.kind = kind
        self.buf, self.off = _locate(ptr, max(int(i.max()) for i in idxs) + 1, dtype, owners)
        self.idxs = [i + self.off for i in idxs]
        self.prefill = prefill

    def got(self, idxs=None):
        """the copies as [copies, N, HW, cols]; a control's wrong indices may point past the buffer, so they are clamped"""
        return torch.stack([self.buf[i.clamp(0, self.buf.numel() - 1)] for i in (idxs or self.idxs)])


class Launch2d:
    """One descriptor of either entry point: __init__ snapshots its operands and every buffer it touches, then fills the
    described writes with NaN (U8_FILL for uint8) unless an output is also read as a residual; check() applies bars 1-3."""

    def __init__(self, d, owners=()):
        torch.cuda.synchronize()
        self.d = d = type(d).from_buffer_copy(d)
        self.rife = isinstance(d, nv.RifeConvDesc)
        owners = list(owners)
        N, H, W = self.N, self.H, self.W = d.N, d.H, d.W
        self.HW = HW = H * W
        self.kh, self.kw = (d.kh, d.kw) if self.rife else (3, 3)
        self.pad_h, self.pad_w = (d.pad_h, d.pad_w) if self.rife else (1, 1)
        self.C_in, self.C_out = d.C_in, d.C_out
        self.ktot = self.kh * self.kw * _ceil(d.C_in, 64)
        C = d.C_out
        if self.rife:
            in_H, in_W = d.in_H, d.in_W
            self.x = _view(d.x, N * in_H * in_W * d.C_in, torch.bfloat16).view(N, in_H, in_W, d.C_in).clone()
        else:
            n = ((N * HW - 1) * d.in_ld + d.C_in)
            self.x = _view(d.x, n, torch.bfloat16).as_strided((N, H, W, d.C_in), (HW * d.in_ld, W * d.in_ld, d.in_ld, 1)).clone()
        self.wp = _view(d.w_packed, (d.w_rows - 1) * d.w_ld + self.ktot, torch.bfloat16) \
            .as_strided((C, self.ktot), (d.w_ld, 1)).clone()
        self.bias = _view(d.bias, C, torch.float32).clone()
        t_ = torch.arange(N, device=dev).view(N, 1, 1)
        p_ = torch.arange(HW, device=dev).view(1, HW, 1)
        n_ = torch.arange(C, device=dev).view(1, 1, C)
        self.g = dict(t=t_, y=p_ // W, x=p_ % W, n=n_)
        self.f32_idx = self.dst_f32()
        self.res = self.res2 = None
        if d.residual:
            self.res = _view(d.residual, int(self.f32_idx.max()) + 1, torch.float32)[self.f32_idx].clone()
        if self.rife:
            self.act = _view(d.prelu, C, torch.float32).clone() if d.prelu else None
        else:
            if d.residual2:
                self.res2 = _view(d.residual2, int(self.f32_idx.max()) + 1, torch.float32)[self.f32_idx].clone()
            self.act = d.slope if d.slope != 0.0 else None
        reads = {p for p in (d.residual, getattr(d, "residual2", None)) if p}
        self.targets = []
        if d.out:
            self.targets.append(_Target("f32", d.out, [self.f32_idx], owners, prefill=d.out not in reads))
        if d.out_bf16:
            self.targets.append(_Target("bf16", d.out_bf16, self.dst_bf16(), owners))
        if not self.rife and d.out_u8:
            self.targets.append(_Target("u8", d.out_u8, [self.dst_u8()], owners))
        # every buffer the launch reads or writes, as it was: bar 3 compares all of it outside the described writes
        self.watch = {}
        for tg in self.targets:
            self.watch.setdefault(tg.buf.data_ptr(), [tg.buf, tg.buf.clone(), []])[2].extend(tg.idxs)
        for ptr, n, dt in ((d.x, self.x.numel(), torch.bfloat16), (d.residual, 1, torch.float32),
                           (getattr(d, "residual2", None), 1, torch.float32)):
            if ptr:
                buf, _ = _locate(ptr, n, dt, owners)
                self.watch.setdefault(buf.data_ptr(), [buf, buf.clone(), []])
        for tg in self.targets:
            if tg.prefill:
                for i in tg.idxs:
                    tg.buf[i] = U8_FILL if tg.kind == "u8" else float("nan")

    # ------------------------------------------------------------------------------------------ destinations
    def dst_f32(self, swap_phase=False):
        d, g = self.d, self.g
        if self.rife:
            Y, X, c = self._rife_pixel(swap_phase)
            return g["t"] * d.out_img_stride + (Y * self.W * self.up + X) * d.out_ld + c
        return (g["t"] * self.HW + g["y"] * self.W + g["x"]) * d.f_ld + g["n"]

    @property
    def up(self):
        if self.rife:
            return 2 if self.d.C_out == 4 * self.d.phase_cols else 1
        return 2 if self.d.bf_up2 else 1

    def _rife_pixel(self, swap_phase=False):
        g, pc, up = self.g, self.d.phase_cols, self.up
        q, c = g["n"] // pc, g["n"] % pc
        dy, dx = (q & 1, q >> 1) if swap_phase else (q >> 1, q & 1)
        return g["y"] * up + dy, g["x"] * up + dx, c

    def dst_bf16(self, swap_phase=False, swap_s2d=False, shift_up2=False, channel_shift=0):
        """index tensors of the bf16 copies; the keyword arguments make the negative controls"""
        d, g, up = self.d, self.g, self.up
        Wd = self.W * up
        if self.rife:
            Y, X, c = self._rife_pixel(swap_phase)
            if d.bf_s2d:
                ph = (X & 1) * 2 + (Y & 1) if swap_s2d else (Y & 1) * 2 + (X & 1)
                return [g["t"] * d.bf_img_stride + ((Y >> 1) * (Wd >> 1) + (X >> 1)) * d.bf_ld + ph * d.phase_cols + c
                        + channel_shift]
            return [g["t"] * d.bf_img_stride + (Y * Wd + X) * d.bf_ld + c + channel_shift]
        out = []
        for dy in range(up):
            for dx in range(up):
                X = g["x"] * up + dx + (1 if shift_up2 else 0)
                out.append(((g["t"] * self.H * up + g["y"] * up + dy) * Wd + X.clamp(max=Wd - 1)) * d.bf_ld + g["n"]
                           + channel_shift)
        return out

    def dst_u8(self):
        g = self.g
        return (g["t"] * self.HW + g["y"] * self.W + g["x"]) * 3 + g["n"][..., :3]

    # ---------------------------------------------------------------------------------------------- fp64 reference
    def im2col(self, pad_h=None, drop_ci=None, x=None):
        x = self.x if x is None else x
        return im2col(x, [[t] for t in range(self.N)], self.H, self.W, self.kh, self.kw,
                      self.pad_h if pad_h is None else pad_h, self.pad_w, self.C_in, drop_ci)

    def acc64(self, a):
        return (a.double() @ self.wp.double().t()).view(self.N, self.HW, self.C_out)

    def epi64(self, acc, res_first=False, no_act=False):
        """the header's epilogue in fp64 (res_first, no_act: negative controls)"""
        v = acc + self.bias.double()
        if self.rife:
            if res_first and self.res is not None:
                v = v + self.res.double()
            if self.act is not None and not no_act:
                v = torch.where(v > 0, v, v * self.act.double())
            if self.res is not None and not res_first:
                v = v + self.res.double()
            return v
        if self.act is not None and not no_act:
            v = torch.where(v > 0, v, v * self.act)
        if self.res is not None:
            v = v * self.d.res_scale + self.res.double()
        if self.res2 is not None:
            v = v * self.d.res2_scale + self.res2.double()
        return v

    def bound(self, a, acc, v):
        P = (a.double().abs() @ self.wp.double().abs().t()).view(acc.shape)
        K = self.kh * self.kw * self.C_in
        if self.rife:
            L = self.act.double().abs().clamp_min(1.0) if self.act is not None else 1.0
        else:
            L = max(1.0, abs(self.act or 0.0)) * (max(1.0, abs(self.d.res_scale)) if self.res is not None else 1.0) * \
                (max(1.0, abs(self.d.res2_scale)) if self.res2 is not None else 1.0)
        terms = acc.abs() + self.bias.double().abs() + v.abs()
        for r in (self.res, self.res2):
            if r is not None:
                terms = terms + r.double().abs()
        return L * U * (2.0 * K * P + 4.0 * terms)

    # ------------------------------------------------------------------------------------- fp32 composition (bar 2)
    def gemm32(self, a):
        """svi_gemm_bf16 on the explicit im2col (N padded to a multiple of 8 with zero weight rows): RIFE with its bias, the
        accumulator alone for ESRGAN"""
        M, Np = a.shape[0], _ceil(self.C_out, 8)
        w = torch.zeros(Np, self.ktot, dtype=torch.bfloat16, device=dev)
        w[:self.C_out] = self.wp
        bias = None
        if self.rife:
            bias = torch.zeros(Np, device=dev)
            bias[:self.C_out] = self.bias
        out = torch.full((M, Np), float("nan"), device=dev)
        nv.gemm(a, w, out, bias=bias)
        return out[:, :self.C_out].reshape(self.N, self.HW, self.C_out)

    def epi32(self, g32, single_rounding=False):
        """the header's steps, one torch fp32 op each (single_rounding: the residual step as one fused rounding, a control)"""
        f = lambda s: torch.tensor(s, dtype=torch.float32, device=dev)
        if self.rife:
            v = g32
            if self.act is not None:
                v = torch.where(v > 0, v, v * self.act)
            if self.res is not None:
                v = v + self.res
            return v
        v = g32 + self.bias
        if self.act is not None:
            v = torch.where(v > 0, v, v * f(self.act))
        for r, s in ((self.res, self.d.res_scale), (self.res2, self.d.res2_scale)):
            if r is None:
                continue
            if single_rounding:
                v = (v.double() * s + r.double()).float()
            else:
                p = v * f(s)
                v = p + r
        return v

    @staticmethod
    def pack(tg, v32, truncate=False):
        if tg.kind == "f32":
            return v32
        if tg.kind == "bf16":
            return _truncate_bf16(v32) if truncate else v32.to(torch.bfloat16)
        return (v32[..., :3] * 255).clamp(0, 255).to(torch.uint8)

    # ---------------------------------------------------------------------------------------------------- bars
    def bar1(self, tg, v, bnd, got=None):
        """(ok, worst err/bound or share of flips) of one output against the fp64 value v"""
        got = tg.got() if got is None else got
        if tg.kind == "f32":
            err = (got.double() - v).abs()
            return bool((err <= bnd).all()), (err / bnd.clamp_min(1e-300)).max().item()
        if tg.kind == "bf16":
            ref = v.float().to(torch.bfloat16).expand_as(got)
            inside, _ = _bf16_inside(got, ref, bnd.float())
            flips = (got.float() != ref.float()).float().mean().item()
            return bool(inside.all()) and flips <= MAX_FLIP, flips
        ref = (v[..., :3] * 255).clamp(0, 255).trunc()
        err = (got.double() - ref).abs()
        return bool((err <= 1).all()), err.max().item()

    def bar2(self, tg, v32, truncate=False):
        want = self.pack(tg, v32, truncate)
        got = tg.got()
        return all(_same_bits(g.contiguous(), want.contiguous()) for g in got)

    def untouched(self):
        for buf, before, idxs in self.watch.values():
            keep = torch.ones_like(buf, dtype=torch.bool)
            for i in idxs:
                keep[i] = False
            if not _same_bits(buf[keep], before[keep]):
                return False
        return True

    def check(self, name, controls=False):
        """bars 1-3 after the launch; returns a dict of what was measured"""
        torch.cuda.synchronize()
        a = self.im2col()
        acc = self.acc64(a)
        v = self.epi64(acc)
        bnd = self.bound(a, acc, v)
        v32 = self.epi32(self.gemm32(a))
        r = dict(name=name, worst=0.0, flips=0.0, exact=0, outputs=len(self.targets))
        for tg in self.targets:
            ok, m = self.bar1(tg, v, bnd)
            key = {"f32": "worst", "bf16": "flips", "u8": "u8_err"}[tg.kind]
            r[key] = max(r.get(key, 0.0), m)
            assert ok, f"{name}: {tg.kind} output outside the fp64 bar ({key} {m:.3g})"
            exact = self.bar2(tg, v32)
            assert exact, f"{name}: {tg.kind} output differs from svi_gemm_bf16 + the epilogue's fp32 steps"
            r["exact"] += 1
        assert self.untouched(), f"{name}: the launch changed memory outside the described writes"
        if controls:
            r["controls"] = self.controls(a, v, bnd, v32)
        print(f"[OK ] {name}: worst err/bound={r['worst']:.3f} one-ulp flips={100 * r['flips']:.3f} % "
              f"bit-exact {r['exact']}/{r['outputs']}"
              + (f" controls caught={sorted(r['controls'])}" if controls else ""), flush=True)
        return r

    def controls(self, a, v, bnd, v32):
        """negative controls: each plausible wrong reference must fail its bar.  Returns the names of those that ran."""
        d = self.d
        ran = []

        def fails(name, wrong=None, dst=None):
            """bar 1 against a wrong fp64 value, or read through wrong destinations (dst(target): index tensors or None)"""
            caught = False
            for tg in self.targets:
                got = None
                if dst is not None:
                    idxs = dst(tg)
                    if idxs is None:
                        continue
                    got = tg.got([i + tg.off for i in idxs])
                caught |= not self.bar1(tg, v if wrong is None else wrong, bnd, got)[0]
            assert caught, f"control '{name}' passes bar 1"
            ran.append(name)

        def fails_exact(name, wrong32, truncate=False):
            """bar 2 against a wrong fp32 composition or a truncating bf16 pack"""
            caught = any(not self.bar2(tg, wrong32, truncate) for tg in self.targets if tg.kind == "bf16" or not truncate)
            assert caught, f"control '{name}' passes bar 2"
            ran.append(name)

        fails("pad_h + 1", self.epi64(self.acc64(self.im2col(pad_h=self.pad_h + 1))))
        real = (self.x != 0).flatten(0, 2).any(0).nonzero()
        fails("last input channel dropped", self.epi64(self.acc64(self.im2col(drop_ci=int(real.max())))))
        if self.rife and d.in_H > d.H:
            xh = self.x.reshape(-1)[:self.N * d.H * d.in_W * d.C_in].view(self.N, d.H, d.in_W, d.C_in)
            fails("in_H taken as H", self.epi64(self.acc64(self.im2col(x=xh))))
        acc = self.acc64(a)
        if self.rife and self.up == 2:
            fails("phase dy/dx swapped", dst=lambda tg: [self.dst_f32(swap_phase=True)] if tg.kind == "f32"
                  else self.dst_bf16(swap_phase=True))
        if self.rife and d.out_bf16 and d.bf_s2d:
            fails("s2d phase order swapped", dst=lambda tg: self.dst_bf16(swap_s2d=True) if tg.kind == "bf16" else None)
        if not self.rife and d.out_bf16:
            if d.bf_up2:
                fails("x2 replication shifted one pixel",
                      dst=lambda tg: self.dst_bf16(shift_up2=True) if tg.kind == "bf16" else None)
            fails("bf16 channel offset off by 2", dst=lambda tg: self.dst_bf16(channel_shift=2) if tg.kind == "bf16" else None)
        if self.rife and self.res is not None and self.act is not None:
            fails("residual added before PReLU", self.epi64(acc, res_first=True))
        if not self.rife and self.act is not None:
            fails("slope ignored", self.epi64(acc, no_act=True))
        if any(tg.kind == "bf16" for tg in self.targets):
            fails_exact("truncating bf16 pack", v32, truncate=True)
        if not self.rife and self.res is not None:
            fails_exact("residual step rounded once", self.epi32(self.gemm32(a), single_rounding=True))
        return ran


# ------------------------------------------------------------------------------------------------- explicit descriptors
def _weights(g, C_out, taps, C_in, real_cin, bufs, scale=1.0):
    """packed bf16 weight: junk (finite) in the padding channels, NaN in the rows past C_out and the columns past the taps"""
    cpad = _ceil(C_in, 64)
    ktot = taps * cpad
    w_rows, w_ld = C_out + 3, ktot + 8
    wp = torch.full((w_rows, w_ld), float("nan"))
    t = torch.randn(C_out, taps, cpad, generator=g) * scale
    t[:, :, :real_cin] /= (taps * real_cin) ** 0.5
    wp[:C_out, :ktot] = t.reshape(C_out, ktot)
    bufs["w"] = wp.to(dev, torch.bfloat16)
    return bufs["w"].data_ptr(), w_rows, w_ld


def _rife_case(g, *, N, H, W, C_in, C_out, pc=None, kh=3, kw=None, pad_h=1, pad_w=None, in_H=None, in_W=None, real_cin=None,
               prelu=True, residual=None, out=True, out_ld=None, out_gap=0, bf=False, bf_ld=None, s2d=0, bf_gap=0):
    """residual: None, "sep" (its own buffer in out's layout) or "alias" (= out)"""
    kw, pad_w, pc = kh if kw is None else kw, pad_h if pad_w is None else pad_w, C_out if pc is None else pc
    in_H, in_W = H if in_H is None else in_H, W if in_W is None else in_W
    real_cin = C_in if real_cin is None else real_cin
    up = 2 if C_out == 4 * pc else 1
    Hd, Wd = H * up, W * up
    bufs = {}
    x = (torch.randn(N, in_H, in_W, C_in, generator=g) * 0.5).to(torch.bfloat16)
    x[..., real_cin:] = 0
    bufs["x"] = x.to(dev)
    d = nv.RifeConvDesc()
    d.x, d.N, d.in_H, d.in_W, d.C_in = bufs["x"].data_ptr(), N, in_H, in_W, C_in
    d.w_packed, d.w_rows, d.w_ld = _weights(g, C_out, kh * kw, C_in, real_cin, bufs)
    d.kh, d.kw, d.pad_h, d.pad_w, d.H, d.W = kh, kw, pad_h, pad_w, H, W
    d.C_out, d.phase_cols = C_out, pc
    bufs["bias"] = (torch.randn(C_out, generator=g) * 0.1).to(dev)
    d.bias = bufs["bias"].data_ptr()
    if prelu:
        bufs["prelu"] = (torch.rand(C_out, generator=g) * 1.5 - 0.25).to(dev)     # negative slopes and slopes above 1 too
        d.prelu = bufs["prelu"].data_ptr()
    out_ld = pc if out_ld is None else out_ld
    d.out_ld, d.out_img_stride = out_ld, Hd * Wd * out_ld + out_gap
    if out or residual == "alias":
        bufs["out"] = torch.randn(N * d.out_img_stride + 6, generator=g).to(dev)
        d.out = bufs["out"].data_ptr()
    if residual == "sep":
        bufs["res"] = torch.randn(N * d.out_img_stride, generator=g).to(dev)
        d.residual = bufs["res"].data_ptr()
    elif residual == "alias":
        d.residual = d.out
    if bf:
        bf_ld = (4 * pc if s2d else pc) if bf_ld is None else bf_ld
        d.bf_ld, d.bf_s2d = bf_ld, s2d
        d.bf_img_stride = Hd * Wd // (4 if s2d else 1) * bf_ld + bf_gap
        bufs["bf"] = torch.randn(N * d.bf_img_stride + 6, generator=g).to(dev, torch.bfloat16)
        d.out_bf16 = bufs["bf"].data_ptr()
    return d, bufs


def _esrgan_case(g, *, N, H, W, C_in, C_out, in_ld=None, x_off=0, real_cin=None, slope=0.2, res=None, res2=None,
                 out=True, f_ld=None, bf=None, bf_ld=None, bf_off=0, u8=False):
    """res / res2: None, "sep" or "alias" (= out); bf: None, "other" (a buffer of its own at channel offset bf_off), "same"
    (x's buffer just past the read window) or "up2" (nearest x2); u8: a conv_last-like launch with values around [0, 1]"""
    in_ld = C_in if in_ld is None else in_ld
    real_cin = C_in if real_cin is None else real_cin
    bufs = {}
    xb = torch.randn(N, H, W, in_ld, generator=g) * 0.5
    xb[..., x_off + real_cin:x_off + C_in] = 0
    bufs["x"] = xb.to(dev, torch.bfloat16)
    d = nv.EsrganConvDesc()
    d.x, d.N, d.H, d.W, d.C_in, d.in_ld = bufs["x"].data_ptr() + 2 * x_off, N, H, W, C_in, in_ld
    d.w_packed, d.w_rows, d.w_ld = _weights(g, C_out, 9, C_in, real_cin, bufs, scale=0.5 if u8 else 1.0)
    d.C_out, d.slope = C_out, slope
    bufs["bias"] = (torch.randn(C_out, generator=g) * 0.2 + (0.5 if u8 else 0.0)).to(dev)
    d.bias = bufs["bias"].data_ptr()
    d.f_ld = C_out if f_ld is None else f_ld
    n32 = N * H * W * d.f_ld
    if out or "alias" in (res, res2):
        bufs["out"] = torch.randn(n32 + 6, generator=g).to(dev)
        d.out = bufs["out"].data_ptr()
    for k, (kind, s) in {"residual": (res, 0.2), "residual2": (res2, -0.75)}.items():
        if kind == "sep":
            bufs[k] = torch.randn(n32, generator=g).to(dev)
            setattr(d, k, bufs[k].data_ptr())
        elif kind == "alias":
            setattr(d, k, d.out)
        setattr(d, "res_scale" if k == "residual" else "res2_scale", s)
    if bf == "same":
        d.out_bf16, d.bf_ld = d.x + 2 * C_in, in_ld
    elif bf is not None:
        up = 2 if bf == "up2" else 1
        d.bf_ld, d.bf_up2 = bf_ld, int(bf == "up2")
        bufs["bf"] = torch.randn(N * up * H * up * W * bf_ld + 6, generator=g).to(dev, torch.bfloat16)
        d.out_bf16 = bufs["bf"].data_ptr() + 2 * bf_off
    if u8:
        bufs["u8"] = torch.randint(0, 256, (N * H * W * 3 + 64,), generator=g, dtype=torch.uint8).to(dev)
        d.out_u8 = bufs["u8"].data_ptr()
    return d, bufs


RIFE_CASES = {
    # IFNet's conv0a: 2x2 taps, pad 1 over the 48-channel s2d block input (44 real), written as the next conv's s2d operand;
    # 4 x 8 x 12 tiles at tile_w = 8 (and more at the other widths): the persistent loop wraps
    "conv0a kh=2 pad=1 s2d C_out=46": dict(N=4, H=64, W=94, C_in=48, real_cin=44, C_out=46, kh=2, out=False, bf=True, s2d=1),
    "C_out=90 f32 out_ld=94 + bf16 bf_ld=100": dict(N=3, H=37, W=45, C_in=96, real_cin=90, C_out=90, out_ld=94, bf=True,
                                                   bf_ld=100),
    "residual aliasing out": dict(N=2, H=19, W=27, C_in=96, real_cin=90, C_out=90, residual="alias", out_ld=90, bf=True,
                                  bf_ld=96),
    "residual with out=NULL": dict(N=2, H=21, W=17, C_in=96, real_cin=90, C_out=90, residual="sep", out=False, out_ld=92,
                                   bf=True, bf_ld=96),
    # two N tiles of 192: phase 2 (columns 180..269) straddles the tile boundary
    "four phases of 90 (C_out=360)": dict(N=2, H=13, W=22, C_in=96, real_cin=90, C_out=360, pc=90, out=False, bf=True,
                                          bf_ld=96),
    "four phases of 6 f32 out_ld=8": dict(N=4, H=24, W=41, C_in=96, real_cin=90, C_out=24, pc=6, prelu=False, out_ld=8),
    "four phases residual + s2d bf16": dict(N=2, H=11, W=15, C_in=64, C_out=40, pc=10, residual="sep", out_ld=12, bf=True,
                                            bf_ld=44, s2d=1),
    "in_H=H+3 in_W=W-2 C_in=8": dict(N=3, H=17, W=23, in_H=20, in_W=21, C_in=8, C_out=32, out_ld=34),
    "kh=1 kw=3 pad_h=0 pad_w=2 C_in=184": dict(N=2, H=18, W=26, C_in=184, real_cin=180, C_out=64, kh=1, kw=3, pad_h=0,
                                              pad_w=2, bf=True, bf_ld=66),
    "kh=3 kw=2 pad 2/1 C_in=128 image gaps": dict(N=3, H=14, W=19, C_in=128, C_out=48, kh=3, kw=2, pad_h=2, pad_w=1,
                                                  out_ld=50, out_gap=38, bf=True, bf_ld=52, bf_gap=22),
    "single tile kh=kw=1": dict(N=1, H=5, W=7, C_in=64, C_out=16, kh=1, pad_h=0, residual="sep", bf=True),
}

ESRGAN_CASES = {
    "C_out=2 f_ld=6": dict(N=3, H=21, W=29, C_in=8, C_out=2, slope=0.0, f_ld=6),
    # conv_last: 3 x 6 x 17 tiles at tile_w = 8, the persistent loop wraps
    "C_out=4 uint8 + f32 (conv_last)": dict(N=3, H=84, W=131, C_in=64, C_out=4, slope=0.0, u8=True),
    "C_out=32 in place just past the read window": dict(N=2, H=37, W=45, C_in=96, in_ld=192, C_out=32, out=False,
                                                        bf="same"),
    "C_out=64 both residuals, out aliasing residual2": dict(N=2, H=29, W=19, C_in=192, C_out=64, slope=0.0, res="sep",
                                                            res2="alias", bf="other", bf_ld=192),
    # three N tiles of 64, the last one partial; x at channel 16 of a 64-channel pixel
    "C_out=130 x at channel offset, out aliasing residual, up2 bf_ld=136": dict(
        N=2, H=13, W=22, C_in=40, in_ld=64, x_off=16, C_out=130, res="alias", f_ld=132, bf="up2", bf_ld=136),
    "C_out=96 all three outputs": dict(N=2, H=9, W=35, C_in=64, C_out=96, slope=0.0, res="sep", res2="sep", f_ld=98,
                                       bf="other", bf_ld=104, bf_off=6, u8=True),
    "single tile C_out=64 up2": dict(N=1, H=6, W=7, C_in=64, C_out=64, bf="up2", bf_ld=64),
}


def _run_explicit(kind, name, spec):
    """bars 1-3 and the controls at tile_w = 8, every buffer of the other four widths bit-identical to it"""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    d, bufs = (_rife_case if kind == "rife" else _esrgan_case)(g, **spec)
    launch = nv.rife_conv2d_desc if kind == "rife" else nv.esrgan_conv2d_desc
    owners = list(bufs.values())
    init = {k: v.clone() for k, v in bufs.items()}
    first = None
    for tw in TILES:
        for k, v in init.items():
            bufs[k].copy_(v)
        d.tile_w = tw
        L = Launch2d(d, owners)
        launch(d)
        if first is None:
            L.check(f"{kind} {name} tile_w={tw}", controls=True)
            first = {k: v.clone() for k, v in bufs.items()}
        else:
            torch.cuda.synchronize()
            same = all(_same_bits(bufs[k], v) for k, v in first.items())
            print(f"[{'OK ' if same else 'BAD'}] {kind} {name} tile_w={tw} bit-identical to tile_w={TILES[0]}", flush=True)
            assert same, f"{name}: tile_w={tw} differs from tile_w={TILES[0]}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RIFE_CASES))
def test_rife_descriptor_case(name):
    _run_explicit("rife", name, RIFE_CASES[name])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ESRGAN_CASES))
def test_esrgan_descriptor_case(name):
    _run_explicit("esrgan", name, ESRGAN_CASES[name])


# ------------------------------------------------------------------------------------------------ the engines, launch by launch
class Recorder:
    """Stands in for nv.rife_conv2d_desc / nv.esrgan_conv2d_desc: snapshots, launches the kernel, applies bars 1-3, and lets
    the engine carry on with the kernel's own outputs.  Keeps the descriptor of every launch."""

    def __init__(self, launch_fn, owners):
        self.launch_fn, self.owners, self.seen, self.worst, self.flips = launch_fn, owners, [], 0.0, 0.0
        self.exact = self.outputs = 0

    def __call__(self, d):
        L = Launch2d(d, self.owners())
        self.launch_fn(d)
        r = L.check(f"launch {len(self.seen)}")
        self.worst, self.flips = max(self.worst, r["worst"]), max(self.flips, r["flips"])
        self.exact += r["exact"]
        self.outputs += r["outputs"]
        self.seen.append(type(d).from_buffer_copy(d))

    def summary(self, what):
        print(f"[OK ] {what}: {len(self.seen)} launches, worst err/bound={self.worst:.3f} max one-ulp flips="
              f"{100 * self.flips:.3f} % bit-exact {self.exact}/{self.outputs} outputs", flush=True)


def _rife_model():
    from diffsynth.extensions.RIFE import IFNet
    from tools import synth_rife
    m = IFNet().eval()
    m.load_state_dict(synth_rife.make_state_dict(seed=0))
    return m.to(dev)


@pytest.mark.gpu
def test_rife_engine_launches(monkeypatch):
    """every conv launch of RIFEEngine.run (two pairs at 64 x 96, scale 1.0 and 0.5) against the fp64 reference of its own
    descriptor; the engine's result bit-identical to a run without the recorder"""
    eng = _rife_model().engine(dev)
    frames = torch.rand(3, 64, 96, 4, generator=torch.Generator().manual_seed(7)).to(dev)
    lists = ([4.0, 2.0, 1.0], [8.0, 4.0, 2.0])
    plain = [eng.run(frames[:-1], frames[1:], sl).clone() for sl in lists]
    rec = Recorder(nv.rife_conv2d_desc, lambda: [t for B in eng._bufs.values() for t in B.values()])
    monkeypatch.setattr(nv, "rife_conv2d_desc", rec)
    for sl, want in zip(lists, plain):
        got = eng.run(frames[:-1], frames[1:], sl)
        assert torch.equal(_bits(got), _bits(want)), f"scale list {sl}: the recorded run differs from the plain one"
    rec.summary("RIFEEngine.run conv launches")
    seen = rec.seen
    counts = {
        "s2d bf16 copy": sum(bool(d.out_bf16) and d.bf_s2d == 1 for d in seen),
        "four phases C_out=360": sum(d.C_out == 360 and d.phase_cols == 90 for d in seen),
        "four phases f32 out": sum(d.C_out == 4 * d.phase_cols and bool(d.out) for d in seen),
        "out aliasing residual": sum(bool(d.residual) and d.out == d.residual for d in seen),
        "residual, out=NULL": sum(bool(d.residual) and not d.out for d in seen),
        "kh": {k: sum(d.kh == k for d in seen) for k in (2, 3)},
        "tile_w": {t: sum(d.tile_w == t for d in seen) for t in TILES if any(d.tile_w == t for d in seen)},
    }
    print(f"      recorded geometries: {json.dumps(counts)}", flush=True)
    # a later change to the engine must not quietly stop covering one of these
    for k in ("s2d bf16 copy", "four phases C_out=360", "four phases f32 out", "out aliasing residual", "residual, out=NULL"):
        assert counts[k], f"RIFEEngine no longer launches: {k}"


@pytest.mark.gpu
def test_esrgan_engine_launches(monkeypatch):
    """every conv launch of ESRGANEngine.run (RRDBNet with two RRDBs, three 21 x 29 frames, uint8 and f32 conv_last) against
    the fp64 reference of its own descriptor; the engine's outputs bit-identical to a run without the recorder"""
    from diffsynth.extensions.ESRGAN import LAST_COLS, RRDBNet
    from tools import synth_esrgan
    m = RRDBNet(num_block=2).eval()
    m.load_state_dict(synth_esrgan.make_state_dict(2, seed=0))
    eng = m.to(dev).engine(dev)
    N, H, W = 3, 21, 29
    u8 = torch.randint(0, 256, (N, H, W, 3), generator=torch.Generator().manual_seed(8), dtype=torch.uint8).to(dev)

    def run():
        rgb = torch.empty(N, 4 * H, 4 * W, 3, dtype=torch.uint8, device=dev)
        out = torch.empty(N, 4 * H, 4 * W, LAST_COLS, device=dev)
        nv.esrgan_stage_frames(u8, eng.buffers(N, H, W)["x"])
        eng.run(N, H, W, rgb=rgb, out=out)
        return rgb, out

    plain = run()
    holder = {}
    rec = Recorder(nv.esrgan_conv2d_desc, lambda: list(eng._bufs[(N, H, W)].values()) + list(holder.values()))
    rgb = torch.empty(N, 4 * H, 4 * W, 3, dtype=torch.uint8, device=dev)
    out = torch.empty(N, 4 * H, 4 * W, LAST_COLS, device=dev)
    holder.update(rgb=rgb, out=out)
    monkeypatch.setattr(nv, "esrgan_conv2d_desc", rec)
    nv.esrgan_stage_frames(u8, eng.buffers(N, H, W)["x"])
    eng.run(N, H, W, rgb=rgb, out=out)
    assert torch.equal(rgb, plain[0]) and torch.equal(_bits(out), _bits(plain[1])), \
        "the recorded run differs from the plain one"
    rec.summary("ESRGANEngine.run conv launches")
    seen = rec.seen
    inplace = sorted({(d.out_bf16 - d.x) // 2 for d in seen if d.out_bf16 and 0 < d.out_bf16 - d.x < 2 * d.in_ld})
    counts = {
        "in-place channel offsets": inplace,
        "out aliasing residual": sum(bool(d.residual) and d.out == d.residual for d in seen),
        "out aliasing residual2": sum(bool(d.residual2) and d.out == d.residual2 for d in seen),
        "bf_up2": sum(bool(d.out_bf16) and d.bf_up2 == 1 for d in seen),
        "uint8 + f32": sum(bool(d.out_u8) and bool(d.out) for d in seen),
    }
    print(f"      recorded geometries: {json.dumps(counts)}", flush=True)
    assert {64, 96, 128, 160} <= set(inplace), "the dense blocks no longer write in place at every growth offset"
    assert counts["out aliasing residual"] and counts["out aliasing residual2"]
    assert counts["bf_up2"] == 2 and counts["uint8 + f32"] == 1


# ----------------------------------------------------------------------------------------------------- host validation
_REJECT_SCRIPT = textwrap.dedent(r"""
    import ctypes, json
    from diffsynth import _native as nv
    lib = nv.load()

    # fake device pointers, 256-byte aligned: with no device visible nothing is ever dereferenced
    def rife():
        d = nv.RifeConvDesc()
        d.x, d.N, d.in_H, d.in_W, d.C_in = 0x100000, 2, 16, 16, 64
        d.w_packed, d.w_rows, d.w_ld = 0x200000, 96, 9 * 64
        d.kh = d.kw = 3
        d.pad_h = d.pad_w = 1
        d.H = d.W = 16
        d.C_out, d.phase_cols, d.tile_w = 96, 96, 16
        d.bias, d.prelu, d.residual = 0x300000, 0x400000, 0x500000
        d.out, d.out_img_stride, d.out_ld = 0x600000, 256 * 96, 96
        d.out_bf16, d.bf_img_stride, d.bf_ld, d.bf_s2d = 0x700000, 64 * 4 * 96, 4 * 96, 1
        return d

    def esrgan():
        d = nv.EsrganConvDesc()
        d.x, d.N, d.H, d.W, d.C_in, d.in_ld = 0x100000, 2, 8, 8, 64, 128
        d.w_packed, d.w_rows, d.w_ld = 0x200000, 64, 9 * 64
        d.C_out, d.tile_w = 64, 16
        d.bias, d.slope = 0x300000, 0.2
        d.residual, d.res_scale, d.residual2, d.res2_scale = 0x400000, 0.2, 0x500000, 0.2
        d.out, d.f_ld = 0x600000, 64
        d.out_bf16, d.bf_ld, d.bf_up2 = 0x700000, 64, 1
        d.out_u8 = 0x800000
        return d

    def s(**kw):
        return lambda d: [setattr(d, k, v) for k, v in kw.items()]

    # mutation name -> (mutation, the words of the rule the message must contain)
    RIFE = {
        "baseline": (s(), None),
        "x = NULL": (s(x=None), "null pointer"),
        "bias = NULL": (s(bias=None), "null pointer"),
        "no output": (s(out=None, out_bf16=None), "null pointer"),
        "N = 0": (s(N=0), "must be > 0"),
        "in_W = 0": (s(in_W=0), "must be > 0"),
        "kw = 4": (s(kw=4), "kernel extents must be in [1,3]"),
        "pad_h = kh": (s(pad_h=3), "0 <= pad < extent"),
        "pad_w = -1": (s(pad_w=-1), "0 <= pad < extent"),
        "C_in = 60": (s(C_in=60), "C_in must be a multiple of 8"),
        "x misaligned": (s(x=0x100008), "x and w_packed must be 16-byte aligned"),
        "w_packed misaligned": (s(w_packed=0x200008), "x and w_packed must be 16-byte aligned"),
        "phase_cols odd": (s(phase_cols=7), "phase_cols must be even"),
        "C_out = 2 phases": (s(phase_cols=48), "phase_cols must be even"),
        "tile_w = 12": (s(tile_w=12), "tile_w must be 8, 16, 32, 64 or 128"),
        "w_rows < C_out": (s(w_rows=95), "packed weight"),
        "w_ld short": (s(w_ld=9 * 64 - 8), "packed weight"),
        "bias misaligned": (s(bias=0x300004), "bias and prelu must be 8-byte aligned"),
        "prelu misaligned": (s(prelu=0x400004), "bias and prelu must be 8-byte aligned"),
        "out misaligned": (s(out=0x600004), "out and residual must be 8-byte aligned"),
        "residual misaligned": (s(residual=0x500004), "out and residual must be 8-byte aligned"),
        "out_ld odd": (s(out_ld=97), "out_ld must be even and >= phase_cols"),
        "out_ld short": (s(out_ld=94), "out_ld must be even and >= phase_cols"),
        "out_img_stride odd": (s(out_img_stride=256 * 96 + 1), "out_img_stride even and >= one image"),
        "out_img_stride short": (s(out_img_stride=256 * 96 - 2), "out_img_stride even and >= one image"),
        "out_bf16 misaligned": (s(out_bf16=0x700002), "out_bf16 must be 4-byte aligned"),
        "bf_s2d = 2": (s(bf_s2d=2), "bf_s2d must be 0 or 1"),
        "s2d onto an odd grid": (s(H=15, in_H=15, out_img_stride=15 * 16 * 96), "space-to-depth copy needs an even destination"),
        "bf_ld odd": (s(bf_ld=4 * 96 + 1), "bf_ld must be even and hold every channel"),
        "bf_ld short": (s(bf_ld=4 * 96 - 2), "bf_ld must be even and hold every channel"),
        "bf_img_stride odd": (s(bf_img_stride=64 * 4 * 96 + 1), "bf_img_stride even and >= one image"),
        "bf_img_stride short": (s(bf_img_stride=64 * 4 * 96 - 2), "bf_img_stride even and >= one image"),
        "too many tiles": (s(N=1 << 30), "too many tiles"),
    }
    ESRGAN = {
        "baseline": (s(), None),
        "x = NULL": (s(x=None), "null pointer"),
        "w_packed = NULL": (s(w_packed=None), "null pointer"),
        "bias = NULL": (s(bias=None), "null pointer"),
        "no output": (s(out=None, out_bf16=None, out_u8=None), "null pointer"),
        "H = 0": (s(H=0), "N, H, W must be > 0"),
        "N = -1": (s(N=-1), "N, H, W must be > 0"),
        "C_in = 60": (s(C_in=60), "need C_in % 8 == 0, in_ld % 8 == 0 and in_ld >= C_in"),
        "in_ld = 100": (s(in_ld=100), "need C_in % 8 == 0, in_ld % 8 == 0 and in_ld >= C_in"),
        "in_ld < C_in": (s(in_ld=56), "need C_in % 8 == 0, in_ld % 8 == 0 and in_ld >= C_in"),
        "x misaligned": (s(x=0x100008), "x and w_packed must be 16-byte aligned"),
        "w_packed misaligned": (s(w_packed=0x200008), "x and w_packed must be 16-byte aligned"),
        "C_out odd": (s(C_out=63), "C_out must be even and > 0"),
        "tile_w = 256": (s(tile_w=256), "tile_w must be 8, 16, 32, 64 or 128"),
        "w_rows < C_out": (s(w_rows=62), "packed weight"),
        "w_ld odd": (s(w_ld=9 * 64 + 4), "packed weight"),
        "bias misaligned": (s(bias=0x300004), "bias must be 8-byte aligned"),
        "out misaligned": (s(out=0x600004), "out, residual and residual2 must be 8-byte aligned"),
        "residual misaligned": (s(residual=0x400004), "out, residual and residual2 must be 8-byte aligned"),
        "residual2 misaligned": (s(residual2=0x500004), "out, residual and residual2 must be 8-byte aligned"),
        "f_ld odd": (s(f_ld=65, C_out=62), "f_ld must be even and >= C_out"),
        "f_ld < C_out": (s(f_ld=62), "f_ld must be even and >= C_out"),
        "out_bf16 misaligned": (s(out_bf16=0x700002), "out_bf16 must be 4-byte aligned"),
        "bf_up2 = 2": (s(bf_up2=2), "bf_up2 must be 0 or 1"),
        "bf_ld < C_out": (s(bf_ld=62), "bf_ld must be even and >= C_out"),
        "bf_ld odd": (s(bf_ld=65), "bf_ld must be even and >= C_out"),
        "bf16 in x with up2": (s(out_bf16=0x100000 + 2 * 64), "must lie in x's buffer with its pixel layout"),
        "bf16 in x with another pitch": (s(out_bf16=0x100000 + 2 * 64, bf_up2=0, bf_ld=96),
                                         "must lie in x's buffer with its pixel layout"),
        "bf16 before x, overlapping": (s(out_bf16=0x100000 - 64, bf_up2=0), "must lie in x's buffer with its pixel layout"),
        "bf16 in the read window": (s(out_bf16=0x100000 + 2 * 32, bf_up2=0, bf_ld=128), "lies inside the input's read window"),
        "bf16 past the pixel": (s(out_bf16=0x100000 + 2 * 96, bf_up2=0, bf_ld=128), "lies inside the input's read window"),
        "uint8 with C_out = 2": (s(C_out=2), "a uint8 RGB output needs C_out >= 3"),
        "too many tiles": (s(N=1 << 30, H=16, out_bf16=None), "too many tiles"),
    }
    res = {}
    for entry, base, muts in (("svi_rife_conv2d", rife, RIFE), ("svi_esrgan_conv2d", esrgan, ESRGAN)):
        fn = getattr(lib, entry)
        for name, (mut, rule) in muts.items():
            d = base()
            mut(d)
            rc = fn(ctypes.byref(d), None)
            res[f"{entry}: {name}"] = [rc, lib.svi_last_error().decode(), rule]
    print(json.dumps(res))
""")


def test_conv2d_rejects_malformed_descriptors():
    """Every rule svi_rife_conv2d and svi_esrgan_conv2d check is reached by one malformed descriptor and refused before
    any CUDA call, with a message naming the rule.  Runs in a process that sees no GPU, so a missing check fails with a
    different (later) message and can never reach a launch; the unchanged descriptors get past validation."""
    if not os.path.exists(nv.lib_path()):
        pytest.skip("the kernel library is not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]))
    p = subprocess.run([sys.executable, "-c", _REJECT_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    bad = []
    for name, (rc, msg, rule) in res.items():
        print(f"{name}: status {rc}: {msg}")
        entry = name.split(":")[0]
        if rule is None:
            if rc in (0, -1):
                bad.append(f"{name}: the unchanged descriptor should pass validation and fail later without a GPU ({msg})")
        elif rc != -1 or not msg.startswith(entry + ":") or rule not in msg:
            bad.append(f"{name}: not rejected by its rule '{rule}' ({rc}: {msg})")
    assert not bad, "\n".join(bad)
