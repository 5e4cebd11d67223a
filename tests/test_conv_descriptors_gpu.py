"""svi_conv3d_causal against an fp64 reference built from its descriptor alone.

The reference reads what the descriptor points at, through the descriptor's own pointers and strides, and builds the
explicit im2col the header describes (row = (t, h, w), column = ((a*kh + b)*kw + c)*ceil64(C_in) + ci, zero outside the
ring frame and for ci >= C_in).  Every launch is held to four bars:
  1. the fp32 output within a per-element fp64 bound, c K 2^-24 (|A||W|^T) plus a few roundings of the epilogue terms (the
     formula of tools/gpu_check._gemm_bound_report);
  2. the fp32 output bit-identical to svi_gemm_bf16 on the same im2col (both walk K in the same 64-wide chunks of
     m64nNk16 wgmma steps from a zero accumulator, then add bias and residual in fp32);
  3. the fused next input (RMS norm, SiLU, bf16) within one bf16 ulp of the fp64 value, at most 1 % of it one ulp away, and
     bit-identical whether or not the fp32 output is also written;
  4. nothing outside the described writes changes: columns [C_out, out_ld), next-ring channels [C_out, next_ld), slots the
     launch does not name and halo rows.
The explicit cases cover geometry the engines launch or the ABI accepts, each at all five tile widths; every kind of case
carries negative controls (a plausible wrong reference that must fail its bar).  The engine test records every launch of
the VAE (plain and one-rank sharded) and of the SVI-Dance pose stem and checks each one.  test_conv_rejects_* runs the
host validation in a process that sees no GPU.
"""
import json
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

from diffsynth import _native as nv
from test_kernel_conformance_gpu import ULP32, _bf16_inside

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = "cuda"
TILES = (8, 16, 32, 64, 128)
MAX_FLIP = 0.01
_ELEM = {torch.float32: 4, torch.bfloat16: 2}
_BITS = {torch.float32: torch.int32, torch.bfloat16: torch.int16}


def _ceil(a, b):
    return (a + b - 1) // b * b


class _DeviceMemory:
    """n elements at a raw device address, for torch.as_tensor (the descriptor carries pointers, as the C ABI sees them)"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "strides": None,
                                         "version": 2}


def _view(ptr, n, dtype):
    if dtype == torch.bfloat16:
        return torch.as_tensor(_DeviceMemory(ptr, n, "<i2"), device=dev).view(torch.bfloat16)
    return torch.as_tensor(_DeviceMemory(ptr, n, "<f4"), device=dev)


def _region(ptr, n, dtype, owners):
    """(flat tensor, element offset of ptr in it): the owning allocation when one of `owners` holds ptr, so that what lies
    around the described extent (halo rows, other slots) can be checked too; else the n elements at ptr"""
    for o in owners:
        base, size = o.data_ptr(), o.numel() * o.element_size()
        if o.dtype == dtype and o.is_contiguous() and base <= ptr < base + size:
            off = (ptr - base) // _ELEM[dtype]
            assert (ptr - base) % _ELEM[dtype] == 0 and off + n <= o.numel()
            return o.view(-1), off
    return _view(ptr, n, dtype), 0


def _bits(t):
    return t.view(_BITS[t.dtype])


def im2col(ring, slot_rows, H, W, kh, kw, pad_h, pad_w, C_in, drop_ci=None):
    """bf16 [T*H*W, kt*kh*kw*ceil64(C_in)] from the header's semantics: ring[slot[t*3+a], h+b-pad_h, w+c-pad_w, ci], zero
    outside [0,in_H) x [0,in_W) and for ci >= C_in"""
    S, in_H, in_W, _ = ring.shape
    d = ring.device
    T, kt = len(slot_rows), len(slot_rows[0])
    hh = torch.arange(H, device=d)[:, None] + torch.arange(kh, device=d)[None, :] - pad_h          # [H, kh]
    ww = torch.arange(W, device=d)[:, None] + torch.arange(kw, device=d)[None, :] - pad_w          # [W, kw]
    inside = (((hh >= 0) & (hh < in_H))[:, :, None, None] & ((ww >= 0) & (ww < in_W))[None, None])  # [H, kh, W, kw]
    fr = ring[torch.tensor(slot_rows, device=d)]                                                   # [T, kt, in_H, in_W, C]
    x = fr[:, :, hh.clamp(0, in_H - 1)[:, :, None, None], ww.clamp(0, in_W - 1)[None, None]]       # [T, kt, H, kh, W, kw, C]
    x = torch.where(inside[None, None, ..., None], x, torch.zeros((), dtype=x.dtype, device=d))
    if drop_ci is not None:
        x[..., drop_ci] = 0
    a = torch.zeros(T, H, W, kt, kh, kw, _ceil(C_in, 64), dtype=torch.bfloat16, device=d)
    a[..., :C_in] = x.permute(0, 2, 4, 1, 3, 5, 6)
    return a.reshape(T * H * W, -1)


class Launch:
    """One descriptor: __init__ snapshots its operands and the memory it may write (and prefills the described writes with
    NaN), check() applies bars 1-4 after the launch."""

    def __init__(self, d, owners=()):
        torch.cuda.synchronize()
        self.d = d = nv.ConvDesc.from_buffer_copy(d)
        self.T, self.H, self.W = T, H, W = d.T, d.H, d.W
        self.kt, self.kh, self.kw, self.C_in, self.C_out = d.kt, d.kh, d.kw, d.C_in, d.C_out
        C_out, HW = self.C_out, H * W
        self.slot_rows = [[d.slot[t * 3 + a] for a in range(d.kt)] for t in range(T)]
        self.ktot = d.kt * d.kh * d.kw * _ceil(d.C_in, 64)
        self.ring = _view(d.x_ring, d.ring_slots * d.in_H * d.in_W * d.C_in, torch.bfloat16) \
            .view(d.ring_slots, d.in_H, d.in_W, d.C_in).clone()
        self.wp = _view(d.w_packed, (d.w_rows - 1) * d.w_ld + self.ktot, torch.bfloat16) \
            .as_strided((C_out, self.ktot), (d.w_ld, 1)).clone()
        self.bias = _view(d.bias, C_out, torch.float32).clone() if d.bias else None
        self.gamma = _view(d.next_gamma, C_out, torch.float32).clone() if (d.next_ring and d.next_gamma) else None
        t_ = torch.arange(T, device=dev).view(T, 1, 1)
        p_ = torch.arange(HW, device=dev).view(1, HW, 1)
        n_ = torch.arange(C_out, device=dev).view(1, 1, C_out)
        self.res = None
        if d.residual:
            ridx = t_ * d.res_frame_stride + p_ * d.res_ld + n_
            self.res = _view(d.residual, int(ridx.max()) + 1, torch.float32)[ridx].clone()
        self.writes_out = not d.next_ring or bool(d.write_f32)
        self.out = None
        if self.writes_out:
            split = d.n_split > 0
            oidx = t_ * d.out_frame_stride + p_ * d.out_ld + \
                (torch.where(n_ >= d.n_split, d.split_offset + n_ - d.n_split, n_) if split else n_)
            self.out = self._target(d.out, oidx, torch.float32, owners)
        self.nxt = None
        if d.next_ring:
            nslot = torch.tensor([d.next_slot[t] for t in range(T)], device=dev).view(T, 1, 1)
            nidx = nslot * d.next_frame_stride + p_ * d.next_ld + n_
            self.nxt = self._target(d.next_ring, nidx, torch.bfloat16, owners)

    @staticmethod
    def _target(ptr, idx, dtype, owners):
        buf, off = _region(ptr, int(idx.max()) + 1, dtype, owners)
        idx = idx + off
        before = buf.clone()
        buf[idx] = float("nan")
        return dict(buf=buf, idx=idx, before=before)

    # ---------------------------------------------------------------------------------------------- fp64 reference
    def v64(self, slot_rows=None, pad_h=None, drop_ci=None, bias=True, want_operands=False):
        """conv + bias + residual in fp64 [T, H*W, C_out]; the keyword arguments make the negative controls"""
        d = self.d
        a = im2col(self.ring, slot_rows or self.slot_rows, self.H, self.W, self.kh, self.kw,
                   d.pad_h if pad_h is None else pad_h, d.pad_w, self.C_in, drop_ci)
        v = a.double() @ self.wp.double().t()
        if self.bias is not None and bias:
            v = v + self.bias.double()
        v = v.view(self.T, self.H * self.W, self.C_out)
        if self.res is not None:
            v = v + self.res.double()
        return (v, a) if want_operands else v

    def bound(self, a, v):
        """per-element bound of bar 1 (gpu_check._gemm_bound_report with c = 2, K = the terms that can be non-zero)"""
        P = (a.double().abs() @ self.wp.double().abs().t()).view(v.shape)
        epi = (self.bias.double().abs() if self.bias is not None else 0.0) + \
            (self.res.double().abs() if self.res is not None else 0.0)
        K = self.kt * self.kh * self.kw * self.C_in
        return 2.0 ** -24 * (2.0 * K * P + 4 * (epi + v.abs()))

    def y64(self, v, gamma=True):
        d = self.d
        y = v
        if self.gamma is not None and gamma:
            y = v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12) * self.C_out ** 0.5 * self.gamma.double()
        return F.silu(y) if d.next_silu else y

    def next_floor(self, v, bnd, y):
        """a few fp32 ulps of the pixel's scale, plus what the bar-1 bound on v moves the normalised value by"""
        lip = 1.1 if self.d.next_silu else 1.0            # |silu'| <= 1.0998
        if self.gamma is not None:
            s = self.C_out ** 0.5 / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)
            rel = bnd.norm(dim=-1, keepdim=True) / v.norm(dim=-1, keepdim=True).clamp_min(1e-300)
            move = lip * self.gamma.double().abs() * s * (bnd + v.abs() * rel)
        else:
            move = lip * bnd
        return 4 * ULP32 * y.abs().amax(dim=-1, keepdim=True) + move

    # ---------------------------------------------------------------------------------------------------- bars
    def got_out(self):
        return self.out["buf"][self.out["idx"]]

    def got_next(self):
        return self.nxt["buf"][self.nxt["idx"]]

    @staticmethod
    def out_bar(got, v, bnd):
        err = (got.double() - v).abs()
        return bool((err <= bnd).all()), (err / bnd.clamp_min(1e-300)).max().item()

    @staticmethod
    def next_bar(got, y, floor):
        ref = y.float().to(torch.bfloat16)
        inside, _ = _bf16_inside(got.reshape(-1, got.shape[-1]), ref.reshape(-1, ref.shape[-1]),
                                 floor.reshape(-1, floor.shape[-1]).float())
        flips = (got.float() != ref.float()).float().mean().item()
        return bool(inside.all()) and flips <= MAX_FLIP, flips

    @staticmethod
    def untouched(t):
        keep = torch.ones_like(t["buf"], dtype=torch.bool)
        keep[t["idx"]] = False
        return torch.equal(_bits(t["buf"])[keep], _bits(t["before"])[keep])

    def check(self, name, launch_fn, controls=False):
        """bars 1-4 after the launch; returns a dict of what was measured"""
        torch.cuda.synchronize()
        d = self.d
        v, a = self.v64(want_operands=True)
        bnd = self.bound(a, v)
        r = dict(name=name)
        if self.writes_out:
            ok, r["worst"] = self.out_bar(self.got_out(), v, bnd)
            assert ok, f"{name}: fp32 output outside the fp64 bound (worst err/bound {r['worst']:.3g})"
            assert self.untouched(self.out), f"{name}: the launch wrote fp32 memory outside the described output"
            r["gemm_identical"] = self.gemm_identical(a)
            assert r["gemm_identical"], f"{name}: fp32 output differs from svi_gemm_bf16 on the same im2col"
        if self.nxt is not None:
            y = self.y64(v)
            floor = self.next_floor(v, bnd, y)
            got = self.got_next()
            ok, r["flips"] = self.next_bar(got, y, floor)
            assert ok, f"{name}: fused next input beyond one bf16 ulp of fp64 (flips {100 * r['flips']:.3f} %)"
            assert self.untouched(self.nxt), f"{name}: the launch wrote next-ring memory outside the described pixels"
            assert self.other_write_f32_same(launch_fn), f"{name}: next ring depends on write_f32"
        if controls:
            r["controls"] = self.controls(v, bnd)
        print(f"[OK ] conv {name}: worst err/bound={r.get('worst', float('nan')):.3f} "
              f"one-ulp flips={100 * r.get('flips', 0.0):.3f} % gemm bit-identical={r.get('gemm_identical')}"
              + (f" controls caught={sorted(r['controls'])}" if controls else ""), flush=True)
        return r

    def gemm_identical(self, a):
        """bar 2: svi_gemm_bf16 on the explicit im2col (N padded to the GEMM's multiple of 8 with zero weight rows)"""
        M, N = a.shape[0], _ceil(self.C_out, 8)
        w = torch.zeros(N, self.ktot, dtype=torch.bfloat16, device=dev)
        w[:self.C_out] = self.wp
        bias = res = None
        if self.bias is not None:
            bias = torch.zeros(N, device=dev)
            bias[:self.C_out] = self.bias
        if self.res is not None:
            res = torch.zeros(M, N, device=dev)
            res[:, :self.C_out] = self.res.reshape(M, self.C_out)
        out = torch.full((M, N), float("nan"), device=dev)
        nv.gemm(a, w, out, bias=bias, residual=res)
        torch.cuda.synchronize()
        return torch.equal(_bits(out[:, :self.C_out].contiguous()), _bits(self.got_out().reshape(M, self.C_out).contiguous()))

    def other_write_f32_same(self, launch_fn):
        """the same descriptor with write_f32 flipped, into scratch next-ring and output memory: bit-identical next input"""
        d = nv.ConvDesc.from_buffer_copy(self.d)
        T, HW, C = self.T, self.H * self.W, self.C_out
        slots = [self.d.next_slot[t] for t in range(T)]
        lo, nfs = min(slots), self.d.next_frame_stride
        scratch = torch.zeros((max(slots) - lo) * nfs + HW * self.d.next_ld, dtype=torch.bfloat16, device=dev)
        out = torch.empty(T * HW * C, device=dev)
        d.next_ring = scratch.data_ptr()
        for t in range(T):
            d.next_slot[t] = slots[t] - lo
        d.write_f32 = 0 if self.d.write_f32 else 1
        d.out, d.out_frame_stride, d.out_ld = out.data_ptr(), HW * C, C
        launch_fn(d)
        torch.cuda.synchronize()
        idx = (torch.tensor(slots, device=dev).view(T, 1, 1) - lo) * nfs + \
            torch.arange(HW, device=dev).view(1, HW, 1) * self.d.next_ld + torch.arange(C, device=dev).view(1, 1, C)
        return torch.equal(_bits(scratch[idx]), _bits(self.got_next()))

    def controls(self, v, bnd):
        """negative controls: each plausible wrong reference must fail its bar.  Returns the names of those that ran."""
        d = self.d
        ran = []

        def out_fails(name, wrong):
            if self.writes_out:
                assert not self.out_bar(self.got_out(), wrong, bnd)[0], f"control '{name}' passes the fp32 bar"
            if self.nxt is not None:
                y = self.y64(wrong)
                assert not self.next_bar(self.got_next(), y, self.next_floor(v, bnd, y))[0], \
                    f"control '{name}' passes the next-input bar"
            ran.append(name)

        # tap a = 0 read from the nearest slot whose contents differ
        rows = [list(r) for r in self.slot_rows]
        for r in rows:
            s = r[0]
            for k in (1, -1, 2, -2, 3, -3):
                s2 = (s + k) % d.ring_slots
                if not torch.equal(self.ring[s2], self.ring[s]):
                    r[0] = s2
                    break
        out_fails("neighbour slot", self.v64(slot_rows=rows))
        out_fails("pad_h + 1", self.v64(pad_h=d.pad_h + 1))
        real = (self.ring != 0).flatten(0, 2).any(0).nonzero()
        out_fails("last input channel dropped", self.v64(drop_ci=int(real.max())))
        if self.bias is not None and self.bias.abs().max() > 0:
            out_fails("bias left out", self.v64(bias=False))
        if self.nxt is not None:
            got = self.got_next()
            if self.gamma is not None:
                y = self.y64(v, gamma=False)
                assert not self.next_bar(got, y, self.next_floor(v, bnd, y))[0], "control 'next_gamma ignored' passes"
                ran.append("next_gamma ignored")
            y = self.y64(v)
            trunc = _truncate_bf16(y.float())
            assert not self.next_bar(trunc, y, self.next_floor(v, bnd, y))[0], "control 'truncating bf16' passes"
            ran.append("truncating bf16")
        return ran


def _truncate_bf16(x):
    """bf16 by dropping the low 16 bits (rounding toward zero): what a pack that truncates would store"""
    return (x.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------- explicit descriptors
def _case(g, *, C_in, C_out, table, ring_slots, kh=3, kw=3, pad_h=1, pad_w=1, H=9, W=13, in_H=None, real_cin=None,
          bias=True, residual=None, out_ld=None, n_split=0, fuse=None):
    """Buffers and descriptor of one explicit case.  residual = (res_ld, res_frame_stride); fuse = dict(gamma, silu, halo):
    the next ring has `halo` rows above and below the pixels and the descriptor points one halo into each slot.  Packed
    weights hold junk in the padding channels (finite: the ring's zero fill multiplies them), NaN in the rows beyond C_out and
    in the columns beyond the taps."""
    T, kt = len(table), len(table[0])
    in_H = H if in_H is None else in_H
    in_W = W
    real_cin = C_in if real_cin is None else real_cin
    HW = H * W
    bufs = {}
    ring = (torch.randn(ring_slots, in_H, in_W, C_in, generator=g) * 0.5).to(torch.bfloat16)
    ring[..., real_cin:] = 0
    ring[-1] = 0                                             # the all-zero slot of the engines' rings
    bufs["ring"] = ring.to(dev)
    cpad = _ceil(C_in, 64)
    ktot = kt * kh * kw * cpad
    w_rows, w_ld = C_out + 4, ktot + 8
    wp = torch.full((w_rows, w_ld), float("nan"))
    taps = torch.randn(C_out, kt * kh * kw, cpad, generator=g)
    taps[:, :, :real_cin] /= (kt * kh * kw * real_cin) ** 0.5
    wp[:C_out, :ktot] = taps.reshape(C_out, ktot)
    bufs["w"] = wp.to(dev, torch.bfloat16)
    d = nv.ConvDesc()
    d.x_ring, d.ring_slots, d.in_H, d.in_W, d.C_in = bufs["ring"].data_ptr(), ring_slots, in_H, in_W, C_in
    d.w_packed, d.w_rows, d.w_ld = bufs["w"].data_ptr(), w_rows, w_ld
    d.kt, d.kh, d.kw, d.pad_h, d.pad_w = kt, kh, kw, pad_h, pad_w
    d.H, d.W, d.T = H, W, T
    for t in range(T):
        for a in range(kt):
            d.slot[t * 3 + a] = table[t][a]
    d.C_out = C_out
    out_ld = C_out if out_ld is None else out_ld
    if n_split:
        bufs["out"] = torch.full((2 * T * HW * out_ld,), float("nan"), device=dev)
        d.out, d.out_frame_stride, d.out_ld = bufs["out"].data_ptr(), 2 * HW * out_ld, out_ld
        d.n_split, d.split_offset = n_split, HW * out_ld
    else:
        bufs["out"] = torch.full((T * HW * out_ld,), float("nan"), device=dev)
        d.out, d.out_frame_stride, d.out_ld = bufs["out"].data_ptr(), HW * out_ld, out_ld
    if bias:
        bufs["bias"] = (torch.randn(C_out, generator=g) * 0.1).to(dev)
        d.bias = bufs["bias"].data_ptr()
    if residual is not None:
        res_ld, rfs = residual
        bufs["res"] = torch.randn(T * rfs, generator=g).to(dev)
        d.residual, d.res_frame_stride, d.res_ld = bufs["res"].data_ptr(), rfs, res_ld
    if fuse is not None:
        halo, next_ld, nslots = fuse.get("halo", 0), C_out + 12, T + 3
        rows = H + 2 * halo
        bufs["next"] = torch.zeros(nslots * rows * W * next_ld, dtype=torch.bfloat16, device=dev)
        d.next_ring = bufs["next"].data_ptr() + 2 * halo * W * next_ld
        d.next_frame_stride, d.next_ld = rows * W * next_ld, next_ld
        for t in range(T):
            d.next_slot[t] = (2 * t + 1) % nslots               # slots 0, 2, ... stay unnamed (for T < 3)
        if fuse["gamma"]:
            bufs["gamma"] = (torch.randn(C_out, generator=g) * 0.2 + 1).to(dev)
            d.next_gamma = bufs["gamma"].data_ptr()
        d.next_silu = fuse["silu"]
        d.write_f32 = 1
    return d, bufs


Z = 6   # the all-zero slot of a 7-slot ring (6 slots + zero), as the engines' rings of 4 + CACHE_T slots
CASES = {
    # VAE under spatial sharding: halo rows in the input ring, the 3x3x3 conv of a ResidualBlock with its skip and the next
    # conv's input written one row into its slots; a wrapped table
    "halo in_H=H+2 pad_h=0 3x3x3 res+fused": dict(C_in=96, C_out=96, table=[[4, 5, 0], [5, 0, 1]], ring_slots=7, in_H=11,
                                                 pad_h=0, residual=(96, 9 * 13 * 96), fuse=dict(gamma=True, silu=1, halo=1)),
    # the sharded 2x2 space-to-depth downsample: pad_h = -1
    "halo in_H=H+2 pad_h=-1 2x2": dict(C_in=128, C_out=96, table=[[3], [4], [5], [0]], ring_slots=7, in_H=11, kh=2, kw=2,
                                      pad_h=-1, pad_w=0),
    # the pose stem: 2x2 taps with pad 1 over the s2d "before" packing, temporal stride 2 with the zero slot at both ends,
    # 16 real channels of 64
    "pose 2x2 pad=1 stride-2 table": dict(C_in=64, real_cin=16, C_out=16, table=[[Z, 0, 1], [1, 2, 3], [3, 4, Z]], ring_slots=7,
                                        kh=2, kw=2),
    # the pose stem's first conv: 3 real channels of 64; four frames of a wrapped table
    "C_in=64 (3 real) T=4 wrapped": dict(C_in=64, real_cin=3, C_out=16, table=[[3, 4, 5], [4, 5, 0], [5, 0, 1], [0, 1, 2]],
                                        ring_slots=7),
    # first chunk of a causal stream: the zero slot twice
    "C_in=8 C_out=12 T=1 repeated zero slot": dict(C_in=8, C_out=12, table=[[Z, Z, 0]], ring_slots=7),
    "C_in=24 C_out=20 bias=NULL out_ld=C_out+8": dict(C_in=24, C_out=20, table=[[Z, 0, 1], [0, 1, 2]], ring_slots=7, bias=False,
                                                     out_ld=28),
    "C_in=56 C_out=4 fused gamma=NULL silu=0": dict(C_in=56, C_out=4, table=[[Z, Z, 0], [Z, 0, 1], [0, 1, 2]], ring_slots=7,
                                                   fuse=dict(gamma=False, silu=0)),
    "C_in=72 C_out=100 res_ld/res_frame_stride != out": dict(C_in=72, C_out=100, table=[[1, 2, 3], [2, 3, 4]], ring_slots=7,
                                                            residual=(106, 9 * 13 * 106 + 38), out_ld=108),
    "C_in=136 C_out=260 kt=1 T=4": dict(C_in=136, C_out=260, table=[[5], [0], [1], [2]], ring_slots=7),
    "C_in=64 C_out=400 3x1x1 res": dict(C_in=64, C_out=400, table=[[Z, 0, 1], [0, 1, 2]], ring_slots=7, kh=1, kw=1, pad_h=0,
                                       pad_w=0, residual=(400, 9 * 13 * 400)),
    "C_out=768 n_split=384 3x1x1 (time_conv)": dict(C_in=96, C_out=768, table=[[5, 0, 1], [0, 1, 2]], ring_slots=7, kh=1, kw=1,
                                                   pad_h=0, pad_w=0, n_split=384, out_ld=384),
    "C_in=64 C_out=100 fused gamma=NULL silu=1": dict(C_in=64, C_out=100, table=[[2, 3, 4]], ring_slots=7,
                                                     fuse=dict(gamma=False, silu=1, halo=1)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_conv_descriptor_case(name):
    """one explicit descriptor: bars 1-4 and the negative controls at tile_w = 8, the outputs of the other four widths (and,
    for fused cases, of write_f32 = 0) bit-identical to it"""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    d, bufs = _case(g, **CASES[name])
    owners = [b for b in bufs.values()]
    first = None
    for tw in TILES:
        d.tile_w = tw
        bufs["out"].fill_(float("nan"))
        if "next" in bufs:
            bufs["next"].zero_()
        L = Launch(d, owners)
        nv.conv3d_causal(d)
        if first is None:
            L.check(f"{name} tile_w={tw}", nv.conv3d_causal, controls=True)
            first = {k: bufs[k].clone() for k in ("out", "next") if k in bufs}
        else:
            torch.cuda.synchronize()
            same = all(torch.equal(_bits(bufs[k]), _bits(v)) for k, v in first.items())
            print(f"[{'OK ' if same else 'BAD'}] conv {name} tile_w={tw} bit-identical to tile_w={TILES[0]}", flush=True)
            assert same, f"{name}: tile_w={tw} differs from tile_w={TILES[0]}"


# ------------------------------------------------------------------------------------------------ the engines, launch by launch
class Recorder:
    """Stands in for nv.conv3d_causal: snapshots, launches the kernel, applies bars 1-4, and lets the engine carry on with the
    kernel's own outputs.  Keeps the geometry of every launch."""

    def __init__(self, launch_fn, owners=lambda: ()):
        self.launch_fn, self.owners, self.seen, self.worst, self.flips = launch_fn, owners, [], 0.0, 0.0
        self.gemm_identical = self.f32_launches = 0

    def __call__(self, d):
        L = Launch(d, list(self.owners()))
        self.launch_fn(d)
        r = L.check(f"launch {len(self.seen)}", self.launch_fn)
        self.worst = max(self.worst, r.get("worst", 0.0))
        self.flips = max(self.flips, r.get("flips", 0.0))
        self.gemm_identical += bool(r.get("gemm_identical"))
        self.f32_launches += L.writes_out
        zero = d.ring_slots - 1
        table = L.slot_rows
        self.seen.append(dict(
            pad_h=d.pad_h, halo_ring=d.in_H == d.H + 2, kh=d.kh, pad_w=d.pad_w, T=d.T, n_split=d.n_split,
            wrapped=any(any(b <= a for a, b in zip(r_, r_[1:])) for r_ in ([s for s in row if s != zero] for row in table)),
            zero_repeated=sum(s == zero for row in table for s in row) >= 2))


class _OneRankShard:
    """SpatialShard of a one-process group: rank 0 of 1, no neighbours, gathers are the identity"""
    rank, world, group, up, down = 0, 1, None, None, None

    def band(self, latent_rows):
        self.bounds = [0, latent_rows]
        self._latent_rows = latent_rows
        return 0, latent_rows

    def total_rows(self, my_rows):
        return my_rows

    def gather_rows(self, local, full, H, W):
        full[:local.shape[0]] = local
        return full

    def gather_bands(self, t, dim, scale):
        return t


@pytest.mark.gpu
def test_engine_launches(monkeypatch):
    """every conv launch of the tiny-weight VAE (encode 9 frames at 32x48 and decode its latents, unsharded and as a one-rank
    shard) and of the pose stem (5 frames at 32x48) against the fp64 reference of its own descriptor"""
    from diffsynth.models import wan_video_vae as V
    from diffsynth.models.dwpose_embedding import DWPoseEmbeddingEngine, make_dwpose_embedding
    from tools import synth_vae
    sd = {k: v.to(torch.bfloat16).float() if v.dim() > 1 and "gamma" not in k else v
          for k, v in synth_vae.make_vae_state_dict(seed=0).items()}
    vae = V.WanVideoVAE().eval()
    vae.load_state_dict(sd)
    vae.to(dev)
    eng = vae.engine(dev)
    rec = Recorder(nv.conv3d_causal, owners=lambda: [r.buf for r in eng.rings.values()])
    monkeypatch.setattr(nv, "conv3d_causal", rec)
    video = (torch.rand(3, 9, 32, 48, generator=torch.Generator().manual_seed(6)) * 2 - 1).to(dev)
    eng.shard = None
    lat = eng.encode(video)
    dec = eng.decode(lat)
    n_plain = len(rec.seen)
    eng.shard = _OneRankShard()
    lat1 = eng.encode(video)
    dec1 = eng.decode(lat)
    eng.shard = None
    assert torch.equal(lat1, lat), "one-rank-sharded encode differs from the unsharded one"
    assert torch.equal(dec1, dec), "one-rank-sharded decode differs from the unsharded one"
    n_vae = len(rec.seen)
    g = torch.Generator().manual_seed(64)
    seq = make_dwpose_embedding(dim=64)
    seq.load_state_dict({k: (torch.randn(v.shape, generator=g) * (1.5 / v[0].numel() ** 0.5 if k.endswith("weight") else 0.1))
                         .to(torch.bfloat16).float() for k, v in seq.state_dict().items()})
    pose = torch.rand(3, 5, 32, 48, generator=g)
    DWPoseEmbeddingEngine(seq, dev).forward(pose)
    seen = rec.seen
    counts = {
        "launches (vae, vae one-rank shard, pose stem)": (n_plain, n_vae - n_plain, len(seen) - n_vae),
        "pad_h": {p: sum(s["pad_h"] == p for s in seen) for p in sorted({s["pad_h"] for s in seen})},
        "in_H = H + 2": sum(s["halo_ring"] for s in seen),
        "wrapped slot table": sum(s["wrapped"] for s in seen),
        "zero slot repeated": sum(s["zero_repeated"] for s in seen),
        "kh = 2, pad = 1": sum(s["kh"] == 2 and s["pad_h"] == 1 and s["pad_w"] == 1 for s in seen),
        "n_split > 0": sum(s["n_split"] > 0 for s in seen),
        "T": {t: sum(s["T"] == t for s in seen) for t in range(1, 5)},
    }
    print(f"[OK ] engine conv launches: worst err/bound={rec.worst:.3f} max one-ulp flips={100 * rec.flips:.3f} % "
          f"gemm bit-identical={rec.gemm_identical}/{rec.f32_launches}", flush=True)
    print(f"      recorded geometries: {json.dumps(counts)}", flush=True)
    # a later change to the engines must not quietly stop covering one of these
    assert {-1, 0, 1} <= set(counts["pad_h"])
    assert counts["in_H = H + 2"] and counts["wrapped slot table"] and counts["zero slot repeated"]
    assert counts["kh = 2, pad = 1"] and counts["n_split > 0"]
    assert all(counts["T"][t] for t in range(1, 5))


# ----------------------------------------------------------------------------------------------------- host validation
_REJECT_SCRIPT = textwrap.dedent(r"""
    import ctypes, json, sys
    from diffsynth import _native as nv
    lib = nv.load()
    HW, C = 64, 96

    def base():
        # fake device pointers, 256-byte aligned: with no device visible nothing is ever dereferenced
        d = nv.ConvDesc()
        d.x_ring, d.ring_slots, d.in_H, d.in_W, d.C_in = 0x100000, 3, 8, 8, 64
        d.w_packed, d.w_rows, d.w_ld = 0x200000, C, 27 * 64
        d.kt, d.kh, d.kw, d.pad_h, d.pad_w = 3, 3, 3, 1, 1
        d.H, d.W, d.T = 8, 8, 2
        for i, s in enumerate([0, 1, 2, 1, 2, 0]):
            d.slot[i] = s
        d.C_out, d.tile_w = C, 16
        d.out, d.out_frame_stride, d.out_ld = 0x300000, HW * C, C
        d.bias = 0x400000
        d.residual, d.res_frame_stride, d.res_ld = 0x500000, HW * C, C
        d.next_ring, d.next_frame_stride, d.next_ld = 0x600000, HW * C, C
        d.next_slot[0], d.next_slot[1] = 0, 1
        d.next_gamma, d.next_silu, d.write_f32 = 0x700000, 1, 1
        return d

    def split(d, n_split, split_offset, out_ld):
        d.next_ring = None
        d.n_split, d.split_offset, d.out_ld, d.out_frame_stride = n_split, split_offset, out_ld, 2 * HW * out_ld

    MUT = {
        "baseline": lambda d: None,
        "n_split": lambda d: split(d, 47, HW * 48, 48),
        "split_offset": lambda d: split(d, 48, HW * 48 + 1, 48),
        "out_frame_stride": lambda d: setattr(d, "out_frame_stride", HW * C + 1),
        "res_ld": lambda d: setattr(d, "res_ld", C + 1),
        "res_ld ": lambda d: setattr(d, "res_ld", C - 2),
        "res_frame_stride": lambda d: setattr(d, "res_frame_stride", HW * C + 1),
        "next_frame_stride": lambda d: setattr(d, "next_frame_stride", HW * C + 1),
        "out": lambda d: setattr(d, "out", 0x300004),
        "residual": lambda d: setattr(d, "residual", 0x500004),
        "bias": lambda d: setattr(d, "bias", 0x400004),
        "next_ring": lambda d: setattr(d, "next_ring", 0x600002),
        "next_gamma": lambda d: setattr(d, "next_gamma", 0x700004),
        "out_ld": lambda d: setattr(d, "out_ld", C - 4),
        "out_ld ": lambda d: split(d, 32, HW * 64, 60),
    }
    res = {}
    for name, mut in MUT.items():
        d = base()
        mut(d)
        rc = lib.svi_conv3d_causal(ctypes.byref(d), None)
        res[name] = [rc, lib.svi_last_error().decode()]
    print(json.dumps(res))
""")


def test_conv_rejects_what_the_epilogue_cannot_store():
    """Descriptors whose epilogue would make a misaligned vector access, or whose pixels would overlap, are refused before
    any CUDA call, with a message naming the field.  Runs in a process that sees no GPU, so a missing check fails with a
    different (later) message and can never reach a launch; the unchanged descriptor gets past validation."""
    if not os.path.exists(nv.lib_path()):
        pytest.skip("the kernel library is not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]))
    p = subprocess.run([sys.executable, "-c", _REJECT_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    rc, msg = res.pop("baseline")
    print(f"baseline descriptor: status {rc}: {msg}")
    assert rc not in (0, -1), f"the unchanged descriptor should pass validation and fail later without a GPU: {msg}"
    for field, (rc, msg) in res.items():
        print(f"{field.strip()}: status {rc}: {msg}")
        assert rc == -1 and f"svi_conv3d_causal: {field.strip()} must" in msg, f"{field.strip()}: not rejected by name ({msg})"
