"""svi_attn_fwd / svi_attn_fwd_qscale / svi_attn_fwd_sp and svi_attn_small against fp64 references, launch by launch.

Two references, both fp64 and both built from the bf16 values the launch reads:
  * exact: O* = softmax(scale Q K^T) V; with qscale row r of Q is multiplied by rsqrt(S_r / q_dim + eps), S_r the fp32
    partials added in index order; with accumulate O* is added to the prior contents of O;
  * kernel order: what attn_wgmma.cu does, in exact arithmetic except where the kernel rounds on purpose.  Units are
    (head, 128-row Q tile); the plan is (n_full, split) = nv.attention_plan(units, ceil(Lk/128), nv.sm_count(), bytes),
    bytes = 0 with accumulate or without a workspace; units >= n_full are cut into `split` slices, slice s covering
    iterations [n s/split, n (s+1)/split) of the K/V stream, which visits tile (j + kv_first_tile) mod n (kv_first_tile is
    0 except for SP, where it is ceil(self_chunk chunk_rows / 128), wrapped to 0 at n).  Each row keeps a running max
    m_t over the tiles its slice has visited, in the log2 domain x = s scale log2(e) r_q; P_j = 2^(x_j - m_t) is rounded
    fp32 -> bf16 (round to nearest even) for the PV product while the row sum takes the unrounded P; slices merge by
    log-sum-exp.  The rescales commute, so
        O_model = sum_j bf16(P_j) 2^(m_t(j) - m) v_j / sum_j 2^(x_j - m),
    with m the row's final max: tile maxima, then a cummax along each slice's visit order.  scale log2(e) is the fp32
    product the host computes, in both references.

Bars, applied to every launch:
  A. |O - O*| <= eps_r (P|V|)[r, :] / l_r + half a bf16 ulp of the output + 2 fp32 ulps of |O*| (accumulate: the fp32 sum
     with the prior), where (P|V|)/l = sum_j softmax_j |v_j| and, with u = 2^-24,
       eps_r = 2^-8                                 bf16 P: relative error <= 2^-8 per weight (8 significant bits);
             + 2 ln2 (256 u c_r |q_r| max|k| + 8 u max|x|)
                                                    S by fp32 wgmma over 128 exact bf16 products: |dS| <= 2 * 128 u
                                                    sum|q||k| <= 256 u |q||k|max (Cauchy-Schwarz), times c_r = scale
                                                    log2(e) r_q, plus the fp32 scaling / FMA of x; an error dx moves a
                                                    weight by ln2 dx relative, and the normalisation doubles it;
             + 2 (n_kv + split + 1) 2^-21           ex2.approx of every P, of every alpha rescale (at most one per tile
                                                    of a slice: each rise of the running max) and of the merge weights;
             + (3 Lk + split + 8) u                 fp32 accumulation of O over Lk terms (2 Lk u) and of the row sum
                                                    (Lk u), the merge of `split` slices and the final scaling.
     It is a worst-case bound, so it holds for every plan; the worst err/bound per case family is printed.
  B. every element within one bf16 ulp of bf16(O_model) (accumulate: bf16(O_model + prior), one rounding), plus a floor of
     (16 + 8 max|x|) fp32 ulps of (P|V|)/l and a tie term for the P values whose fp32 value lies within the score-error
     window eta_r = 2^-21 + 16 ln2 u (c_r max_j sum|q||k_j| + max|x|) of a bf16 rounding midpoint (the kernel may round
     each of those either way: the term is the sum of their one-ulp steps, or 3 times its root-sum-square where that is
     smaller, i.e. three standard deviations of many steps of independent signs), and at most MAX_FLIP of the elements
     one ulp away.  The max|x| term is the fp32 error
     of the log2-domain scores themselves (a few ulps of |x| from x = s c, the FMA against m and the alpha rescale): it
     moves whole tiles relative to each other, which shows where the output cancels to near zero (one element at Lk = 129
     with a dominant last key needed 35 ulps of (P|V|)/l).  Each launch prints the floor's median size in bf16 ulps of
     |O|, the share of elements where it exceeds one ulp of their own |O| (outputs near zero) and its largest size in
     ulps of the row's rms |O|.
  C. O sits in a wider and taller NaN-filled buffer: nothing but the described [Lq, H*128] region of O's allocation may
     change, Q/K/V (and their NaN padding) stay as they were, and of the workspace only the first slices * 66560 bytes the
     plan uses may change (a NaN guard follows workspace_bytes).
  D. identities: a repeated launch is bit-identical; attention_sp with self_chunk = 0 equals attention() with the same
     workspace; attention_qscale on [L, 1, P] partials equals the same call on [L, 1] holding their fp32 sum.
Negative controls, each of which must fail the bar named (bar B controls by a flip share of at least CONTROL_MARGIN times
MAX_FLIP, or elements beyond one ulp):
  A: O* without the last key (where that key carries weight: Lk <= 512 or a dominant last key); the online softmax
     without the alpha rescale (gpu_check.attn_ref_no_rescale, Lk > 128); qscale from the first partial only;
     accumulate without the prior;
  B: the model under another plan (unsliced where the launch sliced, split - 1, split + 1; not on the ramps, whose row
     max rises in every tile so that every plan rounds alike); for SP the visit order from tile 0; P truncated instead of
     rounded; the row sum over bf16(P) (where the prior cancels most of an accumulated output, so that the row sum's
     rounding shows; elsewhere it moves 1-4 % of the elements by one ulp and is only reported); accumulate with the prior
     added after rounding.  Diffuse scores fail the plan and order controls by flips (35-46 %), peaked ones by elements
     beyond one ulp.
svi_attn_small is fp32 throughout: every element within one bf16 ulp of bf16 of the fp64 softmax (a floor of
(16 + 4 max|s - m|) fp32 ulps of (P|V|)/l for __expf), at most SMALL_MAX_FLIP one-ulp flips.

The explicit cases come first; test_engine_launches then records every attention launch of eager tiny T2V, I2V and Talk
DiT forwards and applies bars A-C to each.  test_attn_rejects_misaligned_pointers runs the host validation in a process
that sees no GPU.  The model's self-tests (test_model_*) run on the CPU.  This module imports without a GPU.
"""
import json
import math
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

from diffsynth import _native as nv
from test_kernel_conformance_gpu import ULP32, _bf16_inside, _bf16_ulp
from tools import gpu_check

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = "cuda"
T = 128                                   # rows of a Q tile and of a K/V tile
SLICE_BYTES = 128 * 128 * 4 + 128 * 8     # one sliced unit: partial O + (row max, row sum)
LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
# one-ulp flips against bf16(O_model), measured on an H100 80GB HBM3 at a 700 W power limit: at most 1.3 % in the explicit
# cases (diffuse scores at Lk 4100-8200), 1.9 % / 2.6 % at L = 32760 with 12 / 40 heads, 0.4 % over the engine launches;
# peaked scores 0.02-0.12 %.  The flips come from the fp32 accumulation noise of long diffuse rows, whose outputs are small
# (|O| ~ (P|V|)/l / sqrt(Lk)).
MAX_FLIP = 0.05
SMALL_MAX_FLIP = 0.002    # svi_attn_small, same card: at most 0.06 % (wav2vec2 length)
CONTROL_MARGIN = 5.0
ROW_ELEMS = 1 << 22                       # rows x keys of one fp64 reference block (a few hundred MB of temporaries)
_BITS = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32}


def _cdiv(a, b):
    return (a + b - 1) // b


# ----------------------------------------------------------------------------------------------------- the two models
def visit_segments(n_kv, split=1, first_tile=0):
    """K/V tiles each slice visits, in order: slice s runs iterations [n s/split, n (s+1)/split), tile (j + first) mod n"""
    return [[(j + first_tile) % n_kv for j in range(n_kv * s // split, n_kv * (s + 1) // split)] for s in range(split)]


def sp_first_tile(Lk, chunk_rows, self_chunk):
    """the first tile fully inside the local chunk (svi_attn_fwd_sp), 0 when that is past the last tile"""
    f = _cdiv(self_chunk * chunk_rows, T)
    return 0 if f >= _cdiv(Lk, T) else f


def scale_log2(scale):
    """scale * log2(e) as the host computes it (fp32 product)"""
    return float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))


def to_bf16(x, mode="rne"):
    """fp64 -> fp32 -> bf16, as a kernel holding the value in fp32 stores it; "trunc" drops the low 16 bits instead"""
    f = x.float()
    if mode == "trunc":
        f = (f.view(torch.int32) & -65536).view(torch.float32)
    return f.to(torch.bfloat16)


def scores(q, k, cs, tile=T):
    """x = (q k^T) c_r in fp64, padded with -inf to whole K/V tiles of `tile` keys: [R, n_kv, tile].  q [G, Lq, d] and
    k [G, Lk, d] give the rows of G independent groups one after the other (R = G Lq); cs is [R] or a number."""
    x = q.double() @ k.double().transpose(-1, -2)
    x = x.reshape(-1, k.shape[-2])
    x = x * (cs[:, None] if torch.is_tensor(cs) else cs)
    Lk = k.shape[-2]
    n = _cdiv(Lk, tile)
    return F.pad(x, (0, n * tile - Lk), value=-math.inf).view(x.shape[0], n, tile)


def _rows_at(w, v):
    """w [R, Lk] times v: [Lk, d] shared by every row, or [G, Lk, d] for G groups of R / G rows each"""
    if v.dim() == 2:
        return w @ v
    return (w.view(v.shape[0], -1, w.shape[1]) @ v).reshape(w.shape[0], v.shape[2])


def exact_softmax(xt, v):
    """(O*, (P|V|)/l) of the rows of xt; the chunk width is xt's last dimension and does not enter the result"""
    R, Lk = xt.shape[0], v.shape[-2]
    x = xt.reshape(R, -1)[:, :Lk]
    e = torch.exp2(x - x.amax(1, keepdim=True))
    l = e.sum(1, keepdim=True)
    v = v.double()
    return _rows_at(e, v) / l, _rows_at(e, v.abs()) / l


def running_max(xt, segments):
    """m_t: the row max over the tiles visited so far, restarting at each slice: [R, n_kv] indexed by tile"""
    tmax = xt.amax(2)
    M = torch.empty_like(tmax)
    for seg in segments:
        idx = torch.tensor(seg, device=xt.device)
        M[:, idx] = torch.cummax(tmax[:, idx], 1).values
    return M


def kernel_order(xt, v, segments, p_round="rne", rowsum="exact", eta=None):
    """O_model of the rows of xt, visiting K/V tiles of xt.shape[2] keys (p_round None: no rounding of P; "trunc":
    truncated), and with eta [R] the tie term of bar B's floor: over the P within eta_r P of a bf16 rounding midpoint,
    t_j = (bf16 step of P_j) 2^(m_t - m) |v_j| / l, combined as min(sum t_j, 3 sqrt(sum t_j^2)): the worst case while few
    such P are involved, three standard deviations of a sum with independent signs when many are.  v is [Lk, d] or
    [G, Lk, d] (see _rows_at).  A row whose keys so far are all masked (x = -inf, running max -inf) takes its P and
    alpha against 0, as svi_quality_attn does: they are exactly 0, so such tiles contribute nothing."""
    R, Lk = xt.shape[0], v.shape[-2]
    v = v.double()
    M = running_max(xt, segments)
    sc = torch.exp2(M - M.amax(1, keepdim=True))[:, :, None]
    P = torch.exp2(xt - M.masked_fill(M == -math.inf, 0.0)[:, :, None])
    Pr = P if p_round is None else to_bf16(P, p_round).double()
    w = (Pr * sc).reshape(R, -1)[:, :Lk]
    l = (w if rowsum == "bf16" else (P * sc).reshape(R, -1)[:, :Lk]).sum(1, keepdim=True)
    o = _rows_at(w, v) / l
    if eta is None:
        return o, None
    b = P.float().view(torch.int32) & -65536
    lo, hi = b.view(torch.float32).double(), (b + 65536).view(torch.float32).double()
    near = (P - (lo + hi) / 2).abs() <= eta.view(R, 1, 1) * P
    amb = torch.where(near, (hi - lo) * sc, torch.zeros((), dtype=P.dtype, device=P.device)).reshape(R, -1)[:, :Lk]
    va = v.abs()
    return o, torch.minimum(_rows_at(amb, va), 3 * _rows_at(amb * amb, va * va).sqrt()) / l


# ------------------------------------------------------------------------------------------------------------- bars
def bar_a(got, ref, pv, eps, extra=0.0):
    """(elements outside, worst err/bound) of bar A; `extra` is an absolute term added to the bound"""
    half = 0.5 * torch.maximum(_bf16_ulp(got.float()), _bf16_ulp(ref.float())).double()
    bound = eps * pv + half + 2 * ULP32 * ref.abs() + extra
    err = (got.double() - ref).abs()
    inside = err <= bound
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    return int((~inside).sum()), (ratio.max().item() if inside.all() else math.inf)


def bar_b(got, ref_bf16, floor):
    """(elements beyond one bf16 ulp + floor, one-ulp flips) of bar B"""
    inside, _ = _bf16_inside(got, ref_bf16, floor.float())
    return int((~inside).sum()), int((got.float() != ref_bf16.float()).sum())


class Tally:
    """n outside / n flips / n elements / worst ratio of one bar or control over the blocks of a launch"""

    def __init__(self):
        self.out = self.flip = self.n = 0
        self.worst = 0.0

    def add(self, n, out=0, flip=0, worst=0.0):
        self.n += n
        self.out += out
        self.flip += flip
        self.worst = max(self.worst, worst)

    @property
    def share(self):
        return self.flip / max(self.n, 1)

    def fails_b(self):
        return self.out > 0 or self.share >= CONTROL_MARGIN * MAX_FLIP


def _store(t):
    """the whole allocation behind t, as a flat tensor of t's dtype"""
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage())


def _bits(t):
    return t.view(_BITS[t.dtype])


def _written(t, rows, cols):
    """flat element indices of t[:rows, :cols] inside its allocation"""
    r = torch.arange(rows, device=t.device)[:, None] * t.stride(0)
    return (t.storage_offset() + r + torch.arange(cols, device=t.device)[None, :]).reshape(-1)


# ---------------------------------------------------------------------------------------------------------- one launch
class Launch:
    """Snapshots one attention launch's arguments and the memory around them; check() applies bars A-C after it."""

    def __init__(self, q, k, v, out, H, scale=None, accumulate=False, workspace=None, q_sumsq=None, q_dim=None,
                 q_eps=None, sp=None):
        torch.cuda.synchronize()
        self.Lq, self.Lk, self.H, self.W = q.shape[0], k.shape[0], H, H * T
        self.scale = 128 ** -0.5 if scale is None else scale
        self.q, self.k, self.v = q.clone(), k.clone(), v.clone()
        self.out, self.accumulate = out, bool(accumulate)
        self.prior = out.clone() if accumulate else None
        ws_bytes = 0 if workspace is None else workspace.numel() * workspace.element_size()
        self.n_qt, self.n_kv = _cdiv(self.Lq, T), _cdiv(self.Lk, T)
        self.units = H * self.n_qt
        self.plan = nv.attention_plan(self.units, self.n_kv, nv.sm_count(), 0 if self.accumulate else ws_bytes)
        self.first = 0 if sp is None else sp_first_tile(self.Lk, sp["chunk_rows"], sp["self_chunk"])
        self.sp = sp
        sl2 = scale_log2(self.scale)
        self.parts = 0
        self.cs = torch.full((self.Lq,), sl2, dtype=torch.float64, device=q.device)
        self.cs_first = None
        if q_sumsq is not None:
            ss = q_sumsq[:, 0] if q_sumsq.dim() == 2 else q_sumsq[:, 0, 0]
            s = ss.clone()
            if q_sumsq.dim() == 3:
                self.parts = q_sumsq.shape[2]
                for j in range(1, self.parts):            # fp32, index order, as the kernel adds them
                    s = s + q_sumsq[:, 0, j]
            self.cs = sl2 * (s.double() / q_dim + q_eps).rsqrt()
            if self.parts > 1:
                self.cs_first = sl2 * (ss.double() / q_dim + q_eps).rsqrt()
        # bar C: every allocation the launch can see, and what of it may change
        self.stores, self.may_write = {}, {}
        named = [("out", out), ("q", q), ("k", k), ("v", v), ("workspace", workspace), ("q_sumsq", q_sumsq),
                 ("kv_flags", None if sp is None else sp["flags"])]
        for name, t in named:
            if t is None:
                continue
            key = t.untyped_storage().data_ptr()
            if key not in self.stores:
                st = _store(t)
                self.stores[key] = (name, st, st.clone())
        self.may_write[out.untyped_storage().data_ptr()] = _written(out, self.Lq, self.W)
        n_full, split = self.plan
        self.ws_used = (self.units - n_full) * split * SLICE_BYTES if split > 1 else 0
        if workspace is not None and self.ws_used:
            off = workspace.storage_offset()
            self.may_write[workspace.untyped_storage().data_ptr()] = torch.arange(
                off, off + self.ws_used // workspace.element_size(), device=q.device)

    # ------------------------------------------------------------------------------------------------------------
    def blocks(self, units=None):
        """(head, r0, r1, sliced) row blocks covering the checked units; units: [(head, q tile)] or None for all"""
        n_full = self.plan[0]
        per_head = max(1, ROW_ELEMS // (T * max(self.Lk, 1)))
        for h in range(self.H):
            tiles = range(self.n_qt) if units is None else sorted({t for hh, t in units if hh == h})
            run, run_sliced = [], False
            for t in tiles:
                sliced = h * self.n_qt + t >= n_full
                if run and (sliced != run_sliced or t != run[-1] + 1 or len(run) >= per_head):
                    yield h, run[0] * T, min((run[-1] + 1) * T, self.Lq), run_sliced
                    run = []
                if not run:
                    run_sliced = sliced
                run.append(t)
            if run:
                yield h, run[0] * T, min((run[-1] + 1) * T, self.Lq), run_sliced

    def check_memory(self, name):
        torch.cuda.synchronize()
        for key, (what, st, before) in self.stores.items():
            same = _bits(st) == _bits(before)
            idx = self.may_write.get(key)
            if idx is not None:
                same[idx] = True
            assert bool(same.all()), f"{name}: the launch changed {int((~same).sum())} elements of the {what} " \
                                     f"allocation outside what it may write"

    def check(self, name, controls=True, bite=(), units=None, quiet=False, unrequire=()):
        """bars A-C (and the negative controls) of this launch; returns what was measured"""
        self.check_memory(name)
        n_full, split = self.plan
        A, B = Tally(), Tally()
        ctl, worst_b = {}, []
        # size of bar B's floor in bf16 ulps: largest block median of floor / ulp(|O|), elements where that exceeds 1, and the
        # largest floor / ulp(rms |O| of the row), i.e. against a typical output of its row
        floor_med, floor_over, floor_typ = 0.0, 0, 0.0

        def tally(cname):
            return ctl.setdefault(cname, Tally())

        for h, r0, r1, sliced in self.blocks(units):
            cols = slice(h * T, (h + 1) * T)
            qh, kh, vh = self.q[r0:r1, cols], self.k[:, cols], self.v[:, cols].double()
            cs = self.cs[r0:r1]
            xt = scores(qh, kh, cs)
            sp_ = split if sliced else 1
            segs = visit_segments(self.n_kv, sp_, self.first)
            o_star, pv = exact_softmax(xt, vh)
            qn, kmax = qh.double().norm(dim=1), kh.double().norm(dim=1).max()
            qk1 = (qh.double().abs() @ kh.double().abs().t()).amax(1)           # max_j sum_d |q_d||k_jd|
            xabs = xt.reshape(xt.shape[0], -1)[:, :self.Lk].abs().amax(1)
            eps = (2.0 ** -8 + 2 * LN2 * (256 * ULP32 * cs * qn * kmax + 8 * ULP32 * xabs)
                   + 2 * (self.n_kv + sp_ + 1) * 2.0 ** -21 + (3 * self.Lk + sp_ + 8) * ULP32)[:, None]
            eta = 2.0 ** -21 + 16 * LN2 * ULP32 * (cs * qk1 + xabs)
            o_mod, amb = kernel_order(xt, vh, segs, eta=eta)
            got = self.out[r0:r1, cols]
            prior = self.prior[r0:r1, cols].double() if self.accumulate else 0.0
            n_el = got.numel()
            out, worst = bar_a(got, o_star + prior, pv, eps)
            A.add(n_el, out=out, worst=worst)
            floor = (16 + 8 * xabs[:, None]) * ULP32 * pv + amb
            ref_b = to_bf16(o_mod + prior)
            out, flip = bar_b(got, ref_b, floor)
            B.add(n_el, out=out, flip=flip)
            f_ulps = floor / _bf16_ulp(ref_b.float()).double().clamp_min(1e-300)     # the floor in bf16 ulps of |O|
            floor_med = max(floor_med, f_ulps.median().item())
            rms = (o_mod + prior).pow(2).mean(1, keepdim=True).sqrt()
            floor_typ = max(floor_typ, (floor / _bf16_ulp(rms.float()).double().clamp_min(1e-300)).max().item())
            floor_over += int((f_ulps > 1).sum())
            if out:                                            # where the worst element beyond bar B sits
                err = (got.double() - ref_b.double()).abs()
                ulp = torch.maximum(_bf16_ulp(got.float()), _bf16_ulp(ref_b.float())).double()
                excess = (err - ulp - floor) / (ULP32 * pv).clamp_min(1e-300)
                i = int(excess.argmax())
                r_, c_ = divmod(i, excess.shape[1])
                worst_b.append((excess.max().item(), f"row {r0 + r_} col {h * T + c_}: got {got[r_, c_].item():.6g} "
                                f"model {o_mod[r_, c_].item() + (prior[r_, c_].item() if self.accumulate else 0):.6g} "
                                f"|O|/pv {abs(o_mod[r_, c_].item()) / pv[r_, c_].item():.3g} excess "
                                f"{excess.max().item():.4g} fp32 ulps of pv, floor {floor[r_, c_].item() / (ULP32 * pv[r_, c_].item()):.4g}"))
            if not controls:
                continue

            def ctl_a(cname, ref):
                tally(cname).add(n_el, out=bar_a(got, ref, pv, eps)[0])

            def ctl_b(cname, o, pre_rounded=False):
                ref = to_bf16(to_bf16(o).double() + prior) if pre_rounded else to_bf16(o + prior)
                out_, flip_ = bar_b(got, ref, floor)
                tally(cname).add(n_el, out=out_, flip=flip_)

            if self.Lk >= 2:
                x = xt.reshape(xt.shape[0], -1)[:, :self.Lk - 1]
                e = torch.exp2(x - x.amax(1, keepdim=True))
                ctl_a("A: last key dropped", (e @ vh[:-1]) / e.sum(1, keepdim=True) + prior)
            if self.n_kv >= 2:
                qs = (qh.float() * (cs / scale_log2(self.scale)).float()[:, None]).contiguous()
                wrong = gpu_check.attn_ref_no_rescale(qs, kh.contiguous(), vh.float().contiguous(), 1, self.scale,
                                                      first_tile=self.first)
                ctl_a("A: no alpha rescale", wrong.double() + prior)
            if self.cs_first is not None:
                ctl_a("A: qscale from the first partial", exact_softmax(
                    scores(qh, kh, self.cs_first[r0:r1]), vh)[0] + prior)
            if self.accumulate:
                ctl_a("A: accumulate without the prior", o_star)
            if sliced and split > 1:
                ctl_b("B: plan unsliced", kernel_order(xt, vh, visit_segments(self.n_kv, 1, self.first))[0])
                if split - 1 >= 2:
                    ctl_b("B: plan split - 1", kernel_order(xt, vh, visit_segments(self.n_kv, split - 1, self.first))[0])
                if split + 1 <= 8 and self.n_kv >= split + 1:
                    ctl_b("B: plan split + 1", kernel_order(xt, vh, visit_segments(self.n_kv, split + 1, self.first))[0])
            if self.first:
                ctl_b("B: SP order from tile 0", kernel_order(xt, vh, visit_segments(self.n_kv, sp_, 0))[0])
            if self.Lk >= 2:
                ctl_b("B: P truncated", kernel_order(xt, vh, segs, p_round="trunc")[0])
                ctl_b("B: row sum of bf16(P)", kernel_order(xt, vh, segs, rowsum="bf16")[0])
            if self.accumulate:
                ctl_b("B: prior added after rounding", o_mod, pre_rounded=True)

        r = dict(name=name, plan=(n_full, split), first_tile=self.first, worst=A.worst, flips=B.share,
                 floor_median_ulps=floor_med, floor_over_one_ulp=floor_over / max(B.n, 1), floor_max_typical_ulps=floor_typ,
                 controls={k: dict(out=t.out, share=t.share, worst=t.worst) for k, t in ctl.items()})
        if not quiet:
            print(f"[{'OK ' if A.out == 0 and B.out == 0 and B.share <= MAX_FLIP else 'BAD'}] attn {name}: "
                  f"plan (n_full, split)={self.plan} first_tile={self.first} A worst err/bound={A.worst:.3f} "
                  f"B one-ulp flips={100 * B.share:.3f} % beyond={B.out} floor: median {floor_med:.3f} bf16 ulps of |O|, "
                  f"above one ulp for {100 * floor_over / max(B.n, 1):.3f} %, at most {floor_typ:.3f} ulps of the row's "
                  f"rms |O|", flush=True)
            for k, t in ctl.items():
                print(f"      control {k}: {'A outside' if k.startswith('A') else 'B beyond'}={t.out} "
                      f"flips={100 * t.share:.2f} % of {t.n}", flush=True)
        if worst_b:
            print(f"      worst element beyond bar B: {max(worst_b)[1]}", flush=True)
        assert A.out == 0, f"{name}: {A.out} elements outside the fp64 bound of bar A"
        assert B.out == 0, f"{name}: {B.out} elements beyond one bf16 ulp of the kernel-order model"
        assert B.share <= MAX_FLIP, f"{name}: {100 * B.share:.3f} % one-ulp flips, more than {100 * MAX_FLIP} %"
        required = {"A: no alpha rescale", "A: qscale from the first partial", "A: accumulate without the prior",
                    "B: plan unsliced", "B: plan split - 1", "B: plan split + 1", "B: SP order from tile 0",
                    "B: P truncated", "B: prior added after rounding"} - set(unrequire) | set(bite)
        for k, t in ctl.items():
            if k in required:
                caught = t.out > 0 if k.startswith("A") else t.fails_b()
                assert caught, f"{name}: negative control '{k}' passes its bar (flips {100 * t.share:.2f} %)"
        return r


# ------------------------------------------------------------------------------------------------------------- inputs
def _nans(*shape, dtype=torch.bfloat16):
    return torch.full(shape, float("nan"), device=dev, dtype=dtype)


def _workspace(nbytes):
    """nbytes of workspace followed, in the same allocation, by a NaN guard"""
    return _nans(nbytes // 4 + 64, dtype=torch.float32)[:nbytes // 4]


def _out(Lq, W, row0=0):
    buf = _nans(row0 + Lq + 40, W + 16)
    return buf[row0:row0 + Lq, :W]


def _layout(q, k, v, layout):
    """q, k, v as views of the buffers the layout names, everything around them NaN"""
    Lq, W = q.shape
    Lk = k.shape[0]
    if layout == "fused":                  # the DiT's q|k|v GEMM output, ld = 3d (self-attention: Lq = Lk)
        qkv = _nans(Lq + 7, 3 * W)
        qkv[:Lq, :W], qkv[:Lk, W:2 * W], qkv[:Lk, 2 * W:] = q, k, v
        return qkv[:Lq, :W], qkv[:Lk, W:2 * W], qkv[:Lk, 2 * W:], 0
    if layout == "context":                # cross-attention: q from the [L, 3d] buffer, K|V of the context [Lk, 2d]
        qb, kv = _nans(Lq + 5, 3 * W), _nans(Lk + 9, 2 * W)
        qb[:Lq, :W], kv[:Lk, :W], kv[:Lk, W:] = q, k, v
        return qb[:Lq, :W], kv[:Lk, :W], kv[:Lk, W:], 0
    if layout == "padded":                 # NaN padding columns and NaN rows past Lq / Lk
        bufs = []
        for t in (q, k, v):
            b = _nans(t.shape[0] + 11, W + 24)
            b[:t.shape[0], :W] = t
            bufs.append(b[:t.shape[0], :W])
        return (*bufs, 0)
    if layout == "row slice":              # the audio branch: Q and O are row slices aq[lo:hi], att[lo:hi]
        qb = _nans(Lq + 333, W + 8)
        qb[200:200 + Lq, :W] = q
        return qb[200:200 + Lq, :W], k, v, 200
    assert layout == "plain"
    return q, k, v, 0


def _inputs(g, Lq, Lk, H, amp, stress=None):
    if stress is not None:
        return gpu_check.attn_online_inputs(g, Lq, Lk, H, amp, **stress)
    q = (torch.randn(Lq, H * T, generator=g) * amp).to(dev, torch.bfloat16)
    k = (torch.randn(Lk, H * T, generator=g) * amp).to(dev, torch.bfloat16)
    v = torch.randn(Lk, H * T, generator=g).to(dev, torch.bfloat16)
    return q, k, v


# ---------------------------------------------------------------------------------------------------- explicit cases
def _budgets(Lq, Lk, H, which):
    """workspace sizes in bytes: "full" (svi_attn_workspace_bytes), k (k slices), "smaller" (one slice per sliced unit
    fewer than the full plan uses, which forces a smaller split), None (no workspace)"""
    out = []
    units, n_kv = H * _cdiv(Lq, T), _cdiv(Lk, T)
    for b in which:
        if b == "full":
            out.append(nv.attention_workspace_bytes(Lq, Lk, H))
        elif b == "smaller":
            n_full, split = nv.attention_plan(units, n_kv, nv.sm_count(), nv.attention_workspace_bytes(Lq, Lk, H))
            assert split > 1, "the 'smaller' budget needs a plan that slices"
            out.append((units - n_full) * (split - 1) * SLICE_BYTES)
        else:
            out.append(b if b is None else b * SLICE_BYTES)
    return out


def _plan_cases():
    """(Lq, Lk, H) of the plan cases, from the SM count: fewer units than a wave, an exact multiple of the SM count,
    partial last waves, n_full = 0"""
    sms = nv.sm_count()
    return {
        "fewer units than one wave": (1000, 4100, 2),
        "units = 2 x SM count": (sms * T - 5, 512, 2),
        "3200 x 12 heads, Lk 4100": (3200, 4100, 12),
        "3000 x 13 heads, Lk 4100": (3000, 4100, 13),
        "SM count + 10 units, Lk 8200": ((sms + 10) * T - 37, 8200, 1),
        "n_full = 0: 34 units": (17 * T - 3, 4100, 2),
    }


PLAN_BUDGETS = ("full", None)
# the row max rises in every tile of a ramp, so every slice's running max is the unsliced one: plans round alike there
PLAN_CONTROLS = ("B: plan unsliced", "B: plan split - 1", "B: plan split + 1")
CASES = {
    # plans (shapes from _plan_cases)
    **{f"plan: {n}": dict(plan=n, amp=1.0, budgets=PLAN_BUDGETS) for n in
       ("fewer units than one wave", "units = 2 x SM count", "3000 x 13 heads, Lk 4100", "SM count + 10 units, Lk 8200",
        "n_full = 0: 34 units")},
    "plan: 3200 x 12 heads, Lk 4100, budgets": dict(plan="3200 x 12 heads, Lk 4100", amp=1.0,
                                                    budgets=("full", 1, "smaller", 100, None)),
    "plan: 3200 x 12 heads, Lk 4100, peaked": dict(plan="3200 x 12 heads, Lk 4100", amp=3.0, budgets=("full",)),
    # lengths and heads
    # one query row: 256 outputs are too few for a rounding-mode control to show in the flip share
    "Lq=1 Lk=4100 H=2 ramp": dict(Lq=1, Lk=4100, H=2, amp=3.5, stress=dict(ramp=120.0),
                                  unrequire=PLAN_CONTROLS + ("B: P truncated",)),
    "Lq=127 Lk=1 H=1": dict(Lq=127, Lk=1, H=1, amp=1.0),
    "Lq=129 Lk=77 H=40 peaked context": dict(Lq=129, Lk=77, H=40, amp=3.0, layout="context",
                                             bite=("A: last key dropped",)),
    "Lq=1000 Lk=128 H=2": dict(Lq=1000, Lk=128, H=2, amp=1.0, bite=("A: last key dropped",)),
    "Lq=129 Lk=129 H=12 fused": dict(Lq=129, Lk=129, H=12, amp=1.0, layout="fused", bite=("A: last key dropped",)),
    "Lq=127 Lk=257 H=2 padded": dict(Lq=127, Lk=257, H=2, amp=1.0, layout="padded", bite=("A: last key dropped",)),
    "Lq=1000 Lk=512 H=1 row slice": dict(Lq=1000, Lk=512, H=1, amp=1.0, layout="row slice",
                                         bite=("A: last key dropped",)),
    "Lq=3200 Lk=3200 H=2 fused peaked": dict(Lq=3200, Lk=3200, H=2, amp=3.0, layout="fused"),
    # the online-softmax stresses of gpu_check.sec_attn_online
    "ramp sliced": dict(Lq=3200, Lk=4100, H=12, amp=3.5, stress=dict(ramp=120.0), unrequire=PLAN_CONTROLS),
    "dominant key in the last tile": dict(Lq=700, Lk=1000, H=2, amp=3.2, stress=dict(dominant=999),
                                          bite=("A: last key dropped",)),
    "dominant key in a middle slice": dict(Lq=3200, Lk=4100, H=12, amp=3.2, stress=dict(dominant=2053)),
    "Lk=129 dominant last": dict(Lq=300, Lk=129, H=3, amp=3.5, stress=dict(ramp=50.0, dominant=128),
                                 bite=("A: last key dropped",)),
}


def _shape(case):
    if "plan" in case:
        return _plan_cases()[case["plan"]]
    return case["Lq"], case["Lk"], case["H"]


@pytest.mark.gpu
def test_plans_are_distinct():
    """the plan cases produce the plans they are named for, and different ones.  Only what holds for any SM count of an
    H100 is asserted; on 132 SMs (H100 SXM) the cases give (0, 4), (264, 1), (264, 3), (264, 2), (132, 8) and (0, 3), and
    the budgets of the 3200 x 12-head case give (264, 3) full, (264, 2) for "smaller" and 100 slices, (300, 1) for one
    slice and none."""
    sms = nv.sm_count()
    seen = {}
    for name, (Lq, Lk, H) in _plan_cases().items():
        units, n_kv = H * _cdiv(Lq, T), _cdiv(Lk, T)
        seen[name] = nv.attention_plan(units, n_kv, sms, nv.attention_workspace_bytes(Lq, Lk, H))
        print(f"plan {name}: {units} units, {n_kv} K/V tiles on {sms} SMs -> (n_full, split) = {seen[name]}")
    assert seen["fewer units than one wave"][0] == 0 and seen["fewer units than one wave"][1] > 1
    assert seen["units = 2 x SM count"][1] == 1
    assert seen["n_full = 0: 34 units"][0] == 0 and seen["n_full = 0: 34 units"][1] > 1
    assert all(seen[n][1] > 1 and seen[n][0] > 0 for n in ("3200 x 12 heads, Lk 4100", "3000 x 13 heads, Lk 4100",
                                                           "SM count + 10 units, Lk 8200"))
    assert len(set(seen.values())) == len(seen), f"plan cases collapse onto the same plan: {seen}"
    splits = {s for _, s in seen.values()}
    assert 1 in splits and len(splits - {1}) >= 3 and max(splits) >= 4, splits
    Lq, Lk, H = _plan_cases()["3200 x 12 heads, Lk 4100"]
    units, n_kv = H * _cdiv(Lq, T), _cdiv(Lk, T)
    by_budget = {b: nv.attention_plan(units, n_kv, sms, n if n is not None else 0)
                 for b, n in zip(("full", 1, "smaller", 100, None), _budgets(Lq, Lk, H, ("full", 1, "smaller", 100, None)))}
    print(f"budgets of 3200 x 12 heads: {by_budget}")
    assert by_budget[1] == by_budget[None] == (units, 1)
    assert by_budget["smaller"][1] < by_budget["full"][1] and by_budget["full"][1] > 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_attention_case(name):
    """one explicit geometry under each of its workspace budgets: bars A-C with the negative controls, and a repeated
    launch bit-identical"""
    case = CASES[name]
    Lq, Lk, H = _shape(case)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    q0, k0, v0 = _inputs(g, Lq, Lk, H, case["amp"], case.get("stress"))
    q, k, v, row0 = _layout(q0, k0, v0, case.get("layout", "plain"))
    for nbytes in _budgets(Lq, Lk, H, case.get("budgets", ("full",))):
        ws = None if nbytes is None else _workspace(nbytes)
        out = _out(Lq, H * T, row0)
        L = Launch(q, k, v, out, H, workspace=ws)
        nv.attention(q, k, v, out, H, workspace=ws)
        L.check(f"{name} workspace={nbytes}", bite=case.get("bite", ()), unrequire=case.get("unrequire", ()))
        again = _out(Lq, H * T, row0)
        nv.attention(q, k, v, again, H, workspace=None if nbytes is None else _workspace(nbytes))
        torch.cuda.synchronize()
        assert torch.equal(_bits(again), _bits(out)), f"{name}: a repeated launch is not bit-identical"


@pytest.mark.gpu
def test_accumulate_image_branch():
    """cross-attention of the I2V DiT: Lk = 512 text keys, then Lk = 257 image keys accumulated onto it; the image
    branch's V is the negated first 257 text values, so the prior partly cancels what is added"""
    g = torch.Generator().manual_seed(41)
    Lq, H = 1000, 12
    q, k_t, v_t = _inputs(g, Lq, 512, H, 1.5)
    k_i, v_i = k_t[:257].clone(), (-v_t[:257].float() + 0.3 * torch.randn(257, H * T, generator=g).to(dev)).bfloat16()
    q, k_t, v_t, _ = _layout(q, k_t, v_t, "context")
    _, k_i, v_i, _ = _layout(q[:1].clone(), k_i, v_i, "context")
    out = _out(Lq, H * T)
    ws = _workspace(nv.attention_workspace_bytes(Lq, 512, H))
    L = Launch(q, k_t, v_t, out, H, workspace=ws)
    nv.attention(q, k_t, v_t, out, H, workspace=ws)
    L.check("image branch: text, Lk=512", bite=("A: last key dropped",))
    first = out.clone()
    L = Launch(q, k_i, v_i, out, H, accumulate=True, workspace=ws)
    nv.attention(q, k_i, v_i, out, H, accumulate=True, workspace=ws)
    # the prior cancels much of the output here, so the rounding of the row sum shows
    r = L.check("image branch: image, Lk=257, accumulate", bite=("A: last key dropped", "B: row sum of bf16(P)"))
    assert r["plan"][1] == 1, "an accumulating launch must not slice"
    cancel = (out.float().abs() < first.float().abs()).float().mean().item()
    print(f"      the prior cancels part of the sum in {100 * cancel:.1f} % of the elements")
    assert cancel > 0.05
    again = first.clone()
    nv.attention(q, k_i, v_i, again, H, accumulate=True)
    torch.cuda.synchronize()
    assert torch.equal(_bits(again), _bits(out)), "a repeated accumulating launch is not bit-identical"


@pytest.mark.gpu
@pytest.mark.parametrize("H,groups,parts", [(2, 1, 0), (12, 1, 12), (40, 1, 40), (12, 2, 12)])
def test_qscale_layouts(H, groups, parts):
    """svi_attn_fwd_qscale on row sums [L, 1] and partials [L, 1, P] (P = d/128: 12 at 1.3B, 40 at 14B), and group 0 of
    [L, 2, P] (q_ss_ld > parts); one Q row is zero.  The partials equal, bit for bit, the [L, 1] call on their fp32 sum."""
    g = torch.Generator().manual_seed(50 + H + groups)
    Lq, Lk = 1000, 257
    d = H * T
    q = (torch.randn(Lq, d, generator=g) * 7.0).to(dev, torch.bfloat16)          # un-normalised q
    q[5] = 0
    k = (torch.randn(Lk, d, generator=g) * 2.0).to(dev, torch.bfloat16)
    v = torch.randn(Lk, d, generator=g).to(dev, torch.bfloat16)
    q, k, v, _ = _layout(q, k, v, "context")
    qf = q.float()
    if parts:
        ss = torch.randn(Lq, groups, parts, generator=g).abs().to(dev)         # group 1: unrelated values
        ss[:, 0] = (qf.reshape(Lq, parts, T) ** 2).sum(2)
    else:
        ss = torch.randn(Lq, groups, generator=g).abs().to(dev)
        ss[:, 0] = (qf ** 2).sum(1)
    out = _out(Lq, d)
    ws = _workspace(nv.attention_workspace_bytes(Lq, Lk, H))
    L = Launch(q, k, v, out, H, workspace=ws, q_sumsq=ss, q_dim=d, q_eps=1e-6)
    nv.attention_qscale(q, k, v, out, H, ss, d, 1e-6, workspace=ws)
    L.check(f"qscale H={H} q_sumsq {tuple(ss.shape)}", bite=("A: last key dropped",))
    if parts:
        s = ss[:, 0, 0].clone()
        for j in range(1, parts):
            s = s + ss[:, 0, j]
        summed = _out(Lq, d)
        nv.attention_qscale(q, k, v, summed, H, s[:, None].contiguous(), d, 1e-6, workspace=ws)
        torch.cuda.synchronize()
        assert torch.equal(_bits(summed), _bits(out)), "partials differ from the [L, 1] call on their fp32 sum"


SP_GEOMETRIES = [(1260, 630, 2, 2.0), (1260, 420, 3, 2.0), (4100, 2050, 2, 2.0),
                 (1000, 900, 2, 2.0)]      # the last chunk starts inside the last K/V tile: kv_first_tile wraps to 0


@pytest.mark.gpu
@pytest.mark.parametrize("L,chunk,H,amp", SP_GEOMETRIES)
def test_sp_one_gpu(L, chunk, H, amp):
    """svi_attn_fwd_sp on one GPU, every self_chunk, with and without workspace.  Every flag holds the epoch, set and
    synchronised before the launch, so the producer never waits."""
    g = torch.Generator().manual_seed(60 + L + chunk)
    q, k, v = _inputs(g, L, L, H, amp)
    q, k, v, _ = _layout(q, k, v, "fused")
    epoch = 7
    n_chunks = _cdiv(L, chunk)
    flags = torch.full((n_chunks + 1,), epoch, dtype=torch.int32, device=dev)[:n_chunks]
    torch.cuda.synchronize()
    firsts = []
    for c in range(n_chunks):
        r0, r1 = c * chunk, min(L, (c + 1) * chunk)
        ql = q[r0:r1]
        for nbytes in (None, nv.attention_workspace_bytes(r1 - r0, L, H)):
            ws = None if nbytes is None else _workspace(nbytes)
            out = _out(r1 - r0, H * T, 3)
            sp = dict(flags=flags, chunk_rows=chunk, self_chunk=c)
            Ln = Launch(ql, k, v, out, H, workspace=ws, sp=sp)
            nv.attention_sp(ql, k, v, out, H, flags, epoch, chunk, c, workspace=ws)
            r = Ln.check(f"sp L={L} chunk_rows={chunk} H={H} self_chunk={c} workspace={nbytes}")
            firsts.append(r["first_tile"])
            if c == 0:
                plain = _out(r1 - r0, H * T, 3)
                nv.attention(ql, k, v, plain, H, workspace=None if nbytes is None else _workspace(nbytes))
                torch.cuda.synchronize()
                assert torch.equal(_bits(plain), _bits(out)), "attention_sp with self_chunk 0 differs from attention()"
    if (n_chunks - 1) * chunk > (_cdiv(L, T) - 1) * T:
        assert firsts[-1] == 0, "kv_first_tile must wrap to 0 when the last chunk starts inside the last tile"
    else:
        assert any(f > 0 for f in firsts)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("H", [12, 40])
def test_bench_shape_sampled(H):
    """self-attention at the benchmark length L = 32760 (fused q|k|v, the engine's workspace), checked on every sliced unit,
    the first unit, the ragged last unit and a few random whole units; the fp64 reference runs in row blocks and its
    peak device memory is printed"""
    L = 32760
    g = torch.Generator().manual_seed(70 + H)
    q, k, v = _inputs(g, L, L, H, 1.0)
    q, k, v, _ = _layout(q, k, v, "fused")
    out = _out(L, H * T)
    ws = _workspace(nv.attention_workspace_bytes(L, L, H))
    Ln = Launch(q, k, v, out, H, workspace=ws)
    nv.attention(q, k, v, out, H, workspace=ws)
    n_full, split = Ln.plan
    n_qt = Ln.n_qt
    units = set(range(n_full, Ln.units)) | {0, Ln.units - 1}
    units |= set(torch.randint(0, max(n_full, 1), (6,), generator=g).tolist())
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    Ln.check(f"bench shape L={L} H={H} ({len(units)} units)", units=[(u // n_qt, u % n_qt) for u in sorted(units)],
             bite=())
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    print(f"      fp64 reference peak device memory above the inputs: {peak:.2f} GiB", flush=True)
    # whether the launch slices depends on the SM count: on 132 SMs the 12-head launch slices its last 36 of 3072 units,
    # and the 40-head one (10240 units) runs whole because slicing would save less than 1.5 %
    print(f"      plan (n_full, split) = {(n_full, split)} on {nv.sm_count()} SMs; sliced units checked: "
          f"{Ln.units - n_full if split > 1 else 0}", flush=True)
    assert peak < 4.0


# ---------------------------------------------------------------------------------------------------- svi_attn_small
def small_ref(q, k, v, H, hd, scale, bias_table=None, bucket=None, key_mask=None):
    """fp64 softmax(Q K^T scale + bias) V with masked keys at -inf (every key masked: 0); returns (O, (P|V|)/l, max|s-m|)"""
    Lq, Lk = q.shape[0], k.shape[0]
    qh, kh, vh = (t.double().reshape(t.shape[0], H, hd).transpose(0, 1) for t in (q, k, v))
    s = qh @ kh.transpose(1, 2) * scale
    if bias_table is not None:
        s = s + bias_table.double()[bucket.long()].permute(2, 0, 1)
    if key_mask is not None:
        s = s.masked_fill(key_mask.view(1, 1, Lk) == 0, -math.inf)
    m = s.amax(2, keepdim=True)
    e = torch.exp(s - m).nan_to_num(0.0)
    l = e.sum(2, keepdim=True)
    o = ((e @ vh) / l).nan_to_num(0.0)
    pv = ((e @ vh.abs()) / l).nan_to_num(0.0)
    xabs = torch.where(e > 0, (s - m).abs(), torch.zeros_like(s)).amax(2, keepdim=True).nan_to_num(0.0)
    back = lambda t: t.transpose(0, 1).reshape(Lq, -1)                      # noqa: E731
    return back(o), back(pv), back(xabs.expand(-1, -1, hd))


SMALL = {
    # the umT5 encoder: scale 1, bucketed relative-position bias, a fully masked 32-key tile mid-sequence, a padded tail
    "T5 hd=64 L=512": dict(L=512, H=4, hd=64, scale=1.0, amp=(0.6, 0.6), t5=True),
    "CLIP hd=80 L=257": dict(L=257, H=3, hd=80, scale=80 ** -0.5, amp=(2.0, 2.0)),
    "wav2vec2 hd=64 L=3050": dict(L=3050, H=12, hd=64, scale=0.125, amp=(2.0, 2.0)),
    "hd=16 strided": dict(L=333, H=5, hd=16, scale=0.25, amp=(1.5, 1.5), pad=40),
    "hd=128 strided": dict(L=200, H=2, hd=128, scale=128 ** -0.5, amp=(2.5, 2.5), pad=24),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SMALL))
def test_attention_small_case(name):
    """svi_attn_small within one bf16 ulp of the fp64 softmax, nothing written outside [L, H*hd], and its negative
    controls (T5: buckets transposed, the neighbouring head's bias column, the mask ignored, scale 1/sqrt(hd); the others:
    the online softmax without its rescale over 32-key tiles) beyond it"""
    c = SMALL[name]
    L, H, hd, scale = c["L"], c["H"], c["hd"], c["scale"]
    W, pad = H * hd, c.get("pad", 8)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    bufs = []
    for a in (c["amp"][0], c["amp"][1], 1.0):
        b = _nans(L + 3, W + pad)
        b[:L, :W] = (torch.randn(L, W, generator=g) * a).to(dev, torch.bfloat16)
        bufs.append(b[:L, :W])
    q, k, v = bufs
    kw = {}
    if c.get("t5"):
        from diffsynth.models.wan_video_text_encoder import relative_position_buckets
        kw["bias_table"] = (torch.randn(32, H, generator=g) * 2.0).to(dev)
        kw["bucket"] = relative_position_buckets(L, L).to(dev)
        mask = torch.ones(L, dtype=torch.int32)
        mask[224:256] = 0                     # one whole 32-key tile
        mask[L - 77:] = 0                     # the padded tail
        kw["key_mask"] = mask.to(dev)
    big = _nans(L + 5, W + 8)
    out = big[:L, :W]
    before = [t.clone() for t in (q, k, v)]
    keep = big.clone()
    nv.attention_small(q, k, v, out, H, hd, scale, **kw)
    torch.cuda.synchronize()
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(before, (q, k, v))), "inputs changed"
    mask_w = torch.ones_like(big, dtype=torch.bool)
    mask_w[:L, :W] = False
    assert torch.equal(_bits(big)[mask_w], _bits(keep)[mask_w]), "svi_attn_small wrote outside [L, H*hd]"
    ref, pv, xabs = small_ref(q, k, v, H, hd, scale, **kw)
    floor = (16 + 4 * xabs) * ULP32 * pv

    def bar(r):
        inside, _ = _bf16_inside(out, to_bf16(r), floor.float())
        return int((~inside).sum()), (out.float() != to_bf16(r).float()).float().mean().item()

    beyond, share = bar(ref)
    ctl = {}
    if c.get("t5"):
        ctl["buckets transposed"] = small_ref(q, k, v, H, hd, scale, kw["bias_table"], kw["bucket"].t().contiguous(),
                                              kw["key_mask"])[0]
        ctl["neighbouring head's bias column"] = small_ref(q, k, v, H, hd, scale, kw["bias_table"].roll(1, 1), kw["bucket"],
                                                           kw["key_mask"])[0]
        ctl["mask ignored"] = small_ref(q, k, v, H, hd, scale, kw["bias_table"], kw["bucket"])[0]
        ctl["scale 1/sqrt(hd)"] = small_ref(q, k, v, H, hd, hd ** -0.5, kw["bias_table"], kw["bucket"], kw["key_mask"])[0]
        assert not torch.equal(kw["bucket"], kw["bucket"].t())
    else:
        ctl["no rescale, 32-key tiles"] = gpu_check.attn_ref_no_rescale(q.contiguous(), k.contiguous(), v.contiguous(), H,
                                                                        scale, hd=hd, tile=32).double()
    print(f"[{'OK ' if beyond == 0 and share <= SMALL_MAX_FLIP else 'BAD'}] attn_small {name}: one-ulp flips "
          f"{100 * share:.3f} % beyond={beyond}", flush=True)
    res = {k_: bar(r) for k_, r in ctl.items()}
    for k_, (b, s) in res.items():
        print(f"      control {k_}: beyond={b} flips={100 * s:.2f} %", flush=True)
    assert beyond == 0 and share <= SMALL_MAX_FLIP, f"{name}: beyond one bf16 ulp of fp64 ({beyond}, {100 * share:.3f} %)"
    for k_, (b, s) in res.items():
        assert b > 0 or s >= CONTROL_MARGIN * SMALL_MAX_FLIP, f"{name}: control '{k_}' passes the bar"


# ------------------------------------------------------------------------------------------------ the engine's launches
class Recorder:
    """Stands in for nv.attention / nv.attention_qscale: snapshots, launches the kernel, applies bars A-C to that launch
    with its own arguments and plan, and lets the engine carry on with the kernel's output.  Keeps each geometry."""

    def __init__(self):
        self.attention, self.attention_qscale = nv.attention, nv.attention_qscale
        self.seen, self.worst, self.flips = [], 0.0, 0.0

    def _record(self, L, q, k, name):
        r = L.check(f"engine launch {len(self.seen)} ({name})", controls=False, quiet=True)
        self.worst, self.flips = max(self.worst, r["worst"]), max(self.flips, r["flips"])
        self.seen.append(dict(fn=name, W=L.W, Lq=L.Lq, Lk=L.Lk, ldq=q.stride(0), ldk=k.stride(0), acc=L.accumulate,
                              parts=L.parts, q_row0=q.storage_offset() // q.stride(0), plan=L.plan))

    def attn(self, q, k, v, out, num_heads, scale=None, accumulate=False, workspace=None):
        L = Launch(q, k, v, out, num_heads, scale, accumulate, workspace)
        self.attention(q, k, v, out, num_heads, scale, accumulate, workspace)
        self._record(L, q, k, "attention")
        return out

    def qscale(self, q, k, v, out, num_heads, q_sumsq, q_dim, q_eps, scale=None, accumulate=False, workspace=None):
        L = Launch(q, k, v, out, num_heads, scale, accumulate, workspace, q_sumsq, q_dim, q_eps)
        self.attention_qscale(q, k, v, out, num_heads, q_sumsq, q_dim, q_eps, scale, accumulate, workspace)
        self._record(L, q, k, "attention_qscale")
        return out


@pytest.mark.gpu
def test_engine_launches(monkeypatch):
    """every attention launch of eager forwards of the tiny T2V, I2V and Talk DiTs, at token counts that are not multiples
    of 128, against the fp64 references of its own arguments"""
    from diffsynth.models.wan_video_dit import WanModel
    from diffsynth.pipelines.svi_video_talk import preprocess_audio
    from tools import synth
    rec = Recorder()
    monkeypatch.setattr(nv, "attention", rec.attn)
    monkeypatch.setattr(nv, "attention_qscale", rec.qscale)
    runs = [("t2v", synth.CFG_TINY_T2V, 3, 16, 22, 40), ("i2v", synth.CFG_TINY_I2V, 2, 14, 20, 24),
            ("talk", synth.CFG_TINY_TALK, 3, 10, 18, 24)]
    counts = {}
    for tag, cfg, f, h, w, ctx in runs:
        seed = len(counts) + 3
        sd = {k_: v_.to(torch.bfloat16).float() for k_, v_ in synth.make_dit_state_dict(cfg, seed=seed).items()}
        m = WanModel(**cfg).eval()
        m.load_state_dict(sd)
        m.to(device="cuda", dtype=torch.bfloat16)
        inp = synth.make_dit_inputs(cfg, f, h, w, seed=seed, ctx_len=ctx)
        eng = m.engine("cuda")
        eng.use_graphs = False
        audio = None
        if tag == "talk":
            audio = tuple(t.cuda() for t in preprocess_audio(
                synth.make_audio_embed(4 * (f - 1) + 1, seed=seed).to(torch.bfloat16).float()))
        n0 = len(rec.seen)
        out = eng.forward(inp["x"].cuda(), torch.tensor([700.0]), inp["context"].cuda(),
                          inp["clip_feature"].cuda() if "clip_feature" in inp else None,
                          inp["y"].cuda() if "y" in inp else None, audio=audio)
        assert torch.isfinite(out).all()
        counts[tag] = len(rec.seen) - n0
        assert (f * (h // 2) * (w // 2)) % T, "the token count should not be a multiple of 128"
    seen = rec.seen
    geo = {
        "launches per forward": counts,
        "Q with ld = 3d": sum(s["ldq"] == 3 * s["W"] for s in seen),
        "context K|V with ld = 2d": sum(s["ldk"] == 2 * s["W"] for s in seen),
        "accumulate": sum(s["acc"] for s in seen),
        "qscale with d/128 partials": sum(s["parts"] == s["W"] // T for s in seen),
        "audio Q row slice at a nonzero row": sum(s["q_row0"] > 0 for s in seen),
        "Lk < 128": sum(s["Lk"] < T for s in seen),
        "ragged Lq": sum(s["Lq"] % T != 0 for s in seen),
        "(Lq, Lk, ld_q, ld_k)": sorted({(s["Lq"], s["Lk"], s["ldq"], s["ldk"]) for s in seen}),
    }
    print(f"[OK ] engine attention launches: {len(seen)}; worst err/bound={rec.worst:.3f} "
          f"max one-ulp flips={100 * rec.flips:.3f} %", flush=True)
    print(f"      recorded geometries: {json.dumps(geo)}", flush=True)
    # a later change to the engine must not quietly stop covering one of these
    for key in ("Q with ld = 3d", "context K|V with ld = 2d", "accumulate", "qscale with d/128 partials",
                "audio Q row slice at a nonzero row", "Lk < 128", "ragged Lq"):
        assert geo[key] > 0, f"the engine no longer launches: {key}"


# ----------------------------------------------------------------------------------------------------- host validation
_REJECT_SCRIPT = textwrap.dedent(r"""
    import ctypes, json
    from diffsynth import _native as nv
    lib = nv.load()
    # fake device pointers, 256-byte aligned: with no device visible nothing is ever dereferenced
    Q, K, V, O, WS, SS, FL, BT, BK, KM = (0x100000 * i for i in range(1, 11))
    L, H, ld = 256, 2, 256

    def fwd_sp(flags=FL):
        return lib.svi_attn_fwd_sp(Q, ld, K, ld, V, ld, O, ld, L, L, H, 0.088, flags, 1, 128, 0, WS, 1 << 20, None)

    def qscale(ss=SS):
        return lib.svi_attn_fwd_qscale(Q, ld, K, ld, V, ld, O, ld, L, L, H, 0.088, 0, ss, 2, 2, ld, 1e-6, None, 0, None)

    def small(bt=BT, bk=BK, km=KM):
        return lib.svi_attn_small(Q, 128, K, 128, V, 128, O, 128, 64, 64, 2, 64, 1.0, bt, bk, km, None)

    calls = {
        "baseline svi_attn_fwd_sp": lambda: fwd_sp(),
        "baseline svi_attn_fwd_qscale": lambda: qscale(),
        "baseline svi_attn_small": lambda: small(),
        "svi_attn_fwd_sp: kv_flags": lambda: fwd_sp(FL + 2),
        "svi_attn_fwd_qscale: q_sumsq": lambda: qscale(SS + 2),
        "svi_attn_small: bias_table": lambda: small(bt=BT + 2),
        "svi_attn_small: bucket": lambda: small(bk=BK + 2),
        "svi_attn_small: key_mask": lambda: small(km=KM + 1),
    }
    res = {}
    for name, call in calls.items():
        rc = call()
        res[name] = [rc, lib.svi_last_error().decode()]
    print(json.dumps(res))
""")


def test_attn_rejects_misaligned_pointers():
    """Pointers the kernels read with 4-byte scalar loads (kv_flags, q_sumsq, bias_table, bucket, key_mask) are refused
    when misaligned, before any CUDA call, with a message naming the field.  Runs in a process that sees no GPU, so a
    missing check fails later with a different message; the aligned calls get past validation."""
    if not os.path.exists(nv.lib_path()):
        pytest.skip("the kernel library is not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]))
    p = subprocess.run([sys.executable, "-c", _REJECT_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    for name, (rc, msg) in res.items():
        print(f"{name}: status {rc}: {msg}")
        if name.startswith("baseline"):
            assert rc not in (0, -1), f"{name} should pass validation and fail later without a GPU: {msg}"
        else:
            assert rc == -1 and f"{name} must be 4-byte aligned" in msg, f"{name}: not rejected by name ({msg})"


# ------------------------------------------------------------------------------------------- the model's self-tests (CPU)
def _rand_case(seed, Lq, Lk, amp):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(Lq, T, generator=g) * amp).bfloat16()
    k = (torch.randn(Lk, T, generator=g) * amp).bfloat16()
    v = torch.randn(Lk, T, generator=g).bfloat16()
    return q, k, v, torch.full((Lq,), scale_log2(T ** -0.5), dtype=torch.float64)


@pytest.mark.parametrize("Lk,split,first", [(1000, 1, 0), (1000, 3, 0), (1000, 2, 5), (4100, 8, 0), (4100, 4, 31),
                                            (129, 1, 1), (77, 1, 0)])
def test_model_without_rounding_is_exact(Lk, split, first):
    """without the bf16 rounding of P the kernel-order model is O* to fp64 precision, for any plan and visit order"""
    q, k, v, cs = _rand_case(Lk + split, 40, Lk, 2.0)
    xt = scores(q, k, cs)
    o_star, pv = exact_softmax(xt, v)
    segs = visit_segments(_cdiv(Lk, T), split, first)
    assert sorted(t for s in segs for t in s) == list(range(_cdiv(Lk, T)))
    o, _ = kernel_order(xt, v, segs, p_round=None)
    assert ((o - o_star).abs() <= 1e-12 * pv).all()


@pytest.mark.parametrize("Lk", [1, 77, 128])
def test_model_one_tile_is_the_emulation_formula(Lk):
    """for Lk <= 128 (one tile, every plan alike) the model is tests/nv_emulation.attention's bf16-P formula, in fp64"""
    import nv_emulation
    q, k, v, cs = _rand_case(Lk, 50, Lk, 3.0)
    s = (q.double() @ k.double().t()) * T ** -0.5
    p = torch.exp(s - s.amax(1, keepdim=True))
    want = (to_bf16(p).double() @ v.double()) / p.sum(1, keepdim=True)
    o, _ = kernel_order(scores(q, k, torch.full_like(cs, LOG2E * T ** -0.5)), v, visit_segments(1))
    assert ((o - want).abs() <= 1e-12 * (want.abs() + 1e-3)).all()
    emu = nv_emulation.attention(q, k, v, torch.empty(50, T, dtype=torch.bfloat16), 1, T ** -0.5)
    inside, _ = _bf16_inside(emu, to_bf16(want), 1e-6 * torch.ones(50, 1))
    assert inside.all(), "the fp32 stand-in is not within one bf16 ulp of the fp64 formula"


def test_model_plans_differ_at_peaked_scores():
    """on a peaked case two plans give different bf16 outputs, and so do two visit orders, and the bar-B check tells them
    apart: a model with one slice deleted, or with the SP order started at tile 0, fails it against the true plan's output"""
    q, k, v, cs = _rand_case(7, 256, 2048, 3.0)
    xt = scores(q, k, cs)
    n = _cdiv(2048, T)
    o1, _ = kernel_order(xt, v, visit_segments(n, 1))
    o2, amb = kernel_order(xt, v, visit_segments(n, 2), eta=torch.full((256,), 2.0 ** -21, dtype=torch.float64))
    o2w, _ = kernel_order(xt, v, visit_segments(n, 2, 5))
    got = to_bf16(o2)
    _, pv = exact_softmax(xt, v)
    floor = 8 * ULP32 * pv + amb
    def fails(o):
        t = Tally()
        out, flip = bar_b(got, to_bf16(o), floor)
        t.add(got.numel(), out=out, flip=flip)
        print(f"beyond {t.out}, flips {100 * t.share:.1f} %")
        return t.fails_b()

    assert bar_b(got, to_bf16(o2), floor) == (0, 0)
    assert fails(o1) and fails(o2w), "another plan or visit order passes bar B"
    o_del, _ = kernel_order(xt[:, :n // 2], v[:n // 2 * T], visit_segments(n // 2, 1))   # the second slice deleted
    assert fails(o_del), "a model with a slice deleted passes bar B"
