"""svi_quality_attn / svi_reward_attn and the scorers' row kernels against fp64 references, launch by launch.

Attention (quality_kernels.cu, attn_kernel<HD>).  One CTA takes 64 query rows of one head of one sequence and walks the
keys in chunks of 64, in order 0..n-1 (no split, no SP order): s = Q K^T by fp32 wgmma over hd in {64, 80} exact bf16
products, a running max m_t of the unscaled fp32 scores, p = exp2f((s - m_t) c) with c = fp32(scale fp32(log2 e)) as
launch_attn computes it, alpha = exp2f((m_old - m_new) c), P rounded fp32 -> bf16 (round to nearest even) for P V while
the row sum l takes the unrounded p, and O = o * (1 / l) (IEEE reciprocal: the library is built without fast math).  Masked
keys, keys past Lk and causal keys past the row get s = -inf; while a row's running max is -inf its reference point is 0,
so its P and alpha are exactly 0.  In exact arithmetic (s - m_t) c = x - c m_t with x = s c, so the kernel-order model of
tests/test_attention_fp64_gpu.py (kernel_order on 64-key tiles, one slice) is this kernel's model, and both references
are built, in fp64, from the bf16 values the launch reads and from the same fp32 c:
  * exact: O* = softmax_j(x_j) V over the kept keys;
  * kernel order: O_model = sum_j bf16(P_j) 2^(m_t(j) - m) v_j / sum_j 2^(x_j - m), m_t the running max in the log2 domain.

Bars, applied to every launch (u = 2^-24):
  A. |O - O*| <= eps_r (P|V|)[r, :] / l_r + half a bf16 ulp of the output + 2 fp32 ulps of |O*| + (Lk + 4 n) 2^-133 max|v|,
     (P|V|)/l = sum_j softmax_j |v_j|, n = ceil(Lk / 64), and
       eps_r = 2^-8                              bf16 P: relative error <= 2^-9 per weight, doubled for safety;
             + 2 ln2 (4 hd u c qk_r + 4 u spread_r)
                                                 s by fp32 wgmma over hd exact products: |ds_j| <= 2 hd u sum|q||k_j|
                                                 <= 2 hd u qk_r (qk_r = max over kept keys of sum|q||k_j|); p_j sees the
                                                 error of s_j and of the s that is its row's max (the intermediate maxima
                                                 telescope through the alphas), c times; the fp32 subtraction and the
                                                 product with c round the log2-domain argument by 2 u |x_j - m_t|, the
                                                 alphas after chunk t by 2 u (m - m_t) in all, spread_r = max_j (m - x_j);
                                                 an argument error dx moves a weight by ln2 dx relative, and the
                                                 normalisation by the same weights doubles it;
             + 2 n (2^-21 + u)                   exp2f (2 ulp, taken as 2^-21 relative) of every P and of at most one alpha
                                                 per chunk, and the o *= alpha / l *= alpha products;
             + (3 Lk + 8) u                      fp32 accumulation of O over Lk terms (2 Lk u) and of the row sum (Lk u),
                                                 the reciprocal and the final product.
     The absolute term covers P in the fp32 subnormal range, where bf16 rounding is absolute (2^-134) rather than relative.
  B. every element within one bf16 ulp of bf16(O_model), plus a floor of (16 + 8 (max|x| + spread)) fp32 ulps of
     (P|V|)/l and a tie term for the P whose fp32 value lies within eta_r = 2^-21 + 16 ln2 u (c qk_r + max|x| + spread_r)
     of a bf16 rounding midpoint (kernel_order's tie term), and at most MAX_FLIP of the elements one ulp away.  max|x| is
     the fp32 rounding of the scores themselves, spread the rounding of (s - m_t) c.
  C. O sits in a wider and taller NaN-filled buffer: only the [batch Lq, heads hd] region may change, and Q, K, V (and the
     NaN around them) and the mask bytes (and the bytes around them) stay bit-identical.
  Identities, bit for bit: a row with exactly one kept key is that key's V row (P = 1, l = 1) -- causal row 0 of every
  sequence among them; a repeated launch is bit-identical; sequence b of a batch of 81 equals the same sequence alone.
Negative controls, each of which must fail the bar named (bar B: a flip share of at least CONTROL_MARGIN MAX_FLIP, or
elements beyond one ulp):
  A: O* without the last kept key (cases in `bite`: a dominant or ramped last key); the causal mask off; the key mask
     ignored; K/V head h instead of head 0 under kv_heads = 1; every sequence reading sequence 0's keys; the chunked
     softmax without the alpha rescale (Lk > 64);
  B: P truncated (every case with rows of two keys or more, but the wide ramp, whose rows are all alike); the row sum over
     bf16(P) (the cases that keep rows few keys: causal diffuse rows up to L = 129 and the padding, shared and leading-chunk
     masks, 4-6 % flips; elsewhere it moves 2-4 % and is only reported); the model at chunk width 128 (Lk > 64, but
     Lk = 65, where a 128-key tile differs only where key 64 is the max, and the ramps, where the even chunk of a tile
     weighs 2^-8.7 of the odd one).

Row kernels (quality_kernels.cu / reward_kernels.cu): per-element bounds derived in each test's docstring from the
kernel's summation order (per-thread strided partials, a 5-level shuffle tree, the 8 warp sums in order), each with a
negative control that must fail it.

The explicit cases come first; test_engine_launches_* then record the launches of the seven scorers on tiny checkpoints
and of every full-size geometry, and apply bars A-C to each.  The model's self-tests (test_model_*) run on the CPU.  This
module imports without a GPU.  Its GPU cases take about 55 s on an H100 80GB HBM3 at a 700 W power limit: the fp64
references run on the device in blocks of ROW_ELEMS rows x keys.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from diffsynth import _native as nv
from test_attention_fp64_gpu import (CONTROL_MARGIN, LN2, ROW_ELEMS, Tally, _bits, _bf16_ulp, _cdiv, _rows_at, _store,
                                     _written, bar_a, bar_b, exact_softmax, kernel_order, running_max, scale_log2, scores,
                                     to_bf16, visit_segments)
from test_kernel_conformance_gpu import ULP32 as U

# entry point -> the cases of this module that check it (test_quality_cpu / test_reward_cpu fail on a name that is missing)
COVERED = {
    "svi_quality_attn": ["test_attn_case", "test_sequence_in_batch_of_81_equals_alone", "test_engine_launches_tiny_scorers",
                         "test_engine_launches_full_size"],
    "svi_reward_attn": ["test_attn_case", "test_sequence_in_batch_of_81_equals_alone", "test_engine_launches_tiny_scorers",
                        "test_engine_launches_full_size"],
    "svi_quality_embed_ln": ["test_embed_ln_fp64"],
    "svi_quality_score": ["test_score_fp64"],
    "svi_quality_quick_gelu": ["test_quality_quick_gelu_fp64"],
    "svi_reward_layernorm": ["test_reward_layernorm_fp64"],
    "svi_reward_cond_mask": ["test_reward_cond_mask_fp64"],
    "svi_reward_head": ["test_reward_head_fp64"],
    "svi_reward_swiglu": ["test_reward_swiglu_fp64"],
}
dev = "cuda"
CHUNK = 64                                # keys per chunk of attn_kernel
# one-ulp flips against bf16(O_model), measured on an H100 80GB HBM3 at a 700 W power limit: at most 0.11 % (the ramps),
# 0.003-0.09 % elsewhere in the explicit cases, 0 where every row keeps one key.  The controls that bite by flips (the row
# sum over bf16(P), the chunk width 128 on diffuse rows) move 2-20 % of the elements.
MAX_FLIP = 0.005
SUB = 2.0 ** -133                         # smallest bf16 subnormal


# ------------------------------------------------------------------------------------------------------------ helpers
def no_rescale(xt, v):
    """the chunked softmax without the alpha rescale: each weight against the running max of its own chunk"""
    R, Lk = xt.shape[0], v.shape[-2]
    M = running_max(xt, visit_segments(xt.shape[1]))
    P = torch.exp2(xt - M.masked_fill(M == -math.inf, 0.0)[:, :, None]).reshape(R, -1)[:, :Lk]
    return _rows_at(P, v.double()) / P.sum(1, keepdim=True)


def masked_scores(q, k, keep, c, tile=CHUNK):
    """scores() of groups q [G, Lq, hd], k [G, Lk, hd] with the keys outside keep [G, Lq, Lk] at -inf"""
    G, Lq, Lk = keep.shape
    xt = scores(q, k, c, tile)
    xt.view(G, Lq, -1)[:, :, :Lk].masked_fill_(~keep, -math.inf)
    return xt


def references(qb, kb, vb, kp, xt, c):
    """(O*, (P|V|)/l, eps_r, bar A's absolute term, O_model, bar B's floor) of groups qb [G, Lq, hd], kb, vb [G, Lk, hd]
    with kept keys kp [G, Lq, Lk] and their masked scores xt (64-key chunks): the terms of the module docstring"""
    G, Lq, Lk = kp.shape
    R, hd, n = G * Lq, qb.shape[-1], xt.shape[1]
    o_star, pv = exact_softmax(xt, vb)
    kept = kp.reshape(R, Lk)
    x = xt.reshape(R, -1)[:, :Lk]
    qk = (qb.double().abs() @ kb.double().abs().transpose(1, 2)).reshape(R, Lk).masked_fill(~kept, 0.0).amax(1)
    m = x.amax(1)
    xabs = x.abs().masked_fill(~kept, 0.0).amax(1)
    spread = (m[:, None] - x).masked_fill(~kept, 0.0).amax(1)
    vmax = vb.double().abs().amax((1, 2)).repeat_interleave(Lq)
    eps = (2.0 ** -8 + 2 * LN2 * (4 * hd * U * c * qk + 4 * U * spread) + 2 * n * (2.0 ** -21 + U)
           + (3 * Lk + 8) * U)[:, None]
    extra = ((Lk + 4 * n) * SUB * vmax)[:, None]
    eta = 2.0 ** -21 + 16 * LN2 * U * (c * qk + xabs + spread)
    o_mod, amb = kernel_order(xt, vb, visit_segments(n), eta=eta)
    floor = (16 + 8 * (xabs + spread))[:, None] * U * pv + amb + extra
    return o_star, pv, eps, extra, o_mod, floor


def _nans(*shape, dtype=torch.bfloat16):
    return torch.full(shape, float("nan"), device=dev, dtype=dtype)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


# ---------------------------------------------------------------------------------------------------------- one launch
class Attn:
    """One attention launch: its arguments as the C entry point sees them (views with row strides, a kv row stride and a
    mask stride in elements), a snapshot of every allocation it can see, and check() for bars A-C after it ran."""

    def __init__(self, fn, q, k, v, out, batch, Lq, Lk, heads, hd=64, kv_heads=None, kv_stride=None, mask=None,
                 mask_stride=0, scale=None, causal=False):
        torch.cuda.synchronize()
        self.fn, self.B, self.Lq, self.Lk, self.H, self.hd = fn, batch, Lq, Lk, heads, hd
        self.kvh = heads if kv_heads is None else kv_heads
        self.kvs = Lk if kv_stride is None else kv_stride
        self.mask, self.ms, self.causal = mask, mask_stride, bool(causal)
        self.scale = hd ** -0.5 if scale is None else scale
        self.q, self.k, self.v, self.out = q, k, v, out
        self.W = heads * hd
        self.stores, self.may_write = {}, {}
        for name, t in (("out", out), ("q", q), ("k", k), ("v", v), ("mask", mask)):
            if t is not None and t.untyped_storage().data_ptr() not in self.stores:
                st = _store(t)
                self.stores[t.untyped_storage().data_ptr()] = (name, st, st.clone())
        self.may_write[out.untyped_storage().data_ptr()] = _written(out, batch * Lq, self.W)
        self.snap = {n: t.clone() for n, t in (("q", q), ("k", k), ("v", v)) if t is not None}
        self.mask_snap = None if mask is None else mask.clone()

    def launch(self, out=None):
        """the C entry point on this launch's arguments (out: another buffer of the same layout)"""
        o = self.out if out is None else out
        lib, st = nv.load(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        ld = lambda t: t.stride(0)                                                   # noqa: E731
        if self.fn == "quality":
            assert self.Lq == self.Lk == self.kvs and self.kvh == self.H and self.mask is None
            rc = lib.svi_quality_attn(_p(self.q), ld(self.q), _p(self.k), ld(self.k), _p(self.v), ld(self.v), _p(o), ld(o),
                                      self.B, self.Lq, self.H, self.hd, self.scale, int(self.causal), st)
        else:
            assert self.hd == 64 and not self.causal
            rc = lib.svi_reward_attn(_p(self.q), ld(self.q), _p(self.k), ld(self.k), _p(self.v), ld(self.v), _p(o), ld(o),
                                     self.B, self.Lq, self.Lk, self.H, self.kvh, self.kvs, _p(self.mask), self.ms,
                                     self.scale, st)
        assert rc == 0, nv.load().svi_last_error().decode()
        return o

    # --------------------------------------------------------------------------------------------------------------
    def check_memory(self, name):
        torch.cuda.synchronize()
        for key, (what, st, before) in self.stores.items():
            same = _bits(st) == _bits(before) if st.dtype != torch.uint8 else st == before
            idx = self.may_write.get(key)
            if idx is not None:
                same[idx] = True
            assert bool(same.all()), f"{name}: the launch changed {int((~same).sum())} elements of the {what} " \
                                     f"allocation outside what it may write"

    def _heads(self, t, head_of=None):
        """K or V of every (sequence, head) as fp64 [B, H, Lk, hd]: rows b kv_stride + j, columns of head
        head_of(h) (default: h, or 0 under kv_heads = 1), read from the snapshot of the launch's view"""
        B, H, Lk, hd = self.B, self.H, self.Lk, self.hd
        rows = (torch.arange(B, device=t.device)[:, None] * self.kvs + torch.arange(Lk, device=t.device)).reshape(-1)
        if head_of is None:
            x = t[rows].double().view(B, Lk, self.kvh, hd).transpose(1, 2)
            return x.expand(B, H, Lk, hd)
        return torch.stack([t[rows, head_of(h) * hd:(head_of(h) + 1) * hd].double().view(B, Lk, hd) for h in range(H)], 1)

    def _keep(self, mask=True, causal=True):
        """kept keys [B, 1, Lq, Lk]"""
        B, Lq, Lk = self.B, self.Lq, self.Lk
        keep = torch.ones(B, 1, Lq, Lk, dtype=torch.bool, device=dev)
        if mask and self.mask is not None:
            idx = torch.arange(B, device=dev)[:, None] * self.ms + torch.arange(Lk, device=dev)
            keep &= (self.mask_snap[idx] != 0)[:, None, None, :]
        if causal and self.causal:
            keep &= (torch.arange(Lk, device=dev)[None, :] <= torch.arange(Lq, device=dev)[:, None])[None, None]
        return keep

    def _groups(self, t, tail):
        """[B, H or 1, ...] -> [B H, *tail], materialised"""
        return t.expand(self.B, self.H, *tail).reshape(self.B * self.H, *tail)

    def check(self, name, controls=True, bite=(), unrequire=(), quiet=False):
        """bars A-C, the single-kept-key identity and the negative controls of this launch; returns what was measured"""
        self.check_memory(name)
        B, H, Lq, Lk, hd = self.B, self.H, self.Lq, self.Lk, self.hd
        G, n = B * H, _cdiv(Lk, CHUNK)
        c = scale_log2(self.scale)
        Q = self._groups(self.snap["q"].double().view(B, Lq, H, hd).transpose(1, 2), (Lq, hd))
        K = self._groups(self._heads(self.snap["k"]), (Lk, hd))
        V = self._groups(self._heads(self.snap["v"]), (Lk, hd))
        keep = self._groups(self._keep(), (Lq, Lk))
        got_all = self.out.view(B, Lq, H, hd).transpose(1, 2).reshape(G, Lq, hd)
        alt = {}                                        # control -> (K, V, keep) replacing the launch's
        if controls:
            if self.causal and Lq > 1:
                alt["A: causal mask off"] = (K, V, self._groups(self._keep(causal=False), (Lq, Lk)))
            if self.mask is not None and not bool(keep.all()):
                alt["A: key mask ignored"] = (K, V, self._groups(self._keep(mask=False), (Lq, Lk)))
            if self.kvh == 1 and H > 1:
                fits = [h for h in range(H) if all(self._cols_fit(t, h) for t in ("k", "v"))]
                if len(fits) > 1:
                    wrong = {t: self._groups(self._heads(self._wide(t), lambda h: h if h in fits else 0), (Lk, hd))
                             for t in ("k", "v")}
                    alt["A: K/V head h instead of head 0"] = (wrong["k"], wrong["v"], keep)
            if B > 1 and self.kvs > 0:
                first = lambda t: t.view(B, H, *t.shape[1:])[:1].expand(B, H, *t.shape[1:]).reshape(t.shape)  # noqa: E731
                alt["A: every sequence reads sequence 0's keys"] = (first(K), first(V), keep)
        A, Bt, ctl = Tally(), Tally(), {}
        ident = 0
        gb = max(1, ROW_ELEMS // (Lq * n * CHUNK))
        for g0 in range(0, G, gb):
            sl = slice(g0, min(G, g0 + gb))
            qb, kb, vb, kp = Q[sl], K[sl], V[sl], keep[sl]
            R = qb.shape[0] * Lq
            xt = masked_scores(qb, kb, kp, c)
            o_star, pv, eps, extra, o_mod, floor = references(qb, kb, vb, kp, xt, c)
            kept = kp.reshape(R, Lk)
            got = got_all[sl].reshape(R, hd)
            n_el = got.numel()
            out, worst = bar_a(got, o_star, pv, eps, extra)
            A.add(n_el, out=out, worst=worst)
            out, flip = bar_b(got, to_bf16(o_mod), floor)
            Bt.add(n_el, out=out, flip=flip)
            # a row with exactly one kept key: P = 1, l = 1, every other P and alpha 0 -> that key's V row, bit for bit
            one = kept.sum(1) == 1
            if bool(one.any()):
                key = kept.float().argmax(1)
                want = vb[torch.arange(R, device=dev) // Lq, key]
                bad = one & (got.double() != want).any(1)
                assert not bool(bad.any()), f"{name}: {int(bad.sum())} rows with one kept key differ from its V row"
                ident += int(one.sum())
            if not controls:
                continue

            def ctl_a(cname, ref):
                ctl.setdefault(cname, Tally()).add(n_el, out=bar_a(got, ref, pv, eps, extra)[0])

            def ctl_b(cname, o):
                out_, flip_ = bar_b(got, to_bf16(o), floor)
                ctl.setdefault(cname, Tally()).add(n_el, out=out_, flip=flip_)

            two = kept.sum(1) >= 2
            if bool(two.any()):
                last = Lk - 1 - kept.flip(1).float().argmax(1)
                k2 = kept.clone()
                rows = two.nonzero().squeeze(1)
                k2[rows, last[rows]] = False
                ctl_a("A: last kept key dropped", exact_softmax(masked_scores(qb, kb, k2.view_as(kp), c), vb)[0])
            for cname, (Ka, Va, keepa) in alt.items():
                ctl_a(cname, exact_softmax(masked_scores(qb, Ka[sl], keepa[sl], c), Va[sl])[0])
            if n >= 2:
                ctl_a("A: no alpha rescale", no_rescale(xt, vb))
            ctl_b("B: P truncated", kernel_order(xt, vb, visit_segments(n), p_round="trunc")[0])
            ctl_b("B: row sum of bf16(P)", kernel_order(xt, vb, visit_segments(n), rowsum="bf16")[0])
            if n >= 2:
                x128 = masked_scores(qb, kb, kp, c, tile=128)
                ctl_b("B: chunk width 128", kernel_order(x128, vb, visit_segments(x128.shape[1]))[0])

        ok = A.out == 0 and Bt.out == 0 and Bt.share <= MAX_FLIP
        if not quiet:
            print(f"[{'OK ' if ok else 'BAD'}] {name}: A worst err/bound={A.worst:.3f} B one-ulp flips="
                  f"{100 * Bt.share:.3f} % beyond={Bt.out} one-key rows={ident}", flush=True)
            for k_, t in ctl.items():
                print(f"      control {k_}: {'A outside' if k_.startswith('A') else 'B beyond'}={t.out} "
                      f"flips={100 * t.share:.2f} % of {t.n}", flush=True)
        assert A.out == 0, f"{name}: {A.out} elements outside the fp64 bound of bar A"
        assert Bt.out == 0, f"{name}: {Bt.out} elements beyond one bf16 ulp of the kernel-order model"
        assert Bt.share <= MAX_FLIP, f"{name}: {100 * Bt.share:.3f} % one-ulp flips, more than {100 * MAX_FLIP} %"
        if not controls:
            return dict(worst=A.worst, flips=Bt.share, n=Bt.n, ident=ident, controls={})
        required = ({k_ for k_ in ctl if k_.startswith("A:")} - {"A: last kept key dropped"}
                    | {"B: P truncated", "B: chunk width 128"} & set(ctl)) - set(unrequire) | set(bite)
        for k_ in sorted(required):
            assert k_ in ctl, f"{name}: control '{k_}' does not apply to this launch"
            t = ctl[k_]
            caught = t.out > 0 if k_.startswith("A") else (t.out > 0 or t.share >= CONTROL_MARGIN * MAX_FLIP)
            assert caught, f"{name}: negative control '{k_}' passes its bar (flips {100 * t.share:.2f} %)"
        return dict(worst=A.worst, flips=Bt.share, n=Bt.n, ident=ident,
                    controls={k_: (t.out, t.share) for k_, t in ctl.items()})

    def _wide(self, which):
        """the snapshot of K or V's whole rows: [rows, ld - column offset] from the launch's view onwards"""
        t = getattr(self, which)
        st = self.stores[t.untyped_storage().data_ptr()][2]
        rows, ld = (self.B - 1) * self.kvs + self.Lk, t.stride(0)
        width = ld - t.storage_offset() % ld
        return torch.as_strided(st, (rows, width), (ld, 1), t.storage_offset())

    def _cols_fit(self, which, h):
        t = getattr(self, which)
        return (h + 1) * self.hd <= t.stride(0) - t.storage_offset() % t.stride(0)


# ------------------------------------------------------------------------------------------------------------- inputs
def _buf(rows, cols, data=None, pad_rows=3, pad_cols=8, row0=0):
    """a NaN-filled [row0 + rows + pad_rows, cols + pad_cols] buffer and its [rows, cols] view at (row0, 0)"""
    b = _nans(row0 + rows + pad_rows, cols + pad_cols)
    v = b[row0:row0 + rows, :cols]
    if data is not None:
        v.copy_(data)
    return v


def _mask(kind, B, Lk, ms, g):
    """the mask bytes of a launch, inside a larger buffer whose other bytes are 0xAB: [(B-1) ms + Lk] (ms > 0) or [Lk]"""
    nseq = B if ms else 1
    m = torch.zeros(nseq, Lk, dtype=torch.uint8)
    for b in range(nseq):
        if kind == "pad":                       # a padded prompt: keys [0, n_b); sequence 0 keeps one key only
            m[b, :1 if b == 0 else int(torch.randint(1, Lk + 1, (1,), generator=g))] = 1
        elif kind == "random":
            m[b] = (torch.rand(Lk, generator=g) > 0.35).to(torch.uint8)
            m[b, int(torch.randint(0, Lk, (1,), generator=g))] = 1
        elif kind == "last":                    # only the last key, alone in a ragged last chunk
            m[b, Lk - 1] = 1
        elif kind == "late":                    # the first two chunks fully masked
            m[b, 2 * CHUNK:] = (torch.rand(Lk - 2 * CHUNK, generator=g) > 0.3).to(torch.uint8)
            m[b, 2 * CHUNK + int(torch.randint(0, Lk - 2 * CHUNK, (1,), generator=g))] = 1
        else:
            raise ValueError(kind)
    n = (B - 1) * ms + Lk if ms else Lk
    buf = torch.full((n + 37,), 0xAB, dtype=torch.uint8)
    for b in range(nseq):
        buf[b * ms:b * ms + Lk] = m[b]
        if ms > Lk and b + 1 < nseq:            # the gap between sequences: bytes that would be read by a wrong stride
            buf[b * ms + Lk:(b + 1) * ms] = torch.tensor([0, 1] * ms)[:ms - Lk].to(torch.uint8)
    d = buf.to(dev)
    return d[:n]


def _qkv(case, g):
    """bf16 q [B Lq, H hd], k, v [kv rows, kvh hd] of a case's score regime (CPU)"""
    B, Lq, Lk, H, hd = case["B"], case["Lq"], case["Lk"], case["H"], case.get("hd", 64)
    kvh = case.get("kvh", H)
    kvs = _kvs(case)
    kv_rows = (B - 1) * kvs + Lk if kvs else Lk
    regime = case.get("regime", "diffuse")
    amp = {"diffuse": 1.0, "peaked": 3.0}.get(regime, 1.0)
    q = torch.randn(B * Lq, H * hd, generator=g) * amp
    k = torch.randn(kv_rows, kvh * hd, generator=g) * amp
    v = torch.randn(kv_rows, kvh * hd, generator=g)
    j = (torch.arange(kv_rows) % max(kvs, Lk) if kvs else torch.arange(kv_rows)).float()
    if regime == "ramp":                        # every score gains 30 key / (Lk - 1): the row max rises in every chunk
        q.view(B * Lq, H, hd)[:, :, 0] = 4.0
        k.view(kv_rows, kvh, hd)[:, :, 0] += 60.0 * j[:, None] / max(Lk - 1, 1)
    elif regime == "wide":                      # x_j ~ 2.45 j: every chunk spans over 150 log2 units
        q.zero_()
        q.view(B * Lq, H, hd)[:, :, 0] = 8.0
        k.zero_()
        k.view(kv_rows, kvh, hd)[:, :, 0] = 1.7 * j[:, None]
    q, k, v = q.bfloat16(), k.bfloat16(), v.bfloat16()
    if regime == "wide":
        # column 0 of every head of V: 1 where the fp32 P of the last chunk is subnormal (2^-148 < P < 2^-128), 0 elsewhere,
        # so the output's column 0 is made of subnormal P alone and shows whether the kernel keeps them
        x = k.view(kv_rows, kvh, hd)[:, 0, 0].double() * 8.0 * scale_log2(hd ** -0.5)
        d = x.max() - x
        sub = (d > 128) & (d < 148) & (torch.arange(kv_rows) >= (Lk - 1) // CHUNK * CHUNK)
        v.view(kv_rows, kvh, hd)[:, :, 0] = sub.to(torch.bfloat16)[:, None]
    return q, k, v


def _kvs(case):
    s = case.get("kvs", "Lk")
    return {"Lk": case["Lk"], "Lk+13": case["Lk"] + 13, 0: 0}[s]


def _ms(case):
    s = case.get("ms", "Lk")
    return {"Lk": case["Lk"], "Lk+5": case["Lk"] + 5, 0: 0}[s]


def make_launch(case, seed):
    """the case's inputs laid out as its layout names, NaN around them, and its Attn"""
    g = torch.Generator().manual_seed(seed)
    B, Lq, Lk, H, hd = case["B"], case["Lq"], case["Lk"], case["H"], case.get("hd", 64)
    kvh, fn = case.get("kvh", H), case.get("fn", "reward")
    q0, k0, v0 = _qkv(case, g)
    W, KW = H * hd, kvh * hd
    layout = case.get("layout", "fused" if fn == "quality" else "cross")
    if layout == "fused":                       # the towers: q | k | v column slices of one [rows, 3d] output (Lq = Lk)
        qkv = _buf(B * Lq, 3 * W)
        qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:] = q0.to(dev), k0.to(dev), v0.to(dev)
        q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    elif layout == "mps self":                  # MPS self-attention: q | k | v of [rows, d + 2 64], one K/V head
        qkv = _buf(B * Lq, W + 2 * KW)
        qkv[:, :W], qkv[:, W:W + KW], qkv[:, W + KW:] = q0.to(dev), k0.to(dev), v0.to(dev)
        q, k, v = qkv[:, :W], qkv[:, W:W + KW], qkv[:, W + KW:]
    elif layout == "cross":                     # q of its own; k | v column slices of one [kv rows, 2 kvh hd] output
        q = _buf(B * Lq, W, q0.to(dev), row0=2)
        kv = _buf(k0.shape[0], 2 * KW)
        kv[:, :KW], kv[:, KW:] = k0.to(dev), v0.to(dev)
        k, v = kv[:, :KW], kv[:, KW:]
    elif layout == "wide kv":                   # one K/V head read from [kv rows, H 64] buffers holding other heads' data
        q = _buf(B * Lq, W, q0.to(dev))
        kw, vw = (torch.randn(k0.shape[0], W, generator=g).bfloat16().to(dev) for _ in range(2))
        kw[:, :KW], vw[:, :KW] = k0.to(dev), v0.to(dev)
        k, v = kw[:, :KW], vw[:, :KW]
    else:
        raise ValueError(layout)
    ms = _ms(case) if case.get("mask") else 0
    mask = _mask(case["mask"], B, Lk, ms, g) if case.get("mask") else None
    obuf = _nans(B * Lq + 9, W + 24)
    out = obuf[4:4 + B * Lq, 8:8 + W]
    return Attn(fn, q, k, v, out, B, Lq, Lk, H, hd, kvh, _kvs(case), mask, ms, hd ** -0.5, case.get("causal", False))


# ---------------------------------------------------------------------------------------------------- explicit cases
RAMP_UNREQUIRE = ("B: chunk width 128",)
# masks that leave rows few keys: the rounding of one P is a visible share of l (4-6 % flips)
ROWSUM = ("B: row sum of bf16(P)",)
# every row keeps one key: P = 1 and l = 1 whatever the rounding, order or chunking
ONE_KEY_UNREQUIRE = ("A: no alpha rescale", "B: P truncated", "B: chunk width 128")


def _quality_cases():
    """svi_quality_attn: every length of {1, 63, 64, 65, 128, 129, 257, 320}, hd 64 and 80, each causal and not"""
    out = {}
    for i, L in enumerate((1, 63, 64, 65, 128, 129, 257, 320)):
        for hd in (64, 80):
            for causal in (False, True):
                B = (1, 7, 81)[(i + hd // 16 + causal) % 3]
                H = 16 if B == 1 else (4 if B == 7 else 2)
                regime = ("diffuse", "peaked")[(i + causal) % 2]
                # one key: P = 1 whatever the rounding; Lk = 65: a 128-key tile differs only where key 64 is the max
                unreq = (("B: P truncated",) if L == 1 else
                         ("B: chunk width 128",) + (("A: no alpha rescale",) if causal else ()) if L == 65 else ())
                # the row sum over bf16(P) separates where rows keep few keys: causal rows of diffuse scores (4-5 % flips)
                bite = ("B: row sum of bf16(P)",) if causal and regime == "diffuse" and L <= 129 and L > 1 else ()
                out[f"quality L={L} hd={hd}{' causal' if causal else ''} B={B} H={H} {regime}"] = dict(
                    fn="quality", B=B, Lq=L, Lk=L, H=H, hd=hd, causal=causal, regime=regime, unrequire=unreq, bite=bite)
    # on ramps the even chunks of a 128-key tile weigh 2^-8.7 of the odd ones (2^-150 on the wide ramp): chunk width 128
    # rounds differently only where it hardly matters
    out["quality L=320 hd=80 causal B=3 H=2 ramp"] = dict(fn="quality", B=3, Lq=320, Lk=320, H=2, hd=80, causal=True,
                                                          regime="ramp", bite=("A: last kept key dropped",),
                                                          unrequire=RAMP_UNREQUIRE)
    out["quality L=257 hd=64 B=2 H=3 ramp"] = dict(fn="quality", B=2, Lq=257, Lk=257, H=3, regime="ramp",
                                                   bite=("A: last kept key dropped",), unrequire=RAMP_UNREQUIRE)
    out["quality L=320 hd=64 B=1 H=2 wide"] = dict(fn="quality", B=1, Lq=320, Lk=320, H=2, regime="wide",
                                                   bite=("A: last kept key dropped",),
                                                   unrequire=RAMP_UNREQUIRE + ("B: P truncated",))
    return out


CASES = {
    **_quality_cases(),
    # svi_reward_attn: Lq != Lk both ways, K/V layouts, masks
    "reward 35->197 B=7 H=12 BERT cross": dict(B=7, Lq=35, Lk=197, H=12),
    "reward 257->77 B=7 H=16 kvh=1 shared K/V, shared mask": dict(B=7, Lq=257, Lk=77, H=16, kvh=1, kvs=0, mask="random",
                                                                  ms=0, bite=ROWSUM),
    "reward 130->77 B=7 H=2 kvh=1 kv stride Lk+13": dict(B=7, Lq=130, Lk=77, H=2, kvh=1, kvs="Lk+13", layout="wide kv"),
    "reward 257 B=7 H=16 kvh=1 MPS self": dict(B=7, Lq=257, Lk=257, H=16, kvh=1, layout="mps self"),
    "reward 257 B=1 H=16 kvh=1 wide kv peaked": dict(B=1, Lq=257, Lk=257, H=16, kvh=1, layout="wide kv", regime="peaked"),
    "reward 35 B=81 H=12 padding mask": dict(B=81, Lq=35, Lk=35, H=12, mask="pad", bite=ROWSUM),
    "reward 65->129 B=7 H=3 padding mask stride Lk+5": dict(B=7, Lq=65, Lk=129, H=3, mask="pad", ms="Lk+5", bite=ROWSUM),
    "reward 63->320 B=7 H=2 shared K/V, per-sequence masks": dict(B=7, Lq=63, Lk=320, H=2, kvs=0, mask="random"),
    "reward 64->129 B=7 H=2 only the last key (ragged chunk) kept": dict(B=7, Lq=64, Lk=129, H=2, mask="last",
                                                                         ms="Lk+5", unrequire=ONE_KEY_UNREQUIRE),
    "reward 129->257 B=1 H=4 kvh=1 only the last key kept": dict(B=1, Lq=129, Lk=257, H=4, kvh=1, mask="last", ms=0,
                                                                 layout="wide kv", unrequire=ONE_KEY_UNREQUIRE),
    "reward 77->200 B=7 H=2 first two chunks masked": dict(B=7, Lq=77, Lk=200, H=2, mask="late", bite=ROWSUM),
    "reward 257->1 B=7 H=2": dict(B=7, Lq=257, Lk=1, H=2, unrequire=("B: P truncated",)),
    "reward 1->320 B=81 H=2 peaked": dict(B=81, Lq=1, Lk=320, H=2, regime="peaked"),
    "reward 320 B=1 H=2 ramp": dict(B=1, Lq=320, Lk=320, H=2, regime="ramp", bite=("A: last kept key dropped",),
                                    unrequire=RAMP_UNREQUIRE),
    "reward 197->35 B=81 H=16 peaked": dict(B=81, Lq=197, Lk=35, H=16, regime="peaked"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_attn_case(name):
    """one explicit launch: bars A-C with the negative controls, the single-kept-key identity, and a repeated launch
    bit-identical"""
    case = CASES[name]
    L = make_launch(case, seed=sum(map(ord, name)))
    L.launch()
    L.check(name, bite=case.get("bite", ()), unrequire=case.get("unrequire", ()))
    again = torch.full_like(L.out, float("nan"))
    L.launch(again)
    torch.cuda.synchronize()
    assert torch.equal(_bits(again), _bits(L.out)), f"{name}: a repeated launch is not bit-identical"
    if case.get("regime") == "wide":
        _check_subnormal_column(L)


def _check_subnormal_column(L):
    """column 0 of every head is made of P in the fp32 subnormal range alone (V is 0 on every other key): the kernel must
    keep them (fp32 P, bf16 P, wgmma accumulation and the final scaling without flush to zero), within 2^-7 relative of
    the kernel-order model plus one bf16 subnormal step"""
    B, H, Lq, Lk, hd = L.B, L.H, L.Lq, L.Lk, L.hd
    c = scale_log2(L.scale)
    q = L.snap["q"].double().view(B * Lq, H, hd)[:, 0]
    k = L._heads(L.snap["k"])[0, 0]
    v = L._heads(L.snap["v"])[0, 0]
    xt = scores(q, k, torch.full((B * Lq,), c, dtype=torch.float64, device=dev), CHUNK)
    o_mod = kernel_order(xt, v, visit_segments(xt.shape[1]))[0][:, 0]
    got = L.out.view(B * Lq, H, hd)[:, :, 0].double()
    n_sub = int(((v[:, 0] != 0)).sum())
    print(f"      subnormal P per row: {n_sub}; column 0 model {o_mod.min().item():.3e}..{o_mod.max().item():.3e}, "
          f"got {got.min().item():.3e}..{got.max().item():.3e}", flush=True)
    assert n_sub > 0 and bool((o_mod > 0).all()) and bool((o_mod < 2.0 ** -126).all())
    assert bool((got > 0).all()), "the kernel flushed subnormal P to zero"
    assert bool(((got - o_mod[:, None]).abs() <= 2.0 ** -7 * o_mod[:, None] + SUB).all())


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ["quality", "reward"])
def test_sequence_in_batch_of_81_equals_alone(fn):
    """sequence b of a batch of 81 is bit-identical to the same sequence launched alone (the header's promise): one CTA
    computes one (64-row block, head, sequence) from that sequence's rows alone"""
    if fn == "quality":
        case = dict(fn="quality", B=81, Lq=257, Lk=257, H=16, hd=80)
    else:
        case = dict(B=81, Lq=35, Lk=197, H=12, mask="pad")
    L = make_launch(case, seed=81)
    L.launch()
    L.check(f"{fn} batch of 81", controls=False)
    Lq, Lk, kvs = L.Lq, L.Lk, L.kvs
    for b in (0, 40, 80):
        kv = slice(b * kvs, b * kvs + Lk)
        mask = None if L.mask is None else L.mask[b * L.ms:b * L.ms + Lk]
        one = Attn(L.fn, L.q[b * Lq:(b + 1) * Lq], L.k[kv], L.v[kv], _nans(Lq, L.W), 1, Lq, Lk, L.H, L.hd, L.kvh, Lk, mask,
                   0, L.scale, L.causal)
        one.launch()
        torch.cuda.synchronize()
        assert torch.equal(_bits(one.out), _bits(L.out[b * Lq:(b + 1) * Lq])), f"{fn}: sequence {b} differs alone"


# ------------------------------------------------------------------------------------------------ the engines' launches
class Recorder:
    """Stands in for nv.quality_attn / nv.reward_attn: snapshots, launches the kernel, applies bars A-C to the launch with
    its own arguments (every launch, or the first of each geometry) and lets the engine carry on with the output."""

    def __init__(self, first_only=False):
        self.quality_attn, self.reward_attn = nv.quality_attn, nv.reward_attn
        self.first_only = first_only
        self.geo, self.count, self.checked, self.worst, self.flips = {}, 0, 0, 0.0, 0.0

    def _run(self, key, make, call):
        self.count += 1
        if self.first_only and key in self.geo:
            return call()
        L = make()
        out = call()
        r = L.check(f"engine {key}", controls=False, quiet=True)
        self.checked += 1
        self.geo.setdefault(key, r)
        self.worst, self.flips = max(self.worst, r["worst"]), max(self.flips, r["flips"])
        return out

    def quality(self, q, k, v, out, batch, num_heads, head_dim, scale, causal=False):
        L = q.shape[0] // batch
        key = ("quality", L, L, num_heads, head_dim, "causal" if causal else "", "")
        return self._run(key, lambda: Attn("quality", q, k, v, out, batch, L, L, num_heads, head_dim, scale=scale,
                                           causal=causal),
                         lambda: self.quality_attn(q, k, v, out, batch, num_heads, head_dim, scale, causal))

    def reward(self, q, k, v, out, batch, num_heads, scale, kv_heads=None, kv_shared=False, key_mask=None):
        Lq = q.shape[0] // batch
        Lk = k.shape[0] if kv_shared else k.shape[0] // batch
        ms = Lk if key_mask is not None and key_mask.numel() == batch * Lk and batch > 1 else 0
        kvh = num_heads if kv_heads is None else kv_heads
        key = ("reward", Lq, Lk, num_heads, kvh, "shared" if kv_shared else "", "" if key_mask is None else "mask")
        return self._run(key, lambda: Attn("reward", q, k, v, out, batch, Lq, Lk, num_heads, 64, kvh, 0 if kv_shared else Lk,
                                           None if key_mask is None else key_mask.reshape(-1), ms, scale),
                         lambda: self.reward_attn(q, k, v, out, batch, num_heads, scale, kv_heads, kv_shared, key_mask))

    def install(self, monkeypatch):
        monkeypatch.setattr(nv, "quality_attn", self.quality)
        monkeypatch.setattr(nv, "reward_attn", self.reward)


@pytest.mark.gpu
def test_engine_launches_tiny_scorers(monkeypatch, tmp_path):
    """every attention launch of the seven scorers scoring frames on the tiny checkpoints, against bars A-C"""
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    from tools import synth_quality as SQ
    from tools import synth_reward as SR
    paths, _ = SQ.write_tiny_checkpoints(str(tmp_path / "quality"))
    paths = dict(paths, **SR.write_reward_checkpoints(str(tmp_path / "reward"))[0])
    frames = [SQ.frames(1, h, w, seed=i)[0] for i, (h, w) in enumerate([(40, 70), (71, 33), (97, 120)])]
    for name in ("CLIP", "HPSv2", "HPSv2.1", "PickScore", "Aesthetic", "ImageReward", "MPS"):
        rec = Recorder()
        rec.install(monkeypatch)
        model = load_preference_model(name, device=dev, path=paths)
        got = model.score(frames, SR.PROMPTS[2])
        assert len(got) == 3 and all(math.isfinite(x) for x in got)
        print(f"[OK ] {name}: {rec.count} attention launches checked; worst err/bound={rec.worst:.3f} "
              f"max one-ulp flips={100 * rec.flips:.3f} %; geometries {sorted(rec.geo)}", flush=True)
        assert rec.count == rec.checked > 0
        monkeypatch.undo()


def _one_layer(conf):
    return {k: (dict(v, num_hidden_layers=1) if k in ("vision_config", "text_config") else v) for k, v in conf.items()}


@pytest.mark.gpu
def test_engine_launches_full_size(monkeypatch):
    """the first launch of every full-size geometry -- ViT-H/14 (257 tokens, 16 heads x 80), ViT-L/14 (257, 16 x 64), the
    causal 77-token text towers, BLIP ViT-L/16 (197), BERT self-attention (35, padding mask) and cross-attention
    (35 -> 197), MPS cross-attention (257 -> 77, shared K/V, one head, condition mask) and self-attention (257, one K/V
    head after RoPE) -- on the synthetic full-size weights with one layer per tower (the launch geometry does not depend
    on the depth)"""
    from diffsynth.extensions.ImageQualityMetric import towers as T
    from diffsynth.extensions.ImageQualityMetric.reward import (CrossModel, ImageRewardEngine, ImageRewardModel,
                                                                MPSEngine, MPSModel)
    from tools import synth_quality as SQ
    from tools import synth_reward as SR
    rec = Recorder(first_only=True)
    rec.install(monkeypatch)
    g = torch.Generator().manual_seed(5)
    fr = SQ.frames(2, 480, 832, seed=3)
    ids = torch.randint(1, 49000, (1, 77), generator=g)
    ids[0, 0], ids[0, 15], ids[0, 16:] = 49406, 49407, 0
    per = {}

    def tally(tag):
        per[tag] = sorted(k for k in rec.geo if k not in sum(per.values(), []))

    cfg = dict(SQ.OPENCLIP_FULL, vision_cfg=dict(SQ.OPENCLIP_FULL["vision_cfg"], layers=1),
               text_cfg=dict(SQ.OPENCLIP_FULL["text_cfg"], layers=1))
    m = T.OpenCLIP(**cfg)
    m.load_state_dict(SQ.openclip_state_dict(cfg, seed=11), strict=True)
    eng = m.engine(dev)
    eng.vision.encode_images(torch.stack([T.openclip_pixels(f, 224) for f in fr]))
    eng.text.encode_text(ids)
    tally("open_clip ViT-H/14")
    conf = _one_layer(SQ.HF_FULL_LARGE)
    h = T.HFCLIPModel(conf)
    h.load_state_dict(SQ.hf_state_dict(conf, seed=21), strict=True)
    eng = h.engine(dev)
    eng.vision.encode_images(torch.stack([T.openclip_pixels(f, 224) for f in fr]))
    eng.text.encode_text(ids[:, :19])
    tally("CLIP ViT-L/14")
    med, vis = SR.med_config(30524, layers=1), dict(SR.FULL_VISION, layers=1)
    sd = SR.imagereward_state_dict(med, vis, seed=51, extra=False)
    with torch.device("meta"):
        ir = ImageRewardModel(med, **vis)
    ir.load_state_dict(sd, strict=True, assign=True)
    bids = torch.randint(1000, 30000, (1, 35), generator=g)
    bids[0, 0], bids[0, 20], bids[0, 21:] = 101, 102, 0
    ImageRewardEngine(ir, dev).score(torch.stack([T.blip_pixels(f, 224) for f in fr]), bids, (bids != 0).long())
    tally("ImageReward")
    conf = _one_layer(SQ.HF_FULL_PICK)
    sd = {k: v for k, v in SR.mps_state_dict(conf, layers=1, seed=61).items() if "inv_freq" not in k}
    with torch.device("meta"):
        mp = MPSModel(conf, CrossModel.sizes(sd))
    mp.load_state_dict(sd, strict=True, assign=True)
    cids = torch.randint(1, 49000, (1, 77), generator=g)
    cids[0, 0], cids[0, 40], cids[0, 41:] = 49406, 49407, 49407
    MPSEngine(mp, dev, T.OPENAI_MEAN, T.OPENAI_STD).score(torch.stack([T.openclip_pixels(f, 224) for f in fr]), ids, cids)
    tally("MPS")
    for tag, keys in per.items():
        w = max((rec.geo[k]["worst"] for k in keys), default=0.0)
        f = max((rec.geo[k]["flips"] for k in keys), default=0.0)
        print(f"[OK ] full size {tag}: geometries {keys}; worst err/bound={w:.3f} max one-ulp flips={100 * f:.3f} %",
              flush=True)
    print(f"      {rec.count} launches, {rec.checked} checked", flush=True)
    want = {"ViT-H/14": ("quality", 257, 257, 16, 80, "", ""), "ViT-L/14": ("quality", 257, 257, 16, 64, "", ""),
            "BERT self-attention": ("reward", 35, 35, 12, 12, "", "mask"),
            "BERT cross-attention": ("reward", 35, 197, 12, 12, "", ""),
            "MPS cross-attention": ("reward", 257, 77, 16, 1, "shared", "mask"),
            "MPS self-attention": ("reward", 257, 257, 16, 1, "", "")}
    for what, key in want.items():
        assert key in rec.geo, f"no launch of {what}: {key} not in {sorted(rec.geo)}"
    assert any(k[0] == "quality" and k[1] == 77 and k[5] == "causal" for k in rec.geo), "no causal text-tower launch"
    assert any(k[1] == k[2] == 197 for k in rec.geo), "no BLIP ViT-L/16 launch"


# ------------------------------------------------------------------------------------------------------ the row kernels
def _depth(n):
    """additions on the longest path of block_sum over n values (256 threads): the per-thread strided partials, the
    5-level shuffle tree, the 8 warp sums in order"""
    return _cdiv(n, 256) + 5 + 8


def _outside(got, ref, bound):
    """elements outside |got - ref| <= bound (NaN counts as outside)"""
    return int((~((got.double() - ref).abs() <= bound)).sum())


def _report(name, got, ref, bound, controls):
    """bar and controls of one row-kernel case: every element inside, every control outside somewhere"""
    err = (got.double() - ref).abs()
    worst = (err / bound.clamp_min(1e-300)).max().item()
    out = _outside(got, ref, bound)
    print(f"[{'OK ' if out == 0 else 'BAD'}] {name}: worst err/bound={worst:.3f}", flush=True)
    res = {}
    for cname, cref in controls.items():
        res[cname] = _outside(got, cref, bound)
        print(f"      control {cname}: outside={res[cname]}", flush=True)
    assert out == 0, f"{name}: {out} elements outside the fp64 bound"
    return res


def ln_bound(v, d, mean_abs, var, rstd, gamma, beta, D, eps, u_in):
    """per-element bound of the LayerNorm kernels (layernorm_kernel, embed_ln_kernel), first order with 1 % slack.
    mean: 21 additions of the block sum (8 per thread, 5 shuffles, 8 warp sums) and the division, plus the inputs'
    own rounding u_in (embed: fp32 src + pos): E_m = (22 u + u_in) mean|v|, the cancellation term (u |mean| rstd when
    the mean is far from 0);  d_j = v_j - mean: E_m + u_in |v_j| + u |d_j|;  variance: 26 u var (the sum of squares, the
    products, the division, the rounding of each d) + the square of the largest d error + 2 u_in sum|d v| / D (the mean's
    own error is common to every d and sum d = 0, so it enters squared);  rstd = rsqrtf (2 ulp = 4 u) of fl(var + eps):
    eps_r = (dvar + u (var + eps)) / (2 (var + eps)) + 4 u;  y = fl(fl(fl(d rstd) gamma) + beta): 2 u |gamma d rstd|
    + u |y|."""
    E_m = (22 * U + u_in) * mean_abs
    e_max = (E_m + u_in * v.abs() + U * d.abs()).amax(1, keepdim=True)
    dvar = 26 * U * var + e_max ** 2 + 2 * u_in * (d.abs() * v.abs()).sum(1, keepdim=True) / D
    eps_r = (dvar + U * (var + eps)) / (2 * (var + eps)) + 4 * U
    a = (gamma * d).abs() * rstd
    y = d * rstd * gamma + beta
    return 1.01 * (gamma.abs() * rstd * (E_m + u_in * v.abs() + U * d.abs()) + a * (eps_r + 3 * U) + U * y.abs()), y


def _ln_ref(v, gamma, beta, eps, u_in, unbiased=False, eps_outside=False):
    D = v.shape[1]
    mean = v.mean(1, keepdim=True)
    d = v - mean
    var = (d * d).sum(1, keepdim=True) / (D - 1 if unbiased else D)
    rstd = 1 / (var.sqrt() + eps) if eps_outside else (var + eps).rsqrt()
    return ln_bound(v, d, v.abs().mean(1, keepdim=True), var, rstd, gamma, beta, D, eps, u_in)


def _ln_rows(M, D, g):
    """rows of every regime: 3 randn + 1, mean 1e4 with std 0.1, std 1e-6 around 0, constant 1.5"""
    x = 3 * torch.randn(M, D, generator=g, dtype=torch.float64) + 1
    q = M // 4
    x[q:2 * q] = 1e4 + 0.1 * torch.randn(q, D, generator=g, dtype=torch.float64)
    x[2 * q:3 * q] = 1e-6 * torch.randn(q, D, generator=g, dtype=torch.float64)
    x[3 * q:] = 1.5
    return x.float(), q


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 260, 2044, 2048])
@pytest.mark.parametrize("inplace", [False, True])
def test_reward_layernorm_fp64(D, inplace):
    """svi_reward_layernorm at eps = 1e-12 (BERT) against the fp64 LayerNorm, y f32 within ln_bound and yb bf16 within it
    plus half a bf16 ulp (and bf16(y) bit for bit); a constant row whose fp32 sums are exact gives y = beta bit for bit.
    Controls: the unbiased variance, eps outside the square root (the std-1e-6 rows, var ~ eps)."""
    g = torch.Generator().manual_seed(D + inplace)
    x, q = _ln_rows(48, D, g)
    gam, bet = (1 + 0.2 * torch.randn(D, generator=g)).float(), (0.1 * torch.randn(D, generator=g)).float()
    xd = x.to(dev)
    y = xd if inplace else torch.full_like(xd, float("nan"))
    yb = torch.full((48, D), float("nan"), device=dev, dtype=torch.bfloat16)
    nv.reward_layernorm(xd, gam.to(dev), bet.to(dev), 1e-12, y, yb)
    torch.cuda.synchronize()
    vd, gd, bd = x.double().to(dev), gam.double().to(dev), bet.double().to(dev)
    bound, ref = _ln_ref(vd, gd, bd, 1e-12, 0.0)
    ctl = {"unbiased variance": _ln_ref(vd, gd, bd, 1e-12, 0.0, unbiased=True)[1],
           "eps outside the square root": _ln_ref(vd, gd, bd, 1e-12, 0.0, eps_outside=True)[1]}
    res = _report(f"reward_layernorm D={D} {'in place' if inplace else 'out of place'}", y, ref, bound, ctl)
    half = 0.5 * torch.maximum(_bf16_ulp(yb.float()), _bf16_ulp(ref.float())).double()
    assert _outside(yb, ref, bound + half) == 0, "yb outside the bound plus half a bf16 ulp"
    assert torch.equal(_bits(yb), _bits(y.to(torch.bfloat16))), "yb is not bf16(y)"
    assert torch.equal(y[3 * q:], bet.to(dev).expand(48 - 3 * q, D)), "a constant row does not give beta"
    assert res["unbiased variance"] > 0 and res["eps outside the square root"] > 0, res


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 260, 2044, 2048])
def test_embed_ln_fp64(D):
    """svi_quality_embed_ln for B = 81 images of 2 patches at eps = 1e-5 (open_clip's ln_pre) and 1e-12: LN([cls; patch]
    + pos) against fp64, within ln_bound with u_in = u for the fp32 sum with the position row.  Control: the class
    token without its position row."""
    g = torch.Generator().manual_seed(D)
    B, n = 81, 2
    patch, _ = _ln_rows(B * n, D, g)
    cls = (3 * torch.randn(D, generator=g)).float()
    pos = (0.5 * torch.randn(n + 1, D, generator=g)).float()
    gam, bet = (1 + 0.2 * torch.randn(D, generator=g)).float(), (0.1 * torch.randn(D, generator=g)).float()
    res = {}
    for eps in (1e-5, 1e-12):
        out = torch.full((B * (n + 1), D), float("nan"), device=dev)
        nv.quality_embed_ln(*(t.to(dev) for t in (patch, cls, pos, gam, bet)), eps, out)
        torch.cuda.synchronize()
        src = torch.cat([cls.double()[None, None].expand(B, 1, D), patch.double().view(B, n, D)], 1)
        v = (src + pos.double()[None]).reshape(-1, D).to(dev)
        gd, bd = gam.double().to(dev), bet.double().to(dev)
        bound, ref = _ln_ref(v, gd, bd, eps, U)
        v_wrong = src.clone()
        v_wrong[:, 1:] += pos.double()[None, 1:]
        ctl = {"a missing pos row": _ln_ref(v_wrong.reshape(-1, D).to(dev), gd, bd, eps, U)[1]}
        res[eps] = _report(f"quality_embed_ln D={D} eps={eps:g}", out, ref, bound, ctl)["a missing pos row"]
    assert all(r > 0 for r in res.values()), res


def _score_ref(img, txt, w, bias, clamp=True):
    """fp64 cosines and aesthetic head with their bounds: per row norm, eps_n = (depth + 1) u / 2 + 2 u for the sum of
    squares, sqrtf (IEEE) and 1 / x (IEEE); each product term fl(fl(x ni) fl(y nt)) 3 u; the dot's block sum depth u"""
    E = img.shape[1]
    dep = _depth(E)
    ni = img.norm(dim=1, keepdim=True)
    nt = txt.norm(dim=1, keepdim=True)
    if clamp:
        ni, nt = ni.clamp_min(1e-12), nt.clamp_min(1e-12)
    en = (dep + 1) * U / 2 + 2 * U
    cos = (img / ni) @ (txt / nt).t()
    cb = ((dep + 3) * U + 2 * en) * ((img.abs() / ni) @ (txt.abs() / nt).t()) * 1.01
    aes = (img / ni) @ w + bias
    ab = (((dep + 2) * U + en) * ((img.abs() / ni) @ w.abs()) + U * aes.abs()) * 1.01
    return cos, cb, aes, ab


@pytest.mark.gpu
@pytest.mark.parametrize("E", [1, 767, 4096])
def test_score_fp64(E):
    """svi_quality_score, B = 81 images against T = 3 texts and the aesthetic head: within the bounds of _score_ref; an
    all-zero feature row gives cosines of exactly 0 and the head's bias exactly.  Control: no 1e-12 clamp (NaN)."""
    g = torch.Generator().manual_seed(E)
    B, T = 81, 3
    img = torch.randn(B, E, generator=g, dtype=torch.float64).float()
    txt = (torch.randn(T, E, generator=g, dtype=torch.float64) * 0.05 + 0.02).float()
    img[7] = 0
    txt[1] = 0
    w = torch.randn(E, generator=g).float()
    cos = torch.full((B, T), float("nan"), device=dev)
    aes = torch.full((B,), float("nan"), device=dev)
    nv.quality_score(img.to(dev), txt.to(dev), cos, w.to(dev), 0.25, aes)
    torch.cuda.synchronize()
    i64, t64, w64 = img.double().to(dev), txt.double().to(dev), w.double().to(dev)
    rc, cb, ra, ab = _score_ref(i64, t64, w64, float(np.float32(0.25)))
    nc = _score_ref(i64, t64, w64, float(np.float32(0.25)), clamp=False)
    res = _report(f"quality_score cos E={E}", cos, rc, cb, {"no 1e-12 clamp on a zero row": nc[0]})
    res |= _report(f"quality_score aesthetic E={E}", aes, ra, ab, {"no 1e-12 clamp on a zero row": nc[2]})
    assert bool((cos[7] == 0).all()) and bool((cos[:, 1] == 0).all()), "a zero feature row gives a nonzero cosine"
    assert aes[7].item() == np.float32(0.25)
    assert res["no 1e-12 clamp on a zero row"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("E", [1, 767, 4096])
def test_reward_head_fp64(E):
    """svi_reward_head: out_b = w . row 0 of sequence b + bias for B = 81 sequences of L = 35 rows with ldx > E: within
    (depth + 1) u sum|x||w| + u |out|.  Control: row 1 of each sequence."""
    g = torch.Generator().manual_seed(E + 1)
    B, L = 81, 35
    x = torch.randn(B * L, E + 3, generator=g)
    w = torch.randn(E, generator=g)
    out = torch.full((B,), float("nan"), device=dev)
    xd = x.to(dev)
    nv.reward_head(xd[:, :E], B, w.to(dev), 0.25, out)
    torch.cuda.synchronize()
    r = x.double().to(dev).view(B, L, E + 3)[:, :, :E]
    w64 = w.double().to(dev)
    ref = r[:, 0] @ w64 + float(np.float32(0.25))
    bound = 1.01 * ((_depth(E) + 1) * U * (r[:, 0].abs() @ w64.abs()) + U * ref.abs())
    res = _report(f"reward_head E={E}", out, ref, bound, {"row 1 of each sequence": r[:, 1] @ w64 + 0.25})
    assert res["row 1 of each sequence"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("E", [1, 767, 4096])
def test_reward_cond_mask_fp64(E):
    """svi_reward_cond_mask: sim_i = max_j t_i . c_j (each dot within delta_ij = (depth + 1) u sum|t_i||c_j|, so the max
    within delta_i = max_j delta_ij), ratio = fl(sim_i / max sim): |r - r*| <= (delta_i + |r*| delta_m) / (mx - delta_m)
    + u |r*|; keep bits exact wherever |r* - threshold| is above that bound.  Control: the similarity to the first
    condition token only."""
    g = torch.Generator().manual_seed(E + 2)
    Lt, Lc, thr = 77, 41, 0.3
    text = (torch.randn(Lt, E, generator=g) * torch.linspace(-0.2, 1.0, Lt)[:, None] + 0.05).float()
    cond = (torch.randn(Lc, E, generator=g) + 0.05).float()
    if E == 1:
        text, cond = text.abs() * torch.linspace(-0.2, 1.0, Lt)[:, None], cond.abs()
    ratio = torch.full((Lt,), float("nan"), device=dev)
    keep = torch.full((Lt,), 7, device=dev, dtype=torch.uint8)
    nv.reward_cond_mask(text.to(dev), cond.to(dev), thr, ratio, keep)
    torch.cuda.synchronize()
    t64, c64 = text.double().to(dev), cond.double().to(dev)
    sims = t64 @ c64.t()
    dl = (_depth(E) + 1) * U * (t64.abs() @ c64.abs().t())
    sim, di = sims.amax(1), dl.amax(1)
    mx, dm = sim.max(), di.max()
    assert mx > 10 * dm
    ref = sim / mx
    bound = 1.01 * ((di + ref.abs() * dm) / (mx - dm) + U * ref.abs())
    wrong = sims[:, 0] / sims[:, 0].max()
    res = _report(f"reward_cond_mask E={E}", ratio, ref, bound, {"first condition token only": wrong})
    far = (ref - float(np.float32(thr))).abs() > bound
    want = (ref > float(np.float32(thr))).to(torch.uint8)
    assert torch.equal(keep[far], want[far]), "keep differs on a token far from the threshold"
    print(f"      {int((~far).sum())} of {Lt} ratios within their bound of the threshold", flush=True)
    assert res["first condition token only"] > 0


def _bf16_bar(got, ref, rel, floor):
    """|got - ref| <= half a bf16 ulp + rel |ref| + floor (the fp32 value's error, then one rounding to bf16)"""
    half = 0.5 * torch.maximum(_bf16_ulp(got.float()), _bf16_ulp(ref.float())).double()
    return half + rel * ref.abs() + floor + SUB / 2


def _act_inputs(M, N, seed):
    x = torch.randn(M, N + 8, generator=torch.Generator().manual_seed(seed)) * 4
    sp = torch.tensor([-100.0, -89.0, -60.0, -20.0, -1e-30, 0.0, -0.0, 1e-30, 20.0, 100.0])
    x.view(-1)[:sp.numel()] = sp
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 767, 4096])
def test_reward_swiglu_fp64(F):
    """svi_reward_swiglu y = bf16(a g / (1 + expf(-g))) against fp64: expf (2 ulp, 4 u), the sum, the division and the
    product leave 7 u relative before the bf16 rounding; below g = -88.7 expf(-g) overflows and the kernel gives 0 where
    the exact value is below 2^-120 |a|.  Control: a and g swapped."""
    M = 37
    x = _act_inputs(M, 2 * F, F)
    y = torch.zeros(M, F + 16, device=dev, dtype=torch.bfloat16)
    nv.reward_swiglu(x.to(dev)[:, :2 * F], y[:, :F])
    torch.cuda.synchronize()
    a, gt = x.double().to(dev)[:, :F], x.double().to(dev)[:, F:2 * F]
    sil = lambda t: t * torch.sigmoid(t)                                                     # noqa: E731
    ref = (sil(gt) * a).nan_to_num(0.0)
    floor = torch.where(gt < -88.0, 2.0 ** -120 * a.abs(), torch.zeros_like(a))
    bound = _bf16_bar(y[:, :F], ref, 7 * U, floor)
    res = _report(f"reward_swiglu F={F}", y[:, :F], ref, bound, {"a and g swapped": (sil(a) * gt).nan_to_num(0.0)})
    assert bool((y[:, F:] == 0).all()), "columns past F were written"
    assert res["a and g swapped"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 767, 4096])
def test_quality_quick_gelu_fp64(N):
    """svi_quality_quick_gelu y = bf16(v / (1 + expf(-1.702f v))) against fp64 with the fp32 constant: the argument's
    rounding (u |1.702 v|) and expf (4 u) scale by e / (1 + e); the sum, the reciprocal and the product add 3 u; below
    v = -52 expf overflows to give 0 where the exact value is below 2^-120.  Control: GELU-erf."""
    M = 37
    x = _act_inputs(M, N, N + 5)[:, :N + 8]
    y = torch.zeros(M, N + 16, device=dev, dtype=torch.bfloat16)
    nv.quality_quick_gelu(x.to(dev)[:, :N], y[:, :N])
    torch.cuda.synchronize()
    v = x.double().to(dev)[:, :N]
    K = float(np.float32(1.702))
    e = torch.exp(-K * v)
    ref = (v * torch.sigmoid(K * v)).nan_to_num(0.0)
    rel = (4 * U + U * (K * v).abs()) * (e / (1 + e)).nan_to_num(1.0) + 3 * U
    floor = torch.where(K * v < -88.0, torch.full_like(v, 2.0 ** -120), torch.zeros_like(v))
    bound = _bf16_bar(y[:, :N], ref, rel, floor)
    erf = (v * 0.5 * (1 + torch.erf(v / math.sqrt(2)))).nan_to_num(0.0)
    res = _report(f"quality_quick_gelu N={N}", y[:, :N], ref, bound, {"GELU-erf": erf})
    assert bool((y[:, N:] == 0).all()), "columns past N were written"
    assert res["GELU-erf"] > 0


# ------------------------------------------------------------------------------------------- the model's self-tests (CPU)
def _cpu_groups(seed, G, Lq, Lk, amp, hd=64):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(G, Lq, hd, generator=g) * amp).bfloat16().double()
    k = (torch.randn(G, Lk, hd, generator=g) * amp).bfloat16().double()
    v = torch.randn(G, Lk, hd, generator=g).bfloat16().double()
    return q, k, v, scale_log2(hd ** -0.5)


def _keep(G, Lq, Lk, seed, causal=False, lead=0):
    g = torch.Generator().manual_seed(seed)
    keep = torch.rand(G, 1, Lk, generator=g) > 0.3
    keep[:, :, lead:lead + 1] = True
    keep[:, :, :lead] = False
    keep = keep.expand(G, Lq, Lk).clone()
    if causal:
        keep &= torch.arange(Lk)[None, :] <= torch.arange(Lq)[:, None]
        keep[:, :, 0] = True
    return keep


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("Lk,causal,lead", [(320, False, 0), (257, True, 0), (129, False, 128), (200, False, 130)])
def test_model_without_rounding_is_exact(tile, Lk, causal, lead):
    """without the bf16 rounding of P the kernel-order model is O* to fp64 precision, at either chunk width, with key
    masks, causal masks and fully masked leading chunks"""
    q, k, v, c = _cpu_groups(Lk + tile, 3, Lk if causal else 40, Lk, 2.0)
    keep = _keep(3, q.shape[1], Lk, Lk, causal, lead)
    xt = masked_scores(q, k, keep, c, tile)
    o_star, pv = exact_softmax(xt, v)
    o, _ = kernel_order(xt, v, visit_segments(xt.shape[1]), p_round=None)
    assert torch.isfinite(o).all() and ((o - o_star).abs() <= 1e-12 * pv).all()


@pytest.mark.parametrize("Lk", [1, 40, 64])
def test_model_one_chunk_is_the_bf16_p_formula(Lk):
    """with one chunk the model is sum bf16(P_j) v_j / sum P_j, P against the row max"""
    q, k, v, c = _cpu_groups(Lk, 2, 50, Lk, 3.0)
    xt = masked_scores(q, k, torch.ones(2, 50, Lk, dtype=torch.bool), c)
    x = xt.reshape(100, -1)[:, :Lk]
    p = torch.exp2(x - x.amax(1, keepdim=True))
    want = (to_bf16(p).double().view(2, 50, Lk) @ v).reshape(100, -1) / p.sum(1, keepdim=True)
    o, _ = kernel_order(xt, v, visit_segments(1))
    assert ((o - want).abs() <= 1e-12 * (want.abs() + 1e-3)).all()


def test_model_fully_masked_leading_chunk_contributes_nothing():
    """a fully masked leading chunk (running max -inf, reference point 0) gives P = alpha = 0, not NaN: the model of keys
    [0, 192) with the first two chunks masked equals, bit for bit, the model of keys [128, 192) alone"""
    q, k, v, c = _cpu_groups(9, 2, 30, 192, 2.0)
    keep = torch.ones(2, 30, 192, dtype=torch.bool)
    keep[:, :, :128] = False
    xt = masked_scores(q, k, keep, c)
    o, _ = kernel_order(xt, v, visit_segments(3))
    tail = masked_scores(q, k[:, 128:], keep[:, :, 128:], c)
    o_tail, _ = kernel_order(tail, v[:, 128:], visit_segments(1))
    assert torch.isfinite(o).all()
    torch.testing.assert_close(o, o_tail, rtol=1e-15, atol=0)


def _model_controls(q, k, v, keep, c, got=None):
    """bars A / B on got (default: bf16 of the model itself) and the outside counts of each control"""
    G, Lq, Lk = keep.shape
    xt = masked_scores(q, k, keep, c)
    o_star, pv, eps, extra, o_mod, floor = references(q, k, v, keep, xt, c)
    got = to_bf16(o_mod) if got is None else got
    n = xt.shape[1]
    res = {"bar A": bar_a(got, o_star, pv, eps, extra)[0], "bar B": bar_b(got, to_bf16(o_mod), floor)}
    res["A: no alpha rescale"] = bar_a(got, no_rescale(xt, v), pv, eps, extra)[0]
    for name, o in (("B: P truncated", kernel_order(xt, v, visit_segments(n), p_round="trunc")[0]),
                    ("B: row sum of bf16(P)", kernel_order(xt, v, visit_segments(n), rowsum="bf16")[0]),
                    ("B: chunk width 128", kernel_order(masked_scores(q, k, keep, c, 128), v,
                                                         visit_segments(_cdiv(Lk, 128)))[0])):
        res[name] = bar_b(got, to_bf16(o), floor)
    return res, o_star, pv, eps, extra


def test_model_negative_controls_fail_their_bars():
    """on model-generated outputs (bf16 of O_model) bars A and B pass, and every negative control fails its bar: the A
    controls by elements outside, the B controls by elements beyond one ulp or a flip share of CONTROL_MARGIN MAX_FLIP"""
    q, k, v, c = _cpu_groups(3, 4, 64, 320, 1.0)
    keep = _keep(4, 64, 320, 4)
    res, o_star, pv, eps, extra = _model_controls(q, k, v, keep, c)
    print(res)
    assert res["bar A"] == 0 and res["bar B"] == (0, 0)
    assert res["A: no alpha rescale"] > 0
    n_el = 4 * 64 * 64
    for name in ("B: P truncated", "B: chunk width 128"):
        out, flip = res[name]
        assert out > 0 or flip >= CONTROL_MARGIN * MAX_FLIP * n_el, name
    # the row sum over bf16(P) shows where a row keeps few keys: the rounding of one P is a visible share of l
    few = torch.zeros(4, 64, 320, dtype=torch.bool)
    few[:, :, 100], few[:, :, 190], few[:, :, 300] = True, True, True
    q3, k3, v3, _ = _cpu_groups(5, 4, 64, 320, 0.5)
    out, flip = _model_controls(q3, k3, v3, few, c)[0]["B: row sum of bf16(P)"]
    assert out > 0 or flip >= CONTROL_MARGIN * MAX_FLIP * n_el
    # the A controls that change the keys or values: the causal mask off, the key mask ignored, another head's or
    # another sequence's K/V, the last kept key dropped (here a dominant one)
    causal = _keep(4, 64, 320, 4, causal=True)
    got = to_bf16(_model_controls(q, k, v, causal, c)[1])
    xt_off = masked_scores(q, k, keep, c)
    _, pv_c, eps_c, extra_c = [_model_controls(q, k, v, causal, c)[i] for i in (0, 2, 3, 4)]
    assert bar_a(got, exact_softmax(xt_off, v)[0], pv_c, eps_c, extra_c)[0] > 0, "causal mask off"
    full = torch.ones_like(keep)
    assert bar_a(to_bf16(o_star), exact_softmax(masked_scores(q, k, full, c), v)[0], pv, eps, extra)[0] > 0, "mask ignored"
    other = exact_softmax(masked_scores(q, k.roll(1, 0), keep, c), v.roll(1, 0))[0]
    assert bar_a(to_bf16(o_star), other, pv, eps, extra)[0] > 0, "another group's K/V"
    k_dom = k.clone()
    k_dom[:, 300] = q.mean(1) * 8                    # the last kept key dominates
    keep_d = keep.clone()
    keep_d[:, :, 301:] = False
    keep_d[:, :, 300] = True
    _, o_d, pv_d, eps_d, extra_d = _model_controls(q, k_dom, v, keep_d, c)
    drop = keep_d.clone()
    drop[:, :, 300] = False
    assert bar_a(to_bf16(o_d), exact_softmax(masked_scores(q, k_dom, drop, c), v)[0], pv_d, eps_d, extra_d)[0] > 0
