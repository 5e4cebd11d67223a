"""GPU: every kernel wrapper of diffsynth._native against its torch stand-in (tests/nv_emulation*.py) on identical device
inputs.  The CPU engine tests assume the stand-ins compute what the kernels compute; this module checks that assumption.

Outputs are prefilled with NaN, so an element the kernel never writes fails, and where a kernel takes a leading dimension
it is larger than the width.  Three bars, by kind of kernel:
  - data movement and plain casts: bit-exact (torch.equal; padding columns must be exactly zero);
  - fp32 math stored as bf16: every element within one bf16 ulp of the stand-in's value, plus an absolute floor of a few
    fp32 ulps of the row's scale (cancellation near zero).  The fp32 results differ by reassociation and by the MUFU
    exp / rcp / rsqrt approximations (~1e-6 relative, common.cuh), below a bf16 ulp, so at most one rounding can flip;
  - fp32 outputs: a few fp32 ulps of the magnitude of the terms (FMA contraction, reassociation).
GEMM and attention keep tolerance bars here; their sharp checks are the gemm_edges section of tools/gpu_check.py and the
per-element fp64 bars of tests/test_attention_fp64_gpu.py.  Every bar has a negative control: a wrong but plausible reference must fail it.

COVERED / EXEMPT list every entry point of include/svi_b200.h; tests/test_kernel_coverage_cpu.py fails when one is missing.
This module imports without a GPU.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import nv_emulation as E
import nv_emulation_audio as EA
from diffsynth import _native as nv

# entry point -> the cases that run it: "A:<test function of this module>", "B:<tools/gpu_check.py section>" or
# "F:<test function of tests/test_attention_fp64_gpu.py>"
COVERED = {
    "svi_gemm_bf16": ("A:test_gemm_matches_standin", "B:gemm", "B:gemm_epi", "B:gemm_edges", "B:ln_fold"),
    "svi_attn_fwd": ("A:test_attention_matches_standin", "B:attn", "B:attn_online", "B:attn_bench", "F:test_attention_case",
                     "F:test_accumulate_image_branch", "F:test_bench_shape_sampled", "F:test_engine_launches"),
    "svi_attn_workspace_bytes": ("B:attn", "B:attn_online", "B:attn_sp_one_gpu", "F:test_attention_case", "F:test_sp_one_gpu"),
    "svi_attn_fwd_qscale": ("A:test_attention_matches_standin", "B:abi3", "F:test_qscale_layouts", "F:test_engine_launches"),
    "svi_attn_fwd_sp": ("B:attn_sp_one_gpu", "F:test_sp_one_gpu"),
    "svi_attn_plan": ("F:test_plans_are_distinct", "F:test_attention_case"),
    "svi_layernorm_modulate": ("A:test_layernorm_modulate",),
    "svi_layernorm_modulate_split": ("A:test_split_forms",),
    "svi_rmsnorm_rope": ("A:test_rmsnorm_rope",),
    "svi_qk_norm_rope": ("A:test_rmsnorm_rope",),
    "svi_patchify_gather": ("A:test_patchify_unpatchify",),
    "svi_patchify_gather_split": ("A:test_patchify_unpatchify",),
    "svi_unpatchify": ("A:test_patchify_unpatchify",),
    "svi_cfg_euler_step": ("A:test_f32_arithmetic",),
    "svi_cast_f32_to_bf16": ("A:test_casts",),
    "svi_cast_bf16_to_f32": ("A:test_casts",),
    "svi_split_f32_to_bf16x2": ("A:test_split_forms",),
    "svi_ln_fold_prepare": ("A:test_ln_fold_vectors",),
    "svi_ln_fold_combine": ("A:test_ln_fold_vectors",),
    "svi_zero": ("A:test_small_data_movement",),
    "svi_act_f32_to_bf16": ("A:test_act_f32_to_bf16",),
    "svi_add_rows": ("A:test_small_data_movement",),
    "svi_axpby": ("A:test_f32_arithmetic",),
    "svi_conv3d_causal": ("B:conv", "B:conv_tiles"),
    "svi_vae_norm_act": ("A:test_vae_norm_act",),
    "svi_vae_upsample2x": ("A:test_vae_layout",),
    "svi_vae_space_to_depth": ("A:test_vae_layout",),
    "svi_vae_space_to_depth_act": ("A:test_vae_layout",),
    "svi_vae_from_planar": ("A:test_vae_planar",),
    "svi_vae_to_planar": ("A:test_vae_planar",),
    "svi_frames_to_uint8": ("B:abi3",),
    "svi_softmax_rows": ("A:test_softmax_rows",),
    "svi_embedding_gather": ("A:test_small_data_movement",),
    "svi_rmsnorm_affine": ("A:test_encoder_norms",),
    "svi_layernorm_f32": ("A:test_encoder_norms",),
    "svi_mul_bf16": ("A:test_small_data_movement",),
    "svi_attn_small": ("A:test_attention_small_matches_standin", "B:attn_small_long", "F:test_attention_small_case"),
    "svi_col_stats_workspace_bytes": ("A:test_col_stats",),
    "svi_col_stats": ("A:test_col_stats",),
    "svi_col_norm_act": ("A:test_col_norm_act",),
    "svi_conv1d_gather": ("A:test_conv1d_gather",),
    "svi_interp_layernorm": ("A:test_interp_layernorm",),
}
EXEMPT = {
    "svi_abi_version": "constant; checked by build()",
    "svi_last_error": "message accessor; every wrapper reads it when a call fails",
    "svi_sm_count": "device query; every grid-capped launch uses it",
    "svi_sp_alloc": "needs two GPUs (test_sp_gpu.py)",
    "svi_sp_free": "needs two GPUs (test_sp_gpu.py)",
    "svi_sp_open": "needs two GPUs (test_sp_gpu.py)",
    "svi_sp_close": "needs two GPUs (test_sp_gpu.py)",
    "svi_sp_push": "needs two GPUs (test_sp_gpu.py)",
}

pytestmark = pytest.mark.gpu
dev = "cuda"
ULP32 = 2.0 ** -24          # half the fp32 spacing at 1: the unit of the fp32 bars
# GELU-tanh on inputs of std 3 (act_f32_to_bf16, split_f32_to_bf16x2): 1.17 % one-ulp flips measured on an H100 80GB HBM3
# at a 400 W power limit (every other case: <= 0.1 %).  The kernels' x * sigmoid(2u) takes exp2 of an fp32 argument that
# grows like x^3, whose rounding costs ~1e-5 relative for x < -3.  Against the former fp32 stand-in the share was 7.5 %.
GELU_TANH_MAX_FLIP = 0.02


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def rnd(g, *shape, scale=1.0, shift=0.0, dtype=torch.float32):
    return (torch.randn(*shape, generator=g) * scale + shift).to(dev, dtype)


def nans(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device=dev, dtype=dtype)


def _bf16_ulp(x):
    """spacing of bf16 numbers at |x| (0 at 0)"""
    _, e = torch.frexp(x.float())
    return torch.where(x == 0, torch.zeros_like(x, dtype=torch.float32), torch.ldexp(torch.ones_like(x, dtype=torch.float32), e - 8))


# ---------------------------------------------------------------------------------------------------------------- bars
def exact(name, got, ref, wrong=None):
    """bit-exact bar; `wrong` (a plausible but wrong reference) must fail it"""
    ok = got.dtype == ref.dtype and got.shape == ref.shape and torch.equal(got, ref)
    print(f"[{'OK ' if ok else 'BAD'}] exact {name}", flush=True)
    if not ok and got.shape == ref.shape:
        d = ~(got == ref)
        print(f"      {int(d.sum())} of {d.numel()} elements differ; first at {d.nonzero()[0].tolist()}")
    assert ok, f"{name}: not bit-exact"
    if wrong is not None:
        caught = not torch.equal(got, wrong)
        print(f"      negative control fails the bar: {caught}")
        assert caught, f"{name}: the exact bar does not catch the wrong reference"


def _bf16_inside(got, ref, floor):
    got, ref = got.float(), ref.float()
    ulp = torch.maximum(_bf16_ulp(got), _bf16_ulp(ref))
    err = (got - ref).abs()
    return err <= ulp + floor, err


def bf16_ulp(name, got, ref, wrong=None, floor_ulps=4.0, max_flip=0.01):
    """each element of the bf16 output within one bf16 ulp of the stand-in's bf16 value, plus floor_ulps fp32 ulps of the
    row's scale, and at most max_flip of the elements one ulp away (a kernel that rounds the wrong way, e.g. truncates,
    flips about half of them).  Measured on an H100 80GB HBM3 at a 400 W power limit: at most 0.1 % flips for every case
    of this module but GELU-tanh (GELU_TANH_MAX_FLIP), most below 0.005 %.  Returns the share of flips."""
    got2, ref2 = got.reshape(-1, got.shape[-1]), ref.reshape(-1, ref.shape[-1])
    floor = floor_ulps * ULP32 * ref2.float().abs().amax(dim=1, keepdim=True)
    ok_el, err = _bf16_inside(got2, ref2, floor)
    flip = (got2.float() != ref2.float()).float().mean().item()
    ok = bool(ok_el.all())
    print(f"[{'OK ' if ok else 'BAD'}] bf16 1-ulp {name}: one-ulp flips {100 * flip:.3f} % max_err={err.max().item():.3e}",
          flush=True)
    if not ok:
        bad = (~ok_el).nonzero()
        r, c = bad[0].tolist()
        print(f"      {bad.shape[0]} elements outside; first [{r},{c}] got={got2[r, c].item()} ref={ref2[r, c].item()}")
    assert ok, f"{name}: elements beyond one bf16 ulp of the stand-in"
    if max_flip is not None:
        assert flip <= max_flip, f"{name}: {100 * flip:.2f} % one-ulp flips, more than {100 * max_flip:.2f} %"
    if wrong is not None:
        wrong2 = wrong.reshape(-1, wrong.shape[-1]).to(ref.dtype)
        caught = not bool(_bf16_inside(got2, wrong2, floor)[0].all())
        print(f"      negative control fails the bar: {caught}")
        assert caught, f"{name}: the 1-ulp bar does not catch the wrong reference"
    return flip


def f32_ulps(name, got, ref, mag, k=4.0, wrong=None):
    """fp32 bar: |got - ref| <= k * 2^-24 * mag elementwise, mag = the magnitude of the terms that were added"""
    err = (got.float() - ref.float()).abs()
    bar = k * ULP32 * mag.float().expand_as(err)
    ok_el = err <= bar
    ok = bool(ok_el.all())
    ratio = (err / bar.clamp_min(1e-38)).max().item()
    print(f"[{'OK ' if ok else 'BAD'}] fp32 {k:g}-ulp {name}: max_err={err.max().item():.3e} worst err/bar={ratio:.3f}", flush=True)
    assert ok, f"{name}: beyond {k} fp32 ulps of the stand-in"
    if wrong is not None:
        caught = not bool(((got.float() - wrong.float()).abs() <= bar).all())
        print(f"      negative control fails the bar: {caught}")
        assert caught, f"{name}: the fp32 bar does not catch the wrong reference"


def tol_bar(name, got, ref, tol):
    """max-norm yardstick for GEMM / attention: max|got - ref| <= tol * max|ref|"""
    err = (got.float() - ref.float()).abs().max().item()
    scale = ref.float().abs().max().item()
    ok = math.isfinite(err) and err <= tol * scale
    print(f"[{'OK ' if ok else 'BAD'}] tol {name}: max_err={err:.3e} ref_max={scale:.3e} tol={tol}", flush=True)
    assert ok, f"{name}: max_err {err:.3e} > {tol} * {scale:.3e}"


def _shift_rows(t):
    """the neighbouring row's values: an off-by-one row / pixel index"""
    return torch.roll(t, 1, dims=0)


# ---------------------------------------------------------------------------------------------------------- bit-exact
def test_casts():
    g = _gen(100)
    n = 1_000_003
    x = rnd(g, n, scale=3.0)
    x[:8] = torch.tensor([0.0, -0.0, 1e-30, -1e-38, 3.0e38, 1.00390625, 1.01171875, -2.00781250], device=dev)   # ties
    got, ref = nans(n, dtype=torch.bfloat16), nans(n, dtype=torch.bfloat16)
    nv.cast_f32_to_bf16(x, got)
    E.cast_f32_to_bf16(x, ref)
    trunc = (x.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)     # truncation instead of RNE
    exact("cast_f32_to_bf16", got, ref, wrong=trunc)
    b = rnd(g, n, scale=5.0, dtype=torch.bfloat16)
    got32, ref32 = nans(n), nans(n)
    nv.cast_bf16_to_f32(b, got32)
    E.cast_bf16_to_f32(b, ref32)
    exact("cast_bf16_to_f32", got32, ref32, wrong=torch.roll(ref32, 1))


def test_small_data_movement():
    g = _gen(101)
    for rows, rows_t, D in [(12, 6, 256), (30, 30, 1536), (40, 1, 36), (6 * 30, 6, 1540)]:
        tb, tt = rnd(g, rows, D), rnd(g, rows_t, D)
        got, ref = nans(rows, D), nans(rows, D)
        nv.add_rows(tb, tt, got)
        E.add_rows(tb, tt, ref)
        wrong = tb + tt.repeat_interleave(rows // rows_t, 0)       # row j using t[j // (rows / rows_t)]
        exact(f"add_rows rows={rows} rows_t={rows_t} D={D}", got, ref, wrong=wrong if rows_t not in (1, rows) else None)
    for nbytes in (4, 12, 4096 + 8, 3 << 20):
        z = rnd(g, nbytes // 4)
        nv.zero_(z)
        exact(f"zero_ {nbytes} bytes", z, torch.zeros_like(z))
    vocab, dim = 1000, 4096 + 2
    table = rnd(g, vocab, dim, dtype=torch.bfloat16)
    ids = torch.randint(0, vocab, (77,), generator=g).to(dev)
    ids[:3] = torch.tensor([0, vocab - 1, 5], device=dev)
    got = nans(77, dim)
    nv.embedding_gather(ids, table, got)
    exact("embedding_gather", got, table[ids].float(), wrong=table[(ids + 1) % vocab].float())
    for n in (2, 1000, 1_000_002):
        a, b = rnd(g, n, scale=3, dtype=torch.bfloat16), rnd(g, n, scale=3, dtype=torch.bfloat16)
        got = nans(n, dtype=torch.bfloat16)
        nv.mul_bf16(a, b, got)
        p = a.float() * b.float()                                  # exact in fp32 (8 x 8 significant bits), then RNE
        exact(f"mul_bf16 n={n}", got, p.to(torch.bfloat16),
              wrong=(p.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16) if n > 2 else None)


def test_patchify_unpatchify():
    g = _gen(102)
    for (C0, C1, Fr, H, W, extra) in [(16, 20, 3, 8, 12, 0), (16, 0, 2, 6, 10, 8), (48, 16, 1, 30, 52, 16)]:
        x, y = rnd(g, C0, Fr, H, W), (rnd(g, C1, Fr, H, W) if C1 else None)
        L, kp = Fr * (H // 2) * (W // 2), 4 * (C0 + C1) + extra
        for split in (False, True):
            got = nans(L, kp * (2 if split else 1), dtype=torch.bfloat16)
            ref = nans(L, kp * (2 if split else 1), dtype=torch.bfloat16)
            nv.patchify_gather(x, y, got, split=split)
            E.patchify_gather(x, y, ref, split=split)
            src = x if y is None else torch.cat([x, y])
            wrong = E.patchify_gather(src.flip(3).contiguous(), None, ref.clone(), split=split)     # columns mirrored
            exact(f"patchify_gather{' split' if split else ''} C={C0}+{C1} {Fr}x{H}x{W} Kpad={kp}", got, ref, wrong=wrong)
        C = C0
        ho = rnd(g, L, 4 * C + 24)
        got, ref = nans(C, Fr, H, W), nans(C, Fr, H, W)
        nv.unpatchify(ho[:, :4 * C + 8], got)        # ldh = 4C + 24 > 4C: the extra head columns are not read
        E.unpatchify(ho[:, :4 * C], ref)
        wrong = E.unpatchify(ho[:, :4 * C], nans(C, Fr, H, W)).flip(3)     # columns mirrored
        exact(f"unpatchify C={C} {Fr}x{H}x{W}", got, ref, wrong=wrong)


def test_vae_layout():
    g = _gen(103)
    for (H, W, C) in [(4, 6, 4), (30, 52, 96), (90, 160, 12)]:
        x = rnd(g, H, W, C, scale=2)
        got, ref = nans(2 * H, 2 * W, C, dtype=torch.bfloat16), nans(2 * H, 2 * W, C, dtype=torch.bfloat16)
        nv.vae_upsample2x(x, H, W, C, got)
        E.vae_upsample2x(x, H, W, C, ref)
        exact(f"vae_upsample2x {H}x{W}x{C}", got, ref, wrong=torch.roll(ref, 1, dims=1))
        got, ref = nans(H // 2, W // 2, 4 * C, dtype=torch.bfloat16), nans(H // 2, W // 2, 4 * C, dtype=torch.bfloat16)
        nv.vae_space_to_depth(x, H, W, C, got)
        E.vae_space_to_depth(x, H, W, C, ref)
        swapped = E.vae_space_to_depth(x.transpose(0, 1).contiguous(), W, H, C, nans(W // 2, H // 2, 4 * C, dtype=torch.bfloat16))
        exact(f"vae_space_to_depth {H}x{W}x{C}", got, ref, wrong=swapped.transpose(0, 1))   # (dx, dy) phase order
        for act in (nv.ACT_NONE, nv.ACT_SILU):
            got = nans(H // 2, W // 2, 4 * C, dtype=torch.bfloat16)
            ref = nans(H // 2, W // 2, 4 * C, dtype=torch.bfloat16)
            nv.vae_space_to_depth_act(x, H, W, C, act, got)
            E.vae_space_to_depth_act(x, H, W, C, act, ref)
            if act == nv.ACT_NONE:
                exact(f"vae_space_to_depth_act none {H}x{W}x{C}", got, ref)
            else:
                wrong = E.vae_space_to_depth(F.gelu(x), H, W, C, ref.clone())
                bf16_ulp(f"vae_space_to_depth_act silu {H}x{W}x{C}", got, ref, wrong=wrong)


def test_vae_planar():
    g = _gen(104)
    for (C, n_pix, ldc, ldo) in [(3, 24 * 40, 5 * 24 * 40, 8), (16, 777, 777, 16), (16, 1001, 1001 + 37, 20)]:
        big = rnd(g, C, ldc, scale=2)
        x = big[:, :n_pix]
        for out_bf16 in (False, True):
            dt = torch.bfloat16 if out_bf16 else torch.float32
            got, ref = nans(n_pix, ldo, dtype=dt), nans(n_pix, ldo, dtype=dt)
            nv.vae_from_planar(x, C, n_pix, None, None, got, ldo, out_bf16, ldc=ldc)
            E.vae_from_planar(x, C, n_pix, None, None, ref, ldo, out_bf16, ldc=ldc)
            exact(f"vae_from_planar C={C} n={n_pix} ldc={ldc} ldo={ldo} bf16={out_bf16}", got, ref, wrong=_shift_rows(ref))
        scale, shift = rnd(g, C, scale=0.5, shift=1.0), rnd(g, C)
        got, ref = nans(n_pix, ldo), nans(n_pix, ldo)
        nv.vae_from_planar(x, C, n_pix, scale, shift, got, ldo, False, ldc=ldc)
        E.vae_from_planar(x, C, n_pix, scale, shift, ref, ldo, False, ldc=ldc)
        mag = torch.zeros(n_pix, ldo, device=dev)
        mag[:, :C] = (x.t() * scale).abs() + shift.abs()
        wrong = torch.zeros(n_pix, ldo, device=dev)
        wrong[:, :C] = (x.t() + shift) * scale                    # shift applied before the scale
        f32_ulps(f"vae_from_planar scale+shift C={C} n={n_pix}", got, ref, mag, k=2, wrong=wrong)
        got_b, ref_b = nans(n_pix, ldo, dtype=torch.bfloat16), nans(n_pix, ldo, dtype=torch.bfloat16)
        nv.vae_from_planar(x, C, n_pix, scale, shift, got_b, ldo, True, ldc=ldc)
        E.vae_from_planar(x, C, n_pix, scale, shift, ref_b, ldo, True, ldc=ldc)
        bf16_ulp(f"vae_from_planar scale+shift bf16 C={C}", got_b[:, :C], ref_b[:, :C], wrong=_shift_rows(ref_b[:, :C]))
        exact("vae_from_planar bf16 padding columns", got_b[:, C:], torch.zeros_like(got_b[:, C:]))
        # channels-last [n_pix, ldx] -> planar rows of pitch ldc, optional clamp
        ldx = C + 5
        xc = rnd(g, n_pix, ldx, scale=1.5)
        pre, sc = rnd(g, C, scale=0.3), rnd(g, C, scale=0.5, shift=1.0)
        for clamp in (False, True):
            got_p, ref_p = nans(C, ldc), nans(C, ldc)
            nv.vae_to_planar(xc, ldx, C, n_pix, pre, sc, clamp, got_p, ldc=ldc)
            E.vae_to_planar(xc, ldx, C, n_pix, pre, sc, clamp, ref_p[:, :n_pix], ldc=ldc)
            mag = ((xc[:, :C].abs() + pre.abs()) * sc.abs()).t()
            wrong = None
            if clamp:
                wrong = E.vae_to_planar(xc, ldx, C, n_pix, pre, sc, False, nans(C, n_pix))
            f32_ulps(f"vae_to_planar C={C} n={n_pix} clamp={clamp}", got_p[:, :n_pix], ref_p[:, :n_pix], mag, k=4, wrong=wrong)
            if ldc > n_pix:
                assert torch.isnan(got_p[:, n_pix:]).all(), "vae_to_planar wrote beyond n_pix inside the plane pitch"


def test_conv1d_gather():
    g = _gen(105)
    # (T_in, C, lds, col0, kernel, stride, pad_l, pad_r, T_out, split, Kpad): conv 0 (split two-term), the strided stack,
    # one group of the positional conv read in place (col0), a truncated T_out
    for (T_in, C, lds, col0, k, s, pl, pr, T_out, split, kp) in [
            (4000, 1, 1, 0, 10, 5, 0, 0, 799, True, 16), (799, 512, 512, 0, 3, 2, 0, 0, 399, False, 1536),
            (300, 48, 768, 96, 128, 1, 64, 64, 300, False, 6144), (50, 16, 24, 8, 2, 2, 0, 0, 20, False, 40)]:
        for src_dtype in (torch.float32, torch.bfloat16):
            src = rnd(g, T_in, lds, dtype=src_dtype)
            w_out = kp * (2 if split else 1)
            got = nans(T_out, w_out + 8, dtype=torch.bfloat16)     # ldo = w_out + 8: the last 8 columns stay untouched
            ref = nans(T_out, w_out, dtype=torch.bfloat16)
            nv.conv1d_gather(src, got[:, :w_out], k, s, pl, pr, col0=col0, C=C, split=split)
            EA.conv1d_gather(src, ref, k, s, pl, pr, col0=col0, C=C, split=split)
            wrong = EA.conv1d_gather(src, ref.clone(), k, s, pl + 1, max(pr - 1, 0), col0=col0, C=C, split=split) if pr else \
                EA.conv1d_gather(src, ref.clone(), k, s, 0, 0, col0=col0 + 1, C=C, split=split) if col0 + C < lds else None
            exact(f"conv1d_gather T_in={T_in} C={C} k={k} s={s} pad=({pl},{pr}) col0={col0} split={split} {src_dtype}",
                  got[:, :w_out], ref, wrong=wrong)
            assert torch.isnan(got[:, w_out:].float()).all(), "conv1d_gather wrote beyond its width"


# ------------------------------------------------------------------------------------------- fp32 math stored as bf16
def _tiny_rows(x, every=7, amp=1e-3):
    """rows whose variance is of the order of eps (1e-6), so the eps term matters"""
    x[::every] *= amp
    return x


def test_act_f32_to_bf16():
    g = _gen(110)
    n = 1000 * 1001
    x = rnd(g, n, scale=3.0)
    for act, wrong_act in [(nv.ACT_GELU_TANH, nv.ACT_GELU_ERF), (nv.ACT_SILU, nv.ACT_GELU_ERF), (nv.ACT_GELU_ERF, nv.ACT_GELU_TANH)]:
        got, ref = nans(n, dtype=torch.bfloat16), nans(n, dtype=torch.bfloat16)
        nv.cast_f32_to_bf16(x, got, act=act)
        E.cast_f32_to_bf16(x, ref, act=act)
        wrong = E._act(x, wrong_act).to(torch.bfloat16)              # the other activation id
        bf16_ulp(f"act_f32_to_bf16 act={act}", got.view(1000, -1), ref.view(1000, -1), wrong=wrong.view(1000, -1),
                 max_flip=GELU_TANH_MAX_FLIP if act == nv.ACT_GELU_TANH else 0.01)


@pytest.mark.parametrize("C,Cpad,ldx", [(4, 8, 8), (12, 64, 16), (96, 96, 100), (384, 448, 384), (1024, 1024, 1028)])
def test_vae_norm_act(C, Cpad, ldx):
    g = _gen(111 + C)
    n_pix = 777
    x = rnd(g, n_pix, ldx, scale=2.0, shift=0.3)
    gamma = rnd(g, C, scale=0.2, shift=1.0)
    for use_gamma in (False, True):
        for silu in (False, True):
            got, ref = nans(n_pix + 3, Cpad, dtype=torch.bfloat16), nans(n_pix + 3, Cpad, dtype=torch.bfloat16)
            gm = gamma if use_gamma else None
            nv.vae_norm_act(x, n_pix, C, ldx, gm, silu, got, Cpad)
            E.vae_norm_act(x, n_pix, C, ldx, gm, silu, ref, Cpad)
            name = f"vae_norm_act C={C} Cpad={Cpad} ldx={ldx} gamma={use_gamma} silu={silu}"
            if not use_gamma and not silu:
                exact(name, got[:n_pix], ref[:n_pix], wrong=_shift_rows(ref[:n_pix]))
            else:
                bf16_ulp(name, got[:n_pix, :C], ref[:n_pix, :C], wrong=_shift_rows(ref[:n_pix, :C]))
                exact(name + " padding columns", got[:n_pix, C:], torch.zeros_like(got[:n_pix, C:]))
            assert torch.isnan(got[n_pix:].float()).all(), "vae_norm_act wrote beyond n_pix"


@pytest.mark.parametrize("D", [1536, 1280, 384, 2048, 5120, 8192])     # warp<12>, warp<10>, generic warp (2), block kernel (2)
def test_layernorm_modulate(D):
    g = _gen(120 + D)
    M = 301
    x = _tiny_rows(rnd(g, M, D, scale=2.0, shift=0.3))
    gamma, beta = rnd(g, D), rnd(g, D)
    scale, shift = rnd(g, D, scale=0.1), rnd(g, D, scale=0.1)
    for kw in ({"scale": scale, "shift": shift}, {"gamma": gamma, "beta": beta}, {}, {"gamma": gamma, "beta": beta, "scale": scale, "shift": shift}):
        got, ref = nans(M, D, dtype=torch.bfloat16), nans(M, D, dtype=torch.bfloat16)
        nv.layernorm_modulate(x, got, 1e-6, **kw)
        E.layernorm_modulate(x, ref, 1e-6, **kw)
        wrong = E.layernorm_modulate(x, ref.clone(), 1e-5, **kw)
        bf16_ulp(f"layernorm_modulate D={D} {'+'.join(kw) or 'plain'}", got, ref, wrong=wrong)


def test_split_forms():
    """two-term bf16 outputs: hi + lo against the stand-in's hi + lo (v to ~2^-17 relative) and hi within one ulp"""
    g = _gen(130)

    def check(name, got, ref, K, max_flip=0.01):
        ref_sum = ref[:, :K].float() + ref[:, K:].float()
        got_sum = got[:, :K].float() + got[:, K:].float()
        rowmax = ref_sum.abs().amax(dim=1, keepdim=True)
        mag = 2.0 ** 8 * ref_sum.abs() + 16 * rowmax        # 2^-16 |v| + 16 fp32 ulps of the row scale, in units of 2^-24
        f32_ulps(name + " hi+lo", got_sum, ref_sum, mag, k=1, wrong=ref[:, :K].float())   # wrong: the lo term dropped
        bf16_ulp(name + " hi", got[:, :K], ref[:, :K], max_flip=max_flip)

    for (M, D) in [(77, 1536), (9, 5120), (33, 256), (5, 1280)]:
        x = _tiny_rows(rnd(g, M, D, scale=2.0, shift=0.3), every=4)
        sc, sh = rnd(g, D, scale=0.1), rnd(g, D, scale=0.1)
        got, ref = nans(M, 2 * D, dtype=torch.bfloat16), nans(M, 2 * D, dtype=torch.bfloat16)
        nv.layernorm_modulate_split(x, got, 1e-6, scale=sc, shift=sh)
        E.layernorm_modulate_split(x, ref, 1e-6, scale=sc, shift=sh)
        check(f"layernorm_modulate_split M={M} D={D}", got, ref, D)
    for (M, K, act) in [(5, 256, 0), (300, 1536, 2), (257, 1280, 3), (512, 96, 1)]:
        src = rnd(g, M, K + 24, scale=3.0)[:, :K]                  # lds = K + 24
        big_got = nans(M, 2 * K + 16, dtype=torch.bfloat16)
        ref = nans(M, 2 * K, dtype=torch.bfloat16)
        nv.split_f32_to_bf16x2(src, big_got[:, :2 * K], act=act)  # ldd = 2K + 16: the last 16 columns stay untouched
        E.split_f32_to_bf16x2(src, ref, act=act)
        check(f"split_f32_to_bf16x2 M={M} K={K} act={act}", big_got[:, :2 * K], ref, K,
              max_flip=GELU_TANH_MAX_FLIP if act == nv.ACT_GELU_TANH else 0.01)
        assert torch.isnan(big_got[:, 2 * K:].float()).all(), "split_f32_to_bf16x2 wrote beyond 2K"


def _rope(M, g):
    ang = torch.rand(M, 64, generator=g, dtype=torch.float64) * 6.28
    return ang.cos().float().to(dev), ang.sin().float().to(dev)


def test_rmsnorm_rope():
    g = _gen(140)
    for (M, H) in [(200, 3), (301, 12), (33, 40)]:
        D = H * 128
        t = _tiny_rows(rnd(g, M, 3 * D + 8, scale=1.5), every=5).to(torch.bfloat16)     # ld = 3D + 8
        tf = t.float()
        ss = torch.stack([(tf[:, :D] ** 2).sum(1), (tf[:, D:2 * D] ** 2).sum(1)], 1).contiguous()
        ssp = (tf[:, :2 * D].reshape(M, 2, H, 128) ** 2).sum(3).contiguous()            # per-128-column partials
        wq, wk = rnd(g, D, scale=0.2, shift=1.0), rnd(g, D, scale=0.2, shift=1.0)
        cos, sin = _rope(M + 9, g)
        for sums, tag in ((ss, "sums"), (ssp, "partials")):
            for rope in (True, False):
                a, b = t.clone(), t.clone()
                rc, rs = (cos, sin) if rope else (None, None)
                nv.rmsnorm_rope(a[:, D:2 * D], sums, 1, 1e-6, wk, rc, rs, row_offset=9)
                E.rmsnorm_rope(b[:, D:2 * D], sums, 1, 1e-6, wk, rc, rs, row_offset=9)
                wrong = E.rmsnorm_rope(t[:, D:2 * D].clone(), sums, 1, 1e-5, wk, rc, rs, row_offset=9)
                bf16_ulp(f"rmsnorm_rope M={M} D={D} {tag} rope={rope}", a[:, D:2 * D], b[:, D:2 * D], wrong=wrong)
                exact("rmsnorm_rope: the other columns stay untouched", torch.cat([a[:, :D], a[:, 2 * D:]], 1),
                      torch.cat([t[:, :D], t[:, 2 * D:]], 1))
            a, b = t.clone(), t.clone()
            nv.qk_norm_rope(a[:, :2 * D], sums, 1e-6, wq, wk, cos, sin, row_offset=9)
            E.qk_norm_rope(b[:, :2 * D], sums, 1e-6, wq, wk, cos, sin, row_offset=9)
            wrong = E.qk_norm_rope(t[:, :2 * D].clone(), sums, 1e-6, wq, wk, cos, sin, row_offset=8)   # rope row off by one
            bf16_ulp(f"qk_norm_rope M={M} D={D} {tag}", a[:, :2 * D], b[:, :2 * D], wrong=wrong)
            exact("qk_norm_rope: v columns stay untouched", a[:, 2 * D:], t[:, 2 * D:])


@pytest.mark.parametrize("rows,N,ldp", [(64, 77, 80), (300, 1024, 1032), (16, 14400, 14408)])
def test_softmax_rows(rows, N, ldp):
    g = _gen(150 + N)
    lds = N + 13
    s = rnd(g, rows, lds, scale=20.0)
    scale = 384 ** -0.5
    got, ref = nans(rows, ldp, dtype=torch.bfloat16), nans(rows, ldp, dtype=torch.bfloat16)     # ldp is the row pitch
    nv.softmax_rows(s, N, scale, got)
    E.softmax_rows(s, N, scale, ref)
    wrong = E.softmax_rows(s, N, 1.0, ref.clone())                 # the scale left out
    bf16_ulp(f"softmax_rows rows={rows} N={N} ldp={ldp}", got[:, :N], ref[:, :N], wrong=wrong[:, :N])
    exact("softmax_rows padding columns", got[:, N:], torch.zeros_like(got[:, N:]))


def test_encoder_norms():
    g = _gen(160)
    for (M, D) in [(77, 4096), (257, 1280), (5, 4)]:
        x = _tiny_rows(rnd(g, M, D, scale=2.0, shift=0.3), every=3)
        w = rnd(g, D, scale=0.2, shift=1.0)
        got = nans(M, D, dtype=torch.bfloat16)
        nv.rmsnorm_affine(x, w, 1e-6, got)
        ref = (w * x * torch.rsqrt((x * x).mean(1, keepdim=True) + 1e-6)).to(torch.bfloat16)
        wrong = (w * x * torch.rsqrt((x * x).mean(1, keepdim=True) + 1e-5)).to(torch.bfloat16)
        bf16_ulp(f"rmsnorm_affine M={M} D={D}", got, ref, wrong=wrong)
        gamma, beta = rnd(g, D), rnd(g, D)
        got32, ref32 = nans(M, D), nans(M, D)
        nv.layernorm_f32(x, gamma, beta, 1e-5, got32)
        EA.layernorm_f32(x, gamma, beta, 1e-5, ref32)
        mean = x.mean(1, keepdim=True)
        rstd = torch.rsqrt(x.var(1, unbiased=False, keepdim=True) + 1e-5)
        mag = (x.abs() + mean.abs()) * rstd * gamma.abs() + beta.abs()
        f32_ulps(f"layernorm_f32 M={M} D={D}", got32, ref32, mag, k=16,
                 wrong=EA.layernorm_f32(x, gamma, beta, 1e-6, nans(M, D)))


def test_col_stats():
    g = _gen(170)
    for (T, C, ldx) in [(799, 512, 512), (3, 8, 12), (40000, 48, 64), (1, 4, 4)]:
        x = rnd(g, T, ldx, scale=2.0, shift=0.5)[:, :C] if ldx > C else rnd(g, T, C, scale=2.0, shift=0.5)
        ws = torch.empty(nv.col_stats_workspace_bytes(T, C) // 8 + 1, device=dev, dtype=torch.float64)
        mean, var = nans(C), nans(C)
        rm, rv = nans(C), nans(C)
        nv.col_stats(x, mean, var, ws)
        EA.col_stats(x, rm, rv, ws)
        xd = x.double()
        f32_ulps(f"col_stats mean T={T} C={C}", mean, rm, xd.abs().mean(0).float(), k=2)
        wrong = (xd.var(0, unbiased=True).float() if T > 1 else None)
        f32_ulps(f"col_stats var T={T} C={C}", var, rv, (xd * xd).mean(0).float(), k=2, wrong=wrong)


def test_col_norm_act():
    g = _gen(171)
    for (T, C, ldx, ldy) in [(799, 512, 520, 520), (199, 48, 48, 64)]:
        x = rnd(g, T, ldx, scale=2.0, shift=0.5)[:, :C]
        mean, var = x.mean(0), x.var(0, unbiased=False)
        var[::5] = 1e-7 * torch.rand(len(var[::5]), generator=g).to(dev)     # columns where eps matters
        gamma, beta = rnd(g, C, scale=0.2, shift=1.0), rnd(g, C, scale=0.1)
        for act in (nv.ACT_NONE, nv.ACT_GELU_ERF, nv.ACT_GELU_TANH, nv.ACT_SILU, nv.ACT_RELU):
            for aff in (True, False):
                big = nans(T, ldy, dtype=torch.bfloat16)
                ref = nans(T, C, dtype=torch.bfloat16)
                ga, be = (gamma, beta) if aff else (None, None)
                nv.col_norm_act(x, mean, var, 1e-5, ga, be, act, big[:, :C])
                EA.col_norm_act(x, mean, var, 1e-5, ga, be, act, ref)
                wrong = EA.col_norm_act(x, mean, var, 1e-6, ga, be, act, ref.clone())
                bf16_ulp(f"col_norm_act T={T} C={C} act={act} affine={aff}", big[:, :C], ref, wrong=wrong)
                assert torch.isnan(big[:, C:].float()).all(), "col_norm_act wrote beyond C"


def test_interp_layernorm():
    g = _gen(172)
    for (T_in, T_out, C, ldx) in [(3050, 1525, 512, 520), (100, 37, 768, 768), (2, 9, 16, 16), (1, 4, 8, 8)]:
        x = rnd(g, T_in, ldx, scale=2.0, shift=0.3)
        x[::3] *= 1e-3                                             # rows (and, at the endpoints, outputs) where eps matters
        x = x[:, :C]
        gamma, beta = rnd(g, C), rnd(g, C, scale=0.1)
        big = nans(T_out, C + 8, dtype=torch.bfloat16)
        ref = nans(T_out, C, dtype=torch.bfloat16)
        nv.interp_layernorm(x, T_out, gamma, beta, 1e-5, big[:, :C])
        EA.interp_layernorm(x.contiguous(), T_out, gamma, beta, 1e-5, ref)
        wrong = EA.interp_layernorm(x.contiguous(), T_out, gamma, beta, 1e-4, ref.clone())
        bf16_ulp(f"interp_layernorm T_in={T_in} T_out={T_out} C={C}", big[:, :C], ref, wrong=wrong)
        assert torch.isnan(big[:, C:].float()).all(), "interp_layernorm wrote beyond C"


# ------------------------------------------------------------------------------------------------ fp32 arithmetic
def test_f32_arithmetic():
    g = _gen(180)
    n = 4 * 250_001
    a, b = rnd(g, n, scale=3.0), rnd(g, n, scale=3.0)
    for alpha, beta in [(1.0, -1.0), (0.7, 1.3), (-2.5, 0.0)]:
        got, ref = nans(n), nans(n)
        nv.axpby(a, alpha, b, beta, got)
        E.axpby(a, alpha, b, beta, ref)
        # measured on an H100 80GB HBM3 (400 W): the error reaches 2 fp32 ulps of the terms exactly (FMA contraction), bar 4
        mag = (alpha * a).abs() + (beta * b).abs()
        f32_ulps(f"axpby alpha={alpha} beta={beta}", got, ref, mag, k=4,
                 wrong=E.axpby(a, beta, b, alpha, nans(n)) if alpha != beta else None)
        al = a.clone()                                             # out aliases a
        nv.axpby(al, alpha, b, beta, al)
        f32_ulps(f"axpby aliased out alpha={alpha} beta={beta}", al, ref, mag, k=4)
    lat, vc, vu = rnd(g, 1000, 7), rnd(g, 1000, 7), rnd(g, 1000, 7)
    for cfg, v_u in [(5.0, vu), (1.0, None)]:
        got, ref = lat.clone(), lat.clone()
        nv.cfg_euler_step(got, vc, v_u, cfg, 0.9, 0.8)
        E.cfg_euler_step(ref, vc, v_u, cfg, 0.9, 0.8)
        vmag = vc.abs() if v_u is None else v_u.abs() + cfg * (vc.abs() + v_u.abs())
        mag = lat.abs() + 4 * 0.1 * vmag
        wrong = E.cfg_euler_step(lat.clone(), vc, v_u, cfg, 0.8, 0.9)    # sigma order swapped
        f32_ulps(f"cfg_euler_step cfg={cfg}", got, ref, mag, k=4, wrong=wrong)


def test_ln_fold_vectors():
    g = _gen(181)
    layers, D = 3, 1536
    mods = rnd(g, 6 * layers + 2, D, scale=0.2)
    gg, rows = nans(layers, 2, D), nans(layers, 2, 4, D, dtype=torch.bfloat16)
    rg, rr = nans(layers, 2, D), nans(layers, 2, 4, D, dtype=torch.bfloat16)
    nv.ln_fold_prepare(mods, layers, gg, rows)
    E.ln_fold_prepare(mods, layers, rg, rr)
    m = mods[:6 * layers].reshape(layers, 2, 3, D)
    f32_ulps("ln_fold_prepare g = 1 + scale", gg, rg, 1 + m[:, :, 1].abs(), k=1, wrong=m[:, :, 1])
    exact("ln_fold_prepare rows (g_hi, g_lo, t_hi, t_lo)", rows, rr, wrong=rr.flip(2))
    N = 4608
    o4, bias = rnd(g, 4, N, scale=3.0), rnd(g, N)
    u, c, ru, rc = nans(N), nans(N), nans(N), nans(N)
    nv.ln_fold_combine(o4, bias, u, c)
    E.ln_fold_combine(o4, bias, ru, rc)
    f32_ulps("ln_fold_combine u", u, ru, o4[0].abs() + o4[1].abs(), k=1)
    f32_ulps("ln_fold_combine c", c, rc, o4[2].abs() + o4[3].abs() + bias.abs(), k=2, wrong=o4[2] + o4[3])
    nv.ln_fold_combine(o4, None, u, c)
    E.ln_fold_combine(o4, None, ru, rc)
    f32_ulps("ln_fold_combine c without bias", c, rc, o4[2].abs() + o4[3].abs(), k=1)


# ----------------------------------------------------------------------------------- tolerance yardsticks (GEMM, attention)
def test_gemm_matches_standin():
    """the stand-in accumulates in fp64; the sharp per-element bound is gpu_check.sec_gemm_edges"""
    g = _gen(190)
    for (M, N, K) in [(300, 1536, 512), (1, 264, 72), (777, 4608, 1536)]:
        a, w = rnd(g, M, K, scale=0.5, dtype=torch.bfloat16), rnd(g, N, K, scale=0.1, dtype=torch.bfloat16)
        bias, gate, res = rnd(g, N), rnd(g, N), rnd(g, M, N)
        for kw, dt in [({}, torch.float32), ({"bias": bias, "act": nv.ACT_GELU_TANH}, torch.bfloat16),
                       ({"bias": bias, "act": nv.ACT_RELU}, torch.bfloat16), ({"bias": bias, "gate": gate, "residual": res}, torch.float32)]:
            got, ref = nans(M, N, dtype=dt), nans(M, N, dtype=dt)
            nv.gemm(a, w, got, **kw)
            E.gemm(a, w, ref, **kw)
            tol_bar(f"gemm M={M} N={N} K={K} {'+'.join(kw) or 'plain'} {dt}", got, ref, 2e-3 if dt == torch.float32 else 1e-2)


def test_attention_matches_standin():
    g = _gen(191)
    for (Lq, Lk, H) in [(300, 333, 2), (1000, 77, 3)]:
        q, k, v = (rnd(g, L, H * 128, dtype=torch.bfloat16) for L in (Lq, Lk, Lk))
        got, ref = nans(Lq, H * 128, dtype=torch.bfloat16), nans(Lq, H * 128, dtype=torch.bfloat16)
        nv.attention(q, k, v, got, H)
        E.attention(q, k, v, ref, H)
        tol_bar(f"attention Lq={Lq} Lk={Lk} H={H}", got, ref, 2e-2)
        ss = (q.float() ** 2).sum(1, keepdim=True).contiguous()
        nv.attention_qscale(q, k, v, got, H, ss, H * 128, 1e-6)
        E.attention_qscale(q, k, v, ref, H, ss, H * 128, 1e-6)
        tol_bar(f"attention_qscale Lq={Lq} Lk={Lk} H={H}", got, ref, 2e-2)


def test_attention_small_matches_standin():
    """svi_attn_small is fp32 throughout, like its stand-in: the outputs agree to one bf16 rounding"""
    g = _gen(192)
    for (L, H, hd) in [(77, 3, 80), (512, 12, 64), (33, 2, 128)]:
        q, k, v = (rnd(g, L, H * hd + 16, dtype=torch.bfloat16)[:, :H * hd] for _ in range(3))
        scale = hd ** -0.5
        big = nans(L, H * hd + 8, dtype=torch.bfloat16)
        ref = nans(L, H * hd, dtype=torch.bfloat16)
        nv.attention_small(q, k, v, big[:, :H * hd], H, hd, scale)
        EA.attention_small(q, k, v, ref, H, hd, scale)
        wrong = EA.attention_small(q, k, v, ref.clone(), H, hd, scale * 1.05)
        bf16_ulp(f"attention_small L={L} H={H} hd={hd}", big[:, :H * hd], ref, wrong=wrong, floor_ulps=256)
        assert torch.isnan(big[:, H * hd:].float()).all(), "attention_small wrote beyond its width"
        for mask in ((torch.rand(L, generator=g) > 0.3).to(torch.int32).to(dev), torch.zeros(L, dtype=torch.int32, device=dev)):
            got, ref = nans(L, H * hd, dtype=torch.bfloat16), nans(L, H * hd, dtype=torch.bfloat16)
            nv.attention_small(q, k, v, got, H, hd, scale, key_mask=mask)
            EA.attention_small(q, k, v, ref, H, hd, scale, key_mask=mask)
            if mask.any():
                bf16_ulp(f"attention_small L={L} key mask", got, ref, wrong=EA.attention_small(q, k, v, ref.clone(), H, hd, scale),
                         floor_ulps=256)
            else:
                exact(f"attention_small L={L} every key masked -> 0", got, torch.zeros_like(got))
