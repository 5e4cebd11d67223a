"""GPU: FastBlend deflickering on the sm_90a kernels (include/svi_b200_fastblend.h).

Each entry point against the oracle's restatement (oracle/fastblend_oracle.py through the stand-ins of
tests/nv_emulation_fastblend.py, run on the same device) bit for bit; the remap and patch error against the reference's
own kernels (compiled by build() into oracle/_ref/libfastblend_ref.so); a full-size estimate_nnf and a 17-frame
smoother run at 832x480 against the oracle, byte for byte."""
import ctypes
import os

import numpy as np
import pytest
import torch

import nv_emulation_fastblend as emu
from oracle import fastblend_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libfastblend_ref.so")
DEV = "cuda:0"

COVERED = {
    "svi_fastblend_stage_frames": ["test_stage_frames_exact"],
    "svi_fastblend_downsample": ["test_downsample_matches_oracle"],
    "svi_fastblend_nnf_identity": ["test_nnf_identity_and_upscale_match_oracle"],
    "svi_fastblend_nnf_upscale": ["test_nnf_identity_and_upscale_match_oracle"],
    "svi_fastblend_remap": ["test_remap_matches_oracle_and_reference_kernel"],
    "svi_fastblend_step": ["test_step_matches_oracle", "test_patch_error_within_reference_contraction"],
    "svi_fastblend_table": ["test_table_ops_match_oracle"],
}


@pytest.fixture(scope="module")
def nv():
    from diffsynth import _native
    _native.load()
    return _native


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF_LIB):
        pytest.skip("oracle/_ref/libfastblend_ref.so was not built (build() makes it where the reference tree exists)")
    lib = ctypes.CDLL(REF_LIB)
    i, p = ctypes.c_int, ctypes.c_void_p
    lib.ref_remap.argtypes = [i] * 6 + [p] * 4
    lib.ref_patch_error.argtypes = [i] * 6 + [p] * 5
    return lib


def bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int64) \
        if t.dtype == torch.float64 else t


def same(a, b):
    return torch.equal(bits(a), bits(b))


def frames4(B, H, W, seed, scale=255.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(B, H, W, 4)
    x[..., :3] = torch.rand(B, H, W, 3, generator=g) * scale
    return x.to(DEV)


def random_nnf(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, H, (B, H, W), generator=g), torch.randint(0, W, (B, H, W), generator=g)],
                       -1).to(torch.int32).to(DEV)


def test_stage_frames_exact(nv):
    rgb = torch.randint(0, 256, (3, 37, 53, 3), dtype=torch.uint8, device=DEV)
    out = nv.fastblend_stage_frames(rgb, torch.full((3, 37, 53, 4), 7.0, device=DEV))
    assert same(out, emu.fastblend_stage_frames(rgb, torch.empty_like(out)))


@pytest.mark.parametrize("k", [2, 4, 8, 16])
def test_downsample_matches_oracle(nv, k):
    x = frames4(2, 480, 832, seed=k)
    out = nv.fastblend_downsample(x, k, torch.full((2, 480 // k, 832 // k, 4), 7.0, device=DEV))
    assert same(out, emu.fastblend_downsample(x, k, torch.empty_like(out)))


@pytest.mark.parametrize("B", [8, 3, 1])
def test_nnf_identity_and_upscale_match_oracle(nv, B):
    nnf = nv.fastblend_nnf_identity(torch.full((B, 30, 52, 2), -5, dtype=torch.int32, device=DEV))
    assert same(nnf, O.identity_nnf(B, 30, 52, DEV))
    src = random_nnf(B, 30, 52, seed=B)
    out = nv.fastblend_nnf_upscale(src, torch.full((B, 60, 104, 2), -5, dtype=torch.int32, device=DEV))
    assert same(out, O.upscale_nnf(src, 60, 104))


@pytest.mark.parametrize("patch", [13, 5, 1])
def test_remap_matches_oracle_and_reference_kernel(nv, ref, patch):
    B, H, W = 4, 60, 104
    style, nnf = frames4(B, H, W, seed=patch), random_nnf(B, H, W, seed=patch)
    out = nv.fastblend_remap(style, nnf, patch, torch.full_like(style, 7.0))
    assert same(out, emu.fastblend_remap(style, nnf, patch, torch.empty_like(style)))
    pad = 6
    src = torch.nn.functional.pad(style[..., :3], (0, 0, pad, pad, pad, pad)).contiguous()
    tgt = torch.zeros_like(src)
    assert ref.ref_remap(B, H, W, 3, patch, pad, src.data_ptr(), nnf.data_ptr(), tgt.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert same(out[..., :3], tgt[:, pad:-pad, pad:-pad])


def _step_inputs(B, H, W, seed):
    sg, ss, tg = frames4(B, H, W, seed), frames4(B, H, W, seed + 1), frames4(B, H, W, seed + 2)
    nnf = random_nnf(B, H, W, seed)
    ts = emu.fastblend_remap(ss, nnf, 13, torch.empty_like(ss))
    err = torch.rand(B, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV) * 4e7
    return sg, ss, tg, ts, nnf, err


@pytest.mark.parametrize("patch", [13, 7, 5])
@pytest.mark.parametrize("mode,dir", [(0, 0), (1, 0), (1, 1), (1, 2), (1, 3), (2, 0)])
def test_step_matches_oracle(nv, patch, mode, dir):
    B, H, W = 3, 45, 80
    sg, ss, tg, ts, nnf, err = _step_inputs(B, H, W, seed=patch)
    kw = dict(dir=dir, draw=12345, radius=4)
    want_n, want_e = torch.empty_like(nnf), torch.empty_like(err)
    emu.fastblend_step(sg, ss, tg, ts, nnf, None if mode == 0 else err, want_n, want_e, patch, mode, 10.0, **kw)
    got_n, got_e = torch.full_like(nnf, -1), torch.full_like(err, -1.0)
    nv.fastblend_step(sg, ss, tg, ts, nnf, None if mode == 0 else err, got_n, got_e, patch, mode, 10.0, **kw)
    assert same(got_n, want_n) and same(got_e, want_e)
    if mode:
        assert 0 < (got_n != nnf).any(-1).float().mean() < 1       # the select kept some entries and replaced others


@pytest.mark.parametrize("patch", [13, 5])
def test_patch_error_within_reference_contraction(nv, ref, patch):
    """guide_weight 0 leaves the style error alone; the reference's compiler contracts e += d * d into FMAs, so the two
    agree within taps * 3 * 2^-24 relative"""
    B, H, W = 3, 45, 80
    sg, ss, tg, ts, nnf, _ = _step_inputs(B, H, W, seed=patch)
    got_n, got_e = torch.empty_like(nnf), torch.empty(B, H, W, device=DEV)
    nv.fastblend_step(sg, ss, tg, ts, nnf, None, got_n, got_e, patch, 0, 0.0)
    pad = 6
    padf = lambda t: torch.nn.functional.pad(t[..., :3], (0, 0, pad, pad, pad, pad)).contiguous()
    src, tgt = padf(ss), padf(ts)
    err = torch.zeros(B, H, W, device=DEV)
    assert ref.ref_patch_error(B, H, W, 3, patch, pad, src.data_ptr(), nnf.data_ptr(), tgt.data_ptr(), err.data_ptr(),
                               None) == 0
    torch.cuda.synchronize()
    rel = ((got_e.double() - err.double()).abs() / err.double().clamp_min(1e-30)).max().item()
    bound = patch * patch * 3 * 2.0 ** -24
    print(f"patch {patch}: max relative difference to the reference kernel {rel:.3e} (bound {bound:.3e})")
    assert rel <= bound


def test_table_ops_match_oracle(nv):
    H, W = 48, 80
    g = torch.Generator().manual_seed(0)
    u8 = torch.randint(0, 256, (H, W, 4), generator=g).float()
    u8[..., 3] = 0
    f1, f2 = frames4(1, H, W, 1)[0], frames4(1, H, W, 2)[0]
    f64 = (frames4(1, H, W, 3)[0].double() * 1.000000001)
    u8 = u8.to(DEV)
    cases = [
        (0, torch.float32, dict(a=f1, sa=2 / 3, b=f2, sb=3)),
        (1, torch.float32, dict(a=u8, b=f2, a_u8=True)),
        (1, torch.float32, dict(a=f1, b=f2)),
        (2, torch.float32, dict(a=f1, sa=5 / 7, b=f2, sb=2 / 7)),
        (2, torch.float64, dict(a=u8, sa=1 / 3, b=f2, sb=2 / 3, a_u8=True)),
        (2, torch.float64, dict(a=f64, sa=3 / 11, b=f2, sb=8 / 11)),
        (2, torch.uint8, dict(a=f64, sa=7 / 9, b=u8, sb=-1 / 9, c=f1, sc=3 / 9, b_u8=True)),
        (2, torch.uint8, dict(a=f1, sa=1.0, b=u8, sb=-1.0, c=u8, sc=1.0, b_u8=True, c_u8=True)),
        (2, torch.uint8, dict(a=f1, sa=3.5, b=u8, sb=-1.0, c=f2, sc=-2.0, b_u8=True)),   # clipped both ways
    ]
    for op, dtype, kw in cases:
        shape = (H, W, 3) if dtype == torch.uint8 else (H, W, 4)
        got = nv.fastblend_table(op, torch.full(shape, 7, dtype=dtype, device=DEV), **kw)
        want = emu.fastblend_table(op, torch.empty(shape, dtype=dtype, device=DEV), **kw)
        assert same(got, want), (op, dtype)


# ------------------------------------------------------------------------------------------- full size
def _video(n, H, W, seed):
    from tools.synth_fastblend import make_frames
    return make_frames(n, H, W, seed)


@pytest.mark.slow
def test_estimate_nnf_832x480_matches_oracle(nv):
    from diffsynth.extensions.FastBlend import PyramidPatchMatcher
    f = _video(9, 480, 832, seed=5)
    sg, tg = f[:8], f[1:]
    m = PyramidPatchMatcher(480, 832, 3, 5)
    nnf, ts = m.estimate_nnf(sg, tg, sg)
    o = O.PyramidPatchMatcher(480, 832)
    t = lambda x: torch.from_numpy(x.astype(np.float32)).to(DEV)
    want_n, want_ts = o.estimate_nnf(t(sg), t(tg), t(sg))
    assert np.array_equal(nnf, want_n.cpu().numpy())
    assert np.array_equal(ts.view(np.uint32), want_ts.cpu().numpy().view(np.uint32))
    ident = np.stack(np.meshgrid(np.arange(480), np.arange(832), indexing="ij"), -1)
    print(f"estimate_nnf 832x480 x8: {(nnf != ident).any(-1).mean():.3f} of the pixels moved off the identity")


@pytest.mark.slow
def test_smoother_832x480_matches_oracle_bytes(nv):
    from PIL import Image
    from diffsynth.extensions.FastBlend import FastBlendSmoother
    f = _video(17, 480, 832, seed=7)
    frames = [Image.fromarray(x) for x in f]
    s = FastBlendSmoother()
    a = np.stack([np.asarray(x) for x in s(frames)])
    b = np.stack([np.asarray(x) for x in s(frames)])
    c = np.stack([np.asarray(x) for x in s(frames, original_frames=list(frames))])
    assert np.array_equal(a, b) and np.array_equal(a, c)
    want = O.run(list(f), list(f), batch_size=8, window_size=64, device=DEV)
    assert np.array_equal(a, want), f"{int((a != want).sum())} bytes differ"
    print(f"smoother 17 x 832x480: mean |out - in| {np.abs(a.astype(int) - f.astype(int)).mean():.3f} grey levels")
