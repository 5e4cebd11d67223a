"""GPU: RIFE entry points against their torch stand-ins on the same bf16-rounded operands, argument checks, the whole
IFNet and RIFEInterpolater against the fp32 oracle at SVI frame sizes, and reproducibility across batch sizes and runs."""
import ctypes

import numpy as np
import pytest
import torch

import nv_emulation_rife as emu
from oracle import rife_oracle as O
from tools import synth_rife as S

pytestmark = pytest.mark.gpu

COVERED = {
    "svi_rife_stage_frames": ["test_stage_frames_exact"],
    "svi_rife_block_input_launch": ["test_block_input_matches_torch"],
    "svi_rife_conv2d": ["test_conv2d_matches_torch", "test_abi_validation_returns_status"],
    "svi_rife_update_warp": ["test_update_warp_matches_torch"],
}

DEV = "cuda"


def _bf(t):
    return t.to(torch.bfloat16).float()


@pytest.fixture(scope="module")
def sd():
    return S.make_state_dict(seed=0)


@pytest.fixture(scope="module")
def model(sd):
    from diffsynth.extensions.RIFE import IFNet
    m = IFNet().eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def test_stage_frames_exact():
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(0)
    rgb = torch.randint(0, 256, (3, 17, 29, 3), generator=g, dtype=torch.uint8)
    out = torch.empty(3, 17, 29, 4, device=DEV)
    nv.rife_stage_frames(rgb.to(DEV), out)
    ref = torch.empty(3, 17, 29, 4)
    emu.rife_stage_frames(rgb, ref)
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("first,s", [(True, 4.0), (False, 2.0), (False, 1.0), (False, 8.0), (False, 0.5)])
def test_block_input_matches_torch(first, s):
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(1)
    P, H, W = 3, 64, 96
    frames = torch.rand(P + 1, H, W, 4, generator=g)
    state = None if first else torch.randn(P, H, W, 12, generator=g) * 3
    h, w = int(H / s), int(W / s)
    out = torch.empty(2 * P, h // 2, w // 2, 48, dtype=torch.bfloat16, device=DEV)
    fd = frames.to(DEV)
    nv.rife_block_input(fd[:-1], fd[1:], None if first else state.to(DEV), h, w, np.float32(s), np.float32(1 / s), out)
    ref = torch.empty(2 * P, h // 2, w // 2, 48, dtype=torch.bfloat16)
    emu.rife_block_input(frames[:-1], frames[1:], state, h, w, np.float32(s), np.float32(1 / s), ref)
    torch.testing.assert_close(out.cpu().float(), ref.float(), atol=1e-6, rtol=2 ** -7)


# (name, C_in, kh, C_out, phase_cols, prelu, residual, f32 out, bf16 out, s2d, H, W)
CONV_CASES = [
    ("conv0a_s2d", 48, 2, 46, 46, True, False, False, True, True, 24, 40),
    ("conv0b", 184, 2, 90, 90, True, False, True, True, False, 12, 20),
    ("convblock_residual", 96, 3, 90, 90, True, True, True, True, False, 37, 45),
    ("head1_subpixel", 96, 3, 360, 90, True, False, False, True, False, 12, 20),
    ("head2_subpixel", 96, 3, 24, 6, False, False, True, False, False, 24, 40),
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv2d_matches_torch(case):
    from diffsynth import _native as nv
    from diffsynth.extensions.RIFE import _pick_tile_w
    name, C_in, k, C_out, cols, use_prelu, use_res, use_out, use_bf, s2d, H, W = case
    g = torch.Generator().manual_seed(2)
    N = 3
    cpad = (C_in + 63) // 64 * 64
    x = _bf(torch.randn(N, H, W, C_in, generator=g)).to(torch.bfloat16)
    wp = _bf(torch.randn(C_out, k * k * cpad, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(C_out, generator=g)
    prelu = torch.rand(C_out, generator=g) if use_prelu else None
    up = 2 if C_out == 4 * cols else 1
    Hd, Wd = H * up, W * up
    ld = cols + (cols % 4 and 2)
    res = torch.randn(N, Hd, Wd, ld, generator=g) if use_res else None
    bfs = (N, Hd // 2, Wd // 2, 4 * cols) if s2d else (N, Hd, Wd, cols + 6)
    outs = {}
    for dev in ("cpu", DEV):
        t = lambda v: None if v is None else v.to(dev)
        out = torch.zeros(N, Hd, Wd, ld, device=dev) if use_out else None
        obf = torch.zeros(bfs, dtype=torch.bfloat16, device=dev) if use_bf else None
        r = t(res.clone()) if use_res else None
        fn = emu.rife_conv2d if dev == "cpu" else nv.rife_conv2d
        fn(t(x), t(wp), k, k, 1, C_out, cols, t(bias), _pick_tile_w(H, W), prelu=t(prelu), residual=r, out=out,
           out_bf16=obf, bf_s2d=s2d)
        outs[dev] = (out, obf)
    if use_out:
        torch.testing.assert_close(outs[DEV][0].cpu(), outs["cpu"][0], atol=2e-4, rtol=1e-4)
    if use_bf:
        torch.testing.assert_close(outs[DEV][1].cpu().float(), outs["cpu"][1].float(), atol=1e-3, rtol=2 ** -7)


@pytest.mark.parametrize("first,s,merged,rgb", [(True, 4.0, False, False), (False, 1.0, True, True), (False, 2.0, True, False),
                                                (False, 0.5, False, True)])
def test_update_warp_matches_torch(first, s, merged, rgb):
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(3)
    P, H, W = 2, 48, 80
    h, w = int(H / s), int(W / s)
    frames = torch.rand(P + 1, H, W, 4, generator=g)
    heads = torch.randn(2 * P, h, w, 8, generator=g) * 2
    state = torch.randn(P, H, W, 12, generator=g) * 2
    res = {}
    for dev in ("cpu", DEV):
        fr, st = frames.to(dev), state.clone().to(dev)
        m = torch.zeros(2 * P, H, W, 4, device=dev)[::2] if merged else None
        u = torch.zeros(P, H, W, 3, dtype=torch.uint8, device=dev) if rgb else None
        fn = emu.rife_update_warp if dev == "cpu" else nv.rife_update_warp
        fn(heads.to(dev), np.float32(1 / s), s, fr[:-1], fr[1:], st, first, merged=m, clip=True, rgb=u)
        res[dev] = (st.cpu(), None if m is None else m.cpu(), None if u is None else u.cpu())
    torch.testing.assert_close(res[DEV][0], res["cpu"][0], atol=1e-4, rtol=1e-4)
    if merged:
        torch.testing.assert_close(res[DEV][1], res["cpu"][1], atol=1e-5, rtol=1e-5)
    if rgb:
        assert (res[DEV][2].int() - res["cpu"][2].int()).abs().max() <= 1


def test_abi_validation_returns_status():
    from diffsynth import _native as nv
    lib = nv.load()
    x = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device=DEV)
    wp = torch.zeros(32, 9 * 64, dtype=torch.bfloat16, device=DEV)
    b = torch.zeros(32, device=DEV)
    out = torch.zeros(1, 8, 8, 32, device=DEV)
    d = nv.RifeConvDesc()
    d.x, d.N, d.in_H, d.in_W, d.C_in = x.data_ptr(), 1, 8, 8, 64
    d.w_packed, d.w_rows, d.w_ld = wp.data_ptr(), 32, 9 * 64
    d.kh = d.kw = 3
    d.pad_h = d.pad_w = 1
    d.H = d.W = 8
    d.C_out, d.phase_cols, d.tile_w = 32, 32, 8
    d.bias, d.out, d.out_img_stride, d.out_ld = b.data_ptr(), out.data_ptr(), out[0].numel(), 32
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.svi_rife_conv2d(ctypes.byref(d), stream) == 0
    torch.cuda.synchronize()
    for field, bad, msg in (("phase_cols", 7, "phase_cols"), ("C_out", 96, "phases"), ("C_in", 60, "C_in"),
                            ("tile_w", 12, "tile_w"), ("kh", 4, "extents"), ("w_ld", 100, "packed weight")):
        old = getattr(d, field)
        setattr(d, field, bad)
        rc = lib.svi_rife_conv2d(ctypes.byref(d), stream)
        setattr(d, field, old)
        assert rc < 0, field
        assert msg in lib.svi_last_error().decode(), (field, lib.svi_last_error())
    bi = nv.RifeBlockInput()
    assert lib.svi_rife_block_input_launch(ctypes.byref(bi), stream) < 0
    up = nv.RifeUpdate()
    assert lib.svi_rife_update_warp(ctypes.byref(up), stream) < 0
    assert lib.svi_rife_stage_frames(None, 4, None, stream) < 0


@pytest.mark.parametrize("H,W,scale", [(480, 832, 1.0), (480, 832, 0.5), (720, 1280, 1.0)])
def test_ifnet_matches_oracle(model, sd, H, W, scale):
    fr = S.make_frames(3, H, W, seed=1)
    x = torch.cat([O.to_tensor(fr[:-1]), O.to_tensor(fr[1:])], 1)
    sl = [4 / scale, 2 / scale, 1 / scale]
    flows, mask, merged = model(x.to(DEV), sl)
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        rf, rm, rmg = O.ifnet({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV), sl)
    err = (flows[2] - rf[2]).abs().mean().item() / rf[2].std().item()
    print(f"IFNet {W}x{H} scale {scale}: final flow mean|d| / std = {err:.4%}, merged mean|d| "
          f"{(merged[2] - rmg[2]).abs().mean().item():.2e}")
    assert err <= 0.01
    # the bf16 rounding study (DESIGN) predicts sigmoid(mask) mean |d| of 0.007-0.010 at these sizes
    assert (mask - rm).abs().mean().item() < 2e-2


def test_interpolate_17_frames_matches_oracle(model, sd):
    from diffsynth.extensions.RIFE import RIFEInterpolater
    frames = S.make_frames(17, 480, 832, seed=2)
    got = np.stack([np.asarray(f) for f in RIFEInterpolater(model, device=DEV).interpolate(frames, batch_size=4)])
    torch.backends.cudnn.allow_tf32 = False
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    x = O.to_tensor(np.stack([np.asarray(f) for f in frames])).to(DEV)
    with torch.no_grad():
        mid = torch.cat([O.ifnet(sdd, torch.cat((x[b:b + 4], x[b + 1:b + 5]), 1))[2][2] for b in range(0, 16, 4)])
    ref = np.empty_like(got)
    ref[0::2] = np.stack([np.asarray(f) for f in frames])
    ref[1::2] = O.to_uint8(mid.clip(0, 1).cpu())
    d = np.abs(got.astype(int) - ref.astype(int))
    print(f"interpolate 17 frames 832x480: mean|d| {d.mean():.3f} grey levels, within 2: {(d <= 2).mean():.4%}")
    assert got.shape == (33, 480, 832, 3)
    assert d.mean() <= 0.5 and (d <= 2).mean() >= 0.99


def test_bit_identical_across_batch_sizes_and_runs(model):
    from diffsynth.extensions.RIFE import RIFEInterpolater
    frames = S.make_frames(6, 480, 832, seed=3)
    r = RIFEInterpolater(model, device=DEV)
    a = np.stack([np.asarray(f) for f in r.interpolate(frames, batch_size=1)])
    b = np.stack([np.asarray(f) for f in r.interpolate(frames, batch_size=4)])
    c = np.stack([np.asarray(f) for f in r.interpolate(frames, batch_size=4)])
    assert np.array_equal(a, b) and np.array_equal(b, c)
    x = torch.cat([O.to_tensor(frames[:-1]), O.to_tensor(frames[1:])], 1).to(DEV)
    f1 = model(x)[0][2]
    f2 = model(x)[0][2]
    assert torch.equal(f1, f2)
