"""GPU: ESRGAN entry points against their torch stand-ins on the same bf16 operands, argument checks, the whole 23-block
RRDBNet and ESRGAN.upscale against the fp32 oracle, and reproducibility across batch sizes and runs."""
import ctypes

import numpy as np
import pytest
import torch

import nv_emulation_esrgan as emu
from oracle import esrgan_oracle as O
from tools import synth_esrgan as S
from tools.synth_rife import make_frames

pytestmark = pytest.mark.gpu

COVERED = {
    "svi_esrgan_stage_frames": ["test_stage_frames_exact"],
    "svi_esrgan_conv2d": ["test_conv2d_matches_torch", "test_conv2d_every_tile_width", "test_abi_validation_returns_status"],
}

DEV = "cuda"


def _bf(t):
    return t.to(torch.bfloat16).float()


@pytest.fixture(scope="module")
def sd():
    return S.make_state_dict(23, seed=0)


@pytest.fixture(scope="module")
def model(sd):
    from diffsynth.extensions.ESRGAN import RRDBNet
    m = RRDBNet().eval()
    m.load_state_dict(sd)
    return m.to(DEV)


def test_stage_frames_exact():
    from diffsynth import _native as nv
    g = torch.Generator().manual_seed(0)
    rgb = torch.randint(0, 256, (3, 17, 29, 3), generator=g, dtype=torch.uint8)
    out = torch.full((3, 17, 29, 8), 7.0, dtype=torch.bfloat16, device=DEV)
    nv.esrgan_stage_frames(rgb.to(DEV), out)
    ref = torch.empty(3, 17, 29, 8, dtype=torch.bfloat16)
    emu.esrgan_stage_frames(rgb, ref)
    assert torch.equal(out.cpu(), ref)


# (name, C_in, in_ld, C_out, slope, residual, residual2, f32 out, bf16 dest, H, W)
#   bf16 dest: None, "same" (the input buffer just past the read window), "other" (channels [0, C_out) of a 192-channel
#   buffer), "up2" (nearest x2 into [N, 2H, 2W, C_out]), "u8" (uint8 RGB, no bf16)
CONV_CASES = [
    ("conv_first", 8, 8, 64, 0.0, False, False, True, "other", 23, 37),
    ("growth_channel_offset", 96, 192, 32, 0.2, False, False, False, "same", 37, 45),
    ("conv5_rdb", 192, 192, 64, 0.0, True, False, True, "other", 29, 19),
    ("conv5_two_residuals", 192, 192, 64, 0.0, True, True, True, "other", 29, 19),
    ("conv_body_up2", 64, 192, 64, 0.0, True, False, False, "up2", 21, 33),
    ("conv_up_lrelu_up2", 64, 64, 64, 0.2, False, False, False, "up2", 42, 66),
    ("conv_last_u8", 64, 64, 4, 0.0, False, False, True, "u8", 84, 132),
]


def _run_case(case, tile_w, seed=2):
    from diffsynth import _native as nv
    from diffsynth.extensions.ESRGAN import _pick_tile_w
    name, C_in, in_ld, C_out, slope, use_res, use_res2, use_out, dest, H, W = case
    g = torch.Generator().manual_seed(seed)
    N = 3
    cpad = (C_in + 63) // 64 * 64
    buf = torch.randn(N, H, W, in_ld, generator=g).to(torch.bfloat16)
    wp = (torch.randn(C_out + 3, 9 * cpad, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(C_out, generator=g)
    if dest == "u8":
        wp, bias = wp * 0.1, bias * 0.2 + 0.5                              # values around [0, 1], some clipped
    res = torch.randn(N, H, W, C_out, generator=g) if use_res else None
    res2 = torch.randn(N, H, W, C_out, generator=g) if use_res2 else None
    outs = {}
    for dev in ("cpu", DEV):
        t = lambda v: None if v is None else v.clone().to(dev)
        b = t(buf)
        r, r2 = t(res), t(res2)
        out = (r2 if use_res2 else torch.zeros(N, H, W, C_out, device=dev)) if use_out else None
        other = torch.zeros(N, H, W, 192, dtype=torch.bfloat16, device=dev)
        up = torch.zeros(N, 2 * H, 2 * W, C_out, dtype=torch.bfloat16, device=dev)
        u8 = torch.zeros(N, H, W, 3, dtype=torch.uint8, device=dev) if dest == "u8" else None
        obf = {"same": b[..., C_in:C_in + C_out], "other": other[..., :C_out], "up2": up}.get(dest)
        fn = emu.esrgan_conv2d if dev == "cpu" else nv.esrgan_conv2d
        fn(b[..., :C_in], t(wp), C_out, t(bias), tile_w or _pick_tile_w(H, W), slope=slope, residual=r, res_scale=0.2,
           residual2=r2, res2_scale=0.2, out=out, out_bf16=obf, bf_up2=dest == "up2", out_u8=u8)
        outs[dev] = [None if v is None else v.cpu() for v in (out, b, other, up, u8)]
    cpu, gpu = outs["cpu"], outs[DEV]
    if use_out:
        torch.testing.assert_close(gpu[0], cpu[0], atol=2e-4, rtol=1e-4)
    for i in (1, 2, 3):                                 # the whole bf16 buffers: nothing written outside the window
        torch.testing.assert_close(gpu[i].float(), cpu[i].float(), atol=1e-3, rtol=2 ** -7)
    if dest == "u8":
        d = (gpu[4].int() - cpu[4].int()).abs()
        assert d.max() <= 1 and (d == 0).float().mean() > 0.99 and 0 < cpu[4].float().mean() < 255


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv2d_matches_torch(case):
    _run_case(case, None)


@pytest.mark.parametrize("tile_w", [8, 16, 32, 64, 128])
def test_conv2d_every_tile_width(tile_w):
    _run_case(("growth_tiles", 128, 192, 32, 0.2, False, False, False, "same", 19, 133), tile_w, seed=tile_w)
    _run_case(("conv5_tiles", 192, 192, 64, 0.0, True, True, True, "other", 45, 37), tile_w, seed=tile_w + 1)


def test_abi_validation_returns_status():
    from diffsynth import _native as nv
    lib = nv.load()
    D = torch.zeros(1, 8, 8, 192, dtype=torch.bfloat16, device=DEV)
    wp = torch.zeros(32, 9 * 128, dtype=torch.bfloat16, device=DEV)
    b = torch.zeros(32, device=DEV)
    d = nv.EsrganConvDesc()
    d.x, d.N, d.H, d.W, d.C_in, d.in_ld = D.data_ptr(), 1, 8, 8, 96, 192
    d.w_packed, d.w_rows, d.w_ld = wp.data_ptr(), 32, 9 * 128
    d.C_out, d.tile_w, d.bias, d.slope = 32, 8, b.data_ptr(), 0.2
    d.out_bf16, d.bf_ld = D.data_ptr() + 2 * 96, 192
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.svi_esrgan_conv2d(ctypes.byref(d), stream) == 0
    torch.cuda.synchronize()
    D.fill_(3.0)
    for field, bad, msg in (("out_bf16", D.data_ptr() + 2 * 64, "read window"),        # writes channels 64..95
                            ("out_bf16", D.data_ptr() + 2 * 97, "4-byte aligned"),     # odd channel offset
                            ("bf_up2", 1, "pixel layout"),
                            ("bf_ld", 96, "pixel layout"),
                            ("in_ld", 64, "in_ld"),
                            ("C_in", 100, "C_in"),
                            ("C_out", 31, "C_out"),
                            ("tile_w", 12, "tile_w"),
                            ("w_ld", 9 * 64, "packed weight")):
        old = getattr(d, field)
        setattr(d, field, bad)
        rc = lib.svi_esrgan_conv2d(ctypes.byref(d), stream)
        setattr(d, field, old)
        assert rc < 0, field
        assert msg in lib.svi_last_error().decode(), (field, lib.svi_last_error())
    torch.cuda.synchronize()
    assert bool((D == 3.0).all()), "a rejected launch wrote its output"
    assert lib.svi_esrgan_conv2d(None, stream) < 0
    assert lib.svi_esrgan_stage_frames(None, 4, None, stream) < 0


def _oracle(sd, x):
    torch.backends.cudnn.allow_tf32 = False
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = O.rrdbnet(sdd, x.to(DEV))
        pred = O.rrdbnet(sdd, x.to(DEV), rnd=_bf)
    return ref, pred


@pytest.mark.parametrize("H,W", [(480, 832), (203, 317)])
def test_rrdbnet_matches_oracle(model, sd, H, W):
    x = O.to_tensor(np.stack([np.asarray(f) for f in make_frames(1, H, W, seed=1)]))
    got = model(x.to(DEV))
    ref, pred = _oracle(sd, x)
    err = (got - ref).abs().mean().item()
    perr = (pred - ref).abs().mean().item()
    d = np.abs(O.to_uint8(got.cpu()).astype(int) - O.to_uint8(ref.cpu()).astype(int))
    print(f"RRDBNet {W}x{H}: mean|d| / std = {err / ref.std().item():.4%} (rounding study {perr / ref.std().item():.4%}), "
          f"max|d| / std = {(got - ref).abs().max().item() / ref.std().item():.3%}, uint8 mean|d| {d.mean():.3f}, "
          f"within 2: {(d <= 2).mean():.4%}")
    assert got.shape == (1, 3, 4 * H, 4 * W)
    assert err <= 1.25 * perr
    assert d.mean() <= 0.5 and (d <= 2).mean() >= 0.995


def test_upscale_matches_oracle_and_is_reproducible(model, sd):
    from diffsynth.extensions.ESRGAN import ESRGAN
    frames = make_frames(5, 241, 419, seed=2)
    esr = ESRGAN(model)
    a = np.stack([np.asarray(f) for f in esr.upscale(frames, batch_size=1)])
    b = np.stack([np.asarray(f) for f in esr.upscale(frames, batch_size=4)])
    c = np.stack([np.asarray(f) for f in esr.upscale(frames, batch_size=4)])
    assert a.shape == (5, 964, 1676, 3)
    assert np.array_equal(a, b) and np.array_equal(b, c)
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ref = O.upscale({k: v.to(DEV) for k, v in sd.items()}, np.stack([np.asarray(f) for f in frames]), batch_size=1)
    d = np.abs(b.astype(int) - ref.astype(int))
    print(f"upscale 5 frames 419x241: uint8 mean|d| {d.mean():.3f}, within 2: {(d <= 2).mean():.4%}")
    assert d.mean() <= 0.5 and (d <= 2).mean() >= 0.995
