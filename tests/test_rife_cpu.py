"""CPU: RIFE frame interpolation — the oracle against the reference's golden outputs, the weight packing of the
space-to-depth and sub-pixel convolutions in fp64, the C header and its ctypes mirrors, checkpoint detection, and the
engine's host logic on the torch stand-ins (tests/nv_emulation_rife.py) against the oracle."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import nv_emulation_rife as emu
from oracle import rife_oracle as O
from tools import synth_rife as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "svi_b200_rife.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "rife_tiny.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def sd():
    return S.make_state_dict(seed=0)


# ------------------------------------------------------------------------------------------- oracle vs reference
def test_golden_weights_are_the_synth_weights(golden, sd):
    assert S.weight_checksum(sd) == pytest.approx(float(golden["checksum"]), rel=1e-12)


@pytest.mark.parametrize("tag,scale", [("s1", 1.0), ("s05", 0.5)])
def test_oracle_ifnet_matches_reference(golden, sd, tag, scale):
    x = torch.from_numpy(golden["x"])
    with torch.no_grad():
        flows, mask, merged = O.ifnet(sd, x, [4 / scale, 2 / scale, 1 / scale])
    np.testing.assert_allclose(torch.stack(flows).numpy(), golden[f"{tag}_flows"], atol=2e-4, rtol=1e-4)
    np.testing.assert_allclose(mask.numpy(), golden[f"{tag}_mask"], atol=2e-5)
    np.testing.assert_allclose(torch.stack(merged).numpy(), golden[f"{tag}_merged"], atol=2e-5)


def test_oracle_interpolate_and_smoother_match_reference(golden, sd):
    frames = golden["frames"]
    with torch.no_grad():
        got = O.interpolate(sd, frames[:3], batch_size=2, num_iter=2)
        sm = O.smooth(sd, frames, batch_size=2)
    for a, b in ((got, golden["interp2"]), (sm, golden["smooth"])):
        assert a.shape == b.shape
        assert np.abs(a.astype(int) - b.astype(int)).max() <= 1


# ------------------------------------------------------------------------------------------- packing, fp64
def test_s2d_packing_reproduces_strided_conv():
    from diffsynth.extensions.RIFE import pack_s2d
    g = torch.Generator().manual_seed(1)
    for I, group, cpad in ((11, 11, 64), (45, 46, 192)):
        w = torch.randn(7, I, 3, 3, generator=g, dtype=torch.float64)
        b = torch.randn(7, generator=g, dtype=torch.float64)
        x = torch.randn(2, I, 12, 20, generator=g, dtype=torch.float64)
        ref = F.conv2d(x, w, b, stride=2, padding=1).permute(0, 2, 3, 1)
        xs = torch.zeros(2, 6, 10, 4 * group, dtype=torch.float64)
        xl = x.permute(0, 2, 3, 1)
        for dy in range(2):
            for dx in range(2):
                xs[..., (dy * 2 + dx) * group:(dy * 2 + dx) * group + I] = xl[:, dy::2, dx::2]
        out = torch.empty(2, 6, 10, 8, dtype=torch.float64)
        wp = torch.cat([pack_s2d(w, group, cpad), torch.zeros(1, 4 * cpad, dtype=torch.float64)])
        emu.rife_conv2d(xs, wp, 2, 2, 1, 8, 8, torch.cat([b, torch.zeros(1, dtype=torch.float64)]), 16, out=out)
        torch.testing.assert_close(out[..., :7], ref, atol=1e-12, rtol=1e-12)


def test_subpixel_packing_reproduces_conv_transpose():
    from diffsynth.extensions.RIFE import pack_subpixel, _phases
    g = torch.Generator().manual_seed(2)
    for I, O_, cols in ((90, 45, 90), (45, 4, 6)):
        w = torch.randn(I, O_, 4, 4, generator=g, dtype=torch.float64)
        b = torch.randn(O_, generator=g, dtype=torch.float64)
        x = torch.randn(2, I, 5, 7, generator=g, dtype=torch.float64)
        ref = F.conv_transpose2d(x, w, b, stride=2, padding=1).permute(0, 2, 3, 1)
        out = torch.empty(2, 10, 14, cols, dtype=torch.float64)
        emu.rife_conv2d(x.permute(0, 2, 3, 1).contiguous(), pack_subpixel(w, cols, (I + 63) // 64 * 64), 3, 3, 1, 4 * cols, cols,
                        _phases(b, cols), 16, out=out)
        torch.testing.assert_close(out[..., :O_], ref, atol=1e-12, rtol=1e-12)
        assert out[..., O_:].abs().max() == 0


# ------------------------------------------------------------------------------------------- C ABI
def test_rife_header_is_plain_c():
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        HEADER], capture_output=True, text=True)
    assert r.returncode == 0 and not r.stdout and not r.stderr, r.stdout + r.stderr


@pytest.mark.parametrize("cname,pyname", [("svi_rife_conv_desc", "RifeConvDesc"), ("svi_rife_block_input", "RifeBlockInput"),
                                          ("svi_rife_update", "RifeUpdate")])
def test_rife_struct_mirrors_match_the_c_layout(tmp_path, cname, pyname):
    from diffsynth import _native as nv
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    st = getattr(nv, pyname)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "svi_b200_rife.h"', 'int main(void) {',
             f'  printf("sizeof %zu\\n", sizeof({cname}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in st._fields_]
    lines += ['  return 0;', '}']
    (tmp_path / "probe.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(tmp_path / "probe.c"), "-o", str(tmp_path / "probe")],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                                       text=True).stdout.split("\n") if line)
    assert int(got.pop("sizeof")) == ctypes.sizeof(st)
    assert {f: int(v) for f, v in got.items()} == {f: getattr(st, f).offset for f, _ in st._fields_}


def test_every_rife_entry_point_is_bound_exported_and_has_a_gpu_case():
    from diffsynth import _native as nv
    import test_rife_gpu as gpu
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))
    assert names == {"svi_rife_stage_frames", "svi_rife_block_input_launch", "svi_rife_conv2d", "svi_rife_update_warp"}
    assert names == set(nv.RIFE_SIGNATURES), "include/svi_b200_rife.h and RIFE_SIGNATURES disagree"
    assert not names & (set(nv.SIGNATURES) | set(nv.LORA_SIGNATURES))
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)


# ------------------------------------------------------------------------------------------- detection
def test_module_prefixed_state_dict_is_detected_as_rife():
    from diffsynth.models.model_manager import ModelDetectorFromSingleFile, _loader_table
    from diffsynth.extensions.RIFE import IFNet
    sd = S.make_state_dict(seed=0, prefix="module.")
    det = ModelDetectorFromSingleFile(_loader_table())
    assert det.match(state_dict=sd)
    names, models = det.load(state_dict=sd, device="cpu", torch_dtype=torch.float32)
    assert names == ["rife"] and isinstance(models[0], IFNet)
    torch.testing.assert_close(models[0].block1.conv1[2].weight, sd["module.block1.conv1.2.weight"])


# ------------------------------------------------------------------------------------------- engine on the stand-ins
def _model(sd):
    from diffsynth.extensions.RIFE import IFNet
    m = IFNet().eval()
    m.load_state_dict(sd)
    return m


def _bf(t):
    return t.to(torch.bfloat16).float()


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_engine_ifnet_matches_oracle(monkeypatch, golden, sd, scale):
    emu.install(monkeypatch)
    x = torch.from_numpy(golden["x"])
    flows, mask, merged = _model(sd)(x, [4 / scale, 2 / scale, 1 / scale])
    with torch.no_grad():
        rf, rm, rmg = O.ifnet(sd, x, [4 / scale, 2 / scale, 1 / scale], rnd=_bf)
    # bf16 rounding points flip independently of the oracle's (its resizes are ATen's): compare at the engine's bar
    for a, b in zip(flows, rf):
        assert (a - b).abs().mean() <= 1e-2 * b.std()
    assert (mask - rm).abs().mean() < 1e-2 and (merged[2] - rmg[2]).abs().mean() < 1e-2


def _u8(images):
    return np.stack([np.asarray(im) for im in images])


@pytest.mark.parametrize("num_iter", [1, 2])
def test_interpolate_frame_order_and_values(monkeypatch, golden, sd, num_iter):
    from diffsynth.extensions.RIFE import RIFEInterpolater
    emu.install(monkeypatch)
    frames = golden["frames"]
    from PIL import Image
    pil = [Image.fromarray(f) for f in frames]
    got = _u8(RIFEInterpolater(_model(sd), device="cpu").interpolate(pil, batch_size=2, num_iter=num_iter))
    with torch.no_grad():
        ref = O.interpolate(sd, frames, batch_size=2, num_iter=num_iter, rnd=_bf)
    assert got.shape == ref.shape == (2 ** num_iter * 3 + 1, 32, 64, 3)
    assert np.array_equal(got[::2 ** num_iter], frames)              # the input frames keep their places and bytes
    d = np.abs(got.astype(int) - ref.astype(int))
    assert d.mean() <= 0.5 and (d <= 2).mean() >= 0.99


def test_interpolate_underscore_returns_the_new_frames(monkeypatch, golden, sd):
    from diffsynth.extensions.RIFE import RIFEInterpolater
    from PIL import Image
    emu.install(monkeypatch)
    pil = [Image.fromarray(f) for f in golden["frames"]]
    r = RIFEInterpolater(_model(sd), device="cpu")
    assert np.array_equal(_u8(r.interpolate_(pil)), _u8(r.interpolate(pil))[1::2])


def test_smoother_formula(monkeypatch, golden, sd):
    from diffsynth.extensions.RIFE import RIFESmoother
    from PIL import Image
    emu.install(monkeypatch)
    frames = golden["frames"]
    got = _u8(RIFESmoother(_model(sd), device="cpu")([Image.fromarray(f) for f in frames], batch_size=2))
    with torch.no_grad():
        ref = O.smooth(sd, frames, batch_size=2, rnd=_bf)
    d = np.abs(got.astype(int) - ref.astype(int))
    assert np.array_equal(got[[0, -1]], frames[[0, -1]]) and d.mean() <= 0.5 and (d <= 2).mean() >= 0.99


def test_batch_size_invariance(monkeypatch, golden, sd):
    from diffsynth.extensions.RIFE import RIFEInterpolater
    from PIL import Image
    emu.install(monkeypatch)
    pil = [Image.fromarray(f) for f in golden["frames"]]
    r = RIFEInterpolater(_model(sd), device="cpu")
    outs = [_u8(r.interpolate(pil, batch_size=b)) for b in (1, 2, 4)]
    assert all(np.array_equal(outs[0], o) for o in outs[1:])


def test_size_rule():
    from diffsynth.extensions.RIFE import check_size
    for H, W in ((480, 832), (720, 1280), (464, 848), (64, 96)):
        check_size(H, W, [4, 2, 1])                                        # multiples of 16 at scale 1
    check_size(480, 832, [8, 4, 2])
    for H, W, sl in ((720, 1280, [8, 4, 2]), (488, 832, [4, 2, 1]), (480, 830, [4, 2, 1])):
        with pytest.raises(ValueError, match="multiple of 4"):
            check_size(H, W, sl)


def test_size_rule_errors_reach_the_public_interface(monkeypatch, sd):
    from diffsynth.extensions.RIFE import RIFEInterpolater
    emu.install(monkeypatch)
    frames = S.make_frames(2, 40, 64)
    with pytest.raises(ValueError, match="multiple of 4"):
        RIFEInterpolater(_model(sd), device="cpu").interpolate(frames)
    with pytest.raises(ValueError, match="size of the first"):
        RIFEInterpolater(_model(sd), device="cpu").interpolate(frames[:1] + S.make_frames(1, 32, 64))
