"""CPU: ESRGAN 4x upscaling — the oracle against the reference's golden outputs, the weight packing of every conv width
in fp64, the C header and its ctypes mirrors, checkpoint detection and config checks, and the engine's buffer plan on the
torch stand-ins (tests/nv_emulation_esrgan.py) against the oracle."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

import nv_emulation_esrgan as emu
from oracle import esrgan_oracle as O
from tools import synth_esrgan as S
from tools.synth_rife import make_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "svi_b200_esrgan.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "esrgan_tiny.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def sd2():
    return S.make_state_dict(2, seed=0)


@pytest.fixture(scope="module")
def sd23():
    return S.make_state_dict(23, seed=0)


def _model(sd, num_block):
    from diffsynth.extensions.ESRGAN import RRDBNet
    m = RRDBNet(num_block=num_block).eval()
    m.load_state_dict(sd)
    return m


def _bf(t):
    return t.to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------- oracle vs reference
def test_golden_weights_are_the_synth_weights(golden, sd2, sd23):
    assert S.weight_checksum(sd2) == pytest.approx(float(golden["checksum_nb2"]), rel=1e-12)
    assert S.weight_checksum(sd23) == pytest.approx(float(golden["checksum_nb23"]), rel=1e-12)


@pytest.mark.parametrize("nb,i", [(2, 0), (2, 1), (2, 2), (23, 0)])
def test_oracle_rrdbnet_matches_reference(golden, sd2, sd23, nb, i):
    with torch.no_grad():
        y = O.rrdbnet(sd2 if nb == 2 else sd23, torch.from_numpy(golden[f"nb{nb}_x{i}"]))
    np.testing.assert_allclose(y.numpy(), golden[f"nb{nb}_y{i}"], atol=1e-5, rtol=1e-5)


def test_oracle_upscale_bytes_match_reference(golden, sd2):
    """Within one grey level: fp32 round-off moves a few values across a truncation boundary."""
    with torch.no_grad():
        got = O.upscale(sd2, golden["frames"], batch_size=2)
    assert got.shape == golden["upscale"].shape
    d = np.abs(got.astype(int) - golden["upscale"].astype(int))
    assert d.max() <= 1 and (d == 0).mean() >= 0.999


# ------------------------------------------------------------------------------------------- packing, fp64
@pytest.mark.parametrize("C_in,C_out,in_ld", [(3, 64, 8), (64, 32, 192), (96, 32, 192), (128, 32, 192), (160, 32, 192),
                                              (192, 64, 192), (64, 64, 64), (64, 3, 64)])
def test_packing_reproduces_conv2d(C_in, C_out, in_ld):
    """Every conv width of the network through pack_model's packing and the stand-in's descriptor reading (input pitch,
    zero K padding, conv_last's zero fourth column)."""
    from diffsynth.extensions.ESRGAN import LAST_COLS, pack_model
    g = torch.Generator().manual_seed(C_in + C_out)
    conv = torch.nn.Conv2d(C_in, C_out, 3, 1, 1).double()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g, dtype=torch.float64))
        conv.bias.copy_(torch.randn(C_out, generator=g, dtype=torch.float64))
    holder = torch.nn.Module()
    holder.add_module("conv_last" if C_out == 3 else "conv", conv)
    w, b = next(iter(pack_model(holder).values()))
    x = torch.randn(2, C_in, 7, 11, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, conv.weight, conv.bias, padding=1).permute(0, 2, 3, 1)
    buf = torch.randn(2, 7, 11, in_ld, generator=g, dtype=torch.float64)      # channels past C_in must not be read
    buf[..., :C_in] = x.permute(0, 2, 3, 1)
    cols = LAST_COLS if C_out == 3 else C_out
    out = torch.empty(2, 7, 11, cols, dtype=torch.float64)
    emu.esrgan_conv2d(buf[..., :C_in], w, cols, b, 16, out=out)
    torch.testing.assert_close(out[..., :C_out], ref, atol=1e-10, rtol=1e-10)
    assert out[..., C_out:].abs().max() == 0 if cols > C_out else True


# ------------------------------------------------------------------------------------------- C ABI
def test_esrgan_header_is_plain_c():
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        HEADER], capture_output=True, text=True)
    assert r.returncode == 0 and not r.stdout and not r.stderr, r.stdout + r.stderr


def test_esrgan_struct_mirror_matches_the_c_layout(tmp_path):
    from diffsynth import _native as nv
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    st, cname = nv.EsrganConvDesc, "svi_esrgan_conv_desc"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "svi_b200_esrgan.h"', 'int main(void) {',
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


def test_every_esrgan_entry_point_is_bound_exported_and_has_a_gpu_case():
    from diffsynth import _native as nv
    import test_esrgan_gpu as gpu
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))
    assert names == {"svi_esrgan_stage_frames", "svi_esrgan_conv2d"}
    assert names == set(nv.ESRGAN_SIGNATURES), "include/svi_b200_esrgan.h and ESRGAN_SIGNATURES disagree"
    assert not names & (set(nv.SIGNATURES) | set(nv.LORA_SIGNATURES) | set(nv.RIFE_SIGNATURES))
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)


# ------------------------------------------------------------------------------------------- detection, config
def test_default_rrdbnet_hash_and_detection(sd23):
    from diffsynth.extensions.ESRGAN import RRDBNet
    from diffsynth.models.model_manager import ModelDetectorFromSingleFile, _loader_table
    from diffsynth.models.utils import hash_state_dict_keys
    m = RRDBNet()
    assert len(m.state_dict()) == 702 and sum(p.numel() for p in m.parameters()) == 16_697_987
    assert hash_state_dict_keys(m.state_dict(), with_shape=True) == "6b7116078c4170bfbeaedc8fe71f6649"
    det = ModelDetectorFromSingleFile(_loader_table())
    assert det.match(state_dict=sd23)
    names, models = det.load(state_dict=sd23, device="cpu", torch_dtype=torch.float32)
    assert names == ["esrgan"] and isinstance(models[0], RRDBNet)
    torch.testing.assert_close(models[0].body[22].rdb3.conv5.weight, sd23["body.22.rdb3.conv5.weight"])


def test_state_dict_converter_upcasts():
    from diffsynth.extensions.ESRGAN import RRDBNet
    sd = {"a": torch.zeros(1)}
    for fn in ("from_civitai", "from_diffusers"):
        out, extra = getattr(RRDBNet.state_dict_converter(), fn)(sd)
        assert out is sd and extra == {"upcast_to_float32": True}


@pytest.mark.parametrize("field,value", [("num_feat", 32), ("num_grow_ch", 16), ("num_in_ch", 4), ("num_out_ch", 1),
                                         ("num_block", 0)])
def test_unsupported_config_raises(field, value):
    from diffsynth.extensions.ESRGAN import RRDBNet
    with pytest.raises(ValueError, match=field):
        RRDBNet(**{field: value})


# ------------------------------------------------------------------------------------------- engine on the stand-ins
def _u8(images):
    return np.stack([np.asarray(im) for im in images])


@pytest.mark.parametrize("nb,H,W", [(2, 13, 17), (2, 9, 22), (23, 10, 12)])
def test_engine_rrdbnet_matches_oracle(monkeypatch, sd2, sd23, nb, H, W):
    emu.install(monkeypatch)
    sd = sd2 if nb == 2 else sd23
    x = O.to_tensor(_u8(make_frames(2, H, W, seed=nb)))
    got = _model(sd, nb)(x)
    with torch.no_grad():
        ref = O.rrdbnet(sd, x)
        pred = (O.rrdbnet(sd, x, rnd=_bf) - ref).abs().mean().item()
    assert got.shape == (2, 3, 4 * H, 4 * W)
    err = (got - ref).abs().mean().item()
    # the stand-in rounds at the oracle's bf16 points but accumulates in fp64, so its rounding points flip independently
    assert err <= 1.5 * pred + 1e-6, (err, pred)
    d = np.abs(O.to_uint8(got).astype(int) - O.to_uint8(ref).astype(int))
    assert d.mean() <= 0.5 and (d <= 2).mean() >= 0.995


def test_upscale_single_image_and_list(monkeypatch, sd2):
    from diffsynth.extensions.ESRGAN import ESRGAN
    emu.install(monkeypatch)
    frames = make_frames(3, 11, 7, seed=1)
    esr = ESRGAN(_model(sd2, 2))
    many = esr.upscale(frames, batch_size=2)
    one = esr.upscale(frames[1])
    assert isinstance(many, list) and len(many) == 3 and isinstance(one, Image.Image)
    assert one.size == (28, 44) and np.array_equal(np.asarray(one), np.asarray(many[1]))
    grey = esr.upscale([frames[0].convert("L")])[0]                       # non-RGB modes are converted
    assert grey.mode == "RGB" and grey.size == (28, 44)
    with pytest.raises(ValueError, match="size of the first"):
        esr.upscale([frames[0], make_frames(1, 12, 7)[0]])


def test_upscale_matches_oracle_and_ignores_batch_size(monkeypatch, sd2):
    from diffsynth.extensions.ESRGAN import ESRGAN
    emu.install(monkeypatch)
    frames = make_frames(5, 9, 13, seed=2)
    esr = ESRGAN(_model(sd2, 2))
    outs = [_u8(esr.upscale(frames, batch_size=b)) for b in (1, 2, 4)]
    assert all(np.array_equal(outs[0], o) for o in outs[1:])
    with torch.no_grad():
        ref = O.upscale(sd2, _u8(frames))
    d = np.abs(outs[0].astype(int) - ref.astype(int))
    assert outs[0].shape == (5, 36, 52, 3) and d.mean() <= 0.5 and (d <= 2).mean() >= 0.995


def test_no_launch_writes_a_channel_window_it_reads(monkeypatch, sd2):
    """Every launch of the engine's plan, as its descriptor states it: a bf16 destination in the input's buffer keeps
    the input's pixel layout and lies past the read window [0, C_in); f32 outputs are never read as a conv input."""
    from diffsynth.extensions.ESRGAN import ESRGANEngine
    emu.install(monkeypatch)
    eng = ESRGANEngine(_model(sd2, 2), "cpu")
    rgb = torch.empty(2, 20, 28, 3, dtype=torch.uint8)
    steps = eng.plan(2, 5, 7, rgb=rgb, out=torch.empty(2, 20, 28, 4))
    assert len(steps) == 1 + 2 * 15 + 5
    seen_dense = 0
    for name, x, C_out, _, ep in steps:
        assert x.dtype == torch.bfloat16
        o = ep.get("out_bf16")
        if o is None or o.untyped_storage().data_ptr() != x.untyped_storage().data_ptr():
            continue
        seen_dense += 1
        ld = x.stride(2)
        assert o.stride() == x.stride() and not ep.get("bf_up2")
        x0, o0 = x.storage_offset() % ld, o.storage_offset() % ld
        assert x.storage_offset() - x0 == o.storage_offset() - o0           # the same pixels
        assert x0 + x.shape[3] <= o0 and o0 + C_out <= ld, name             # written channels lie past the read window
    assert seen_dense == 2 * 3 * 4                                          # the growth convs of every dense block
