"""CPU: the video processors (diffsynth.processors) — the oracle against the installed Pillow bit for bit over a sweep of
sizes, rates and frame contents, the RIFE smoother's oracle and the editor chain against the reference's own processors
(tests/golden/processors_tiny.npz), dispatch and chaining, the chain's orchestration on the torch stand-ins
(tests/nv_emulation_processors.py), the inputs the processors refuse, and the C header against its bindings and GPU
cases."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from PIL import Image, ImageEnhance, ImageFilter

import nv_emulation_processors as emu
from oracle import processors_oracle as P
from tools import synth_rife as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "svi_b200_processors.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "processors_tiny.npz")
RATES = [0.0, 1.0, 0.25, 0.5, 0.999, 1.5, 2.0, 3.3, 17.0, -0.7, -2.5]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def sd():
    return S.make_state_dict(seed=0)


def _u8(images):
    return np.stack([np.asarray(im) for im in images])


def _pil(frames):
    return [Image.fromarray(f) for f in frames]


# ------------------------------------------------------------------------------------------- oracle vs Pillow
def sweep_frames():
    """(name, uint8 RGB frame): edge sizes, odd and even sides up to a few hundred pixels, random, near-constant and
    saturated content"""
    rng = np.random.default_rng(11)
    sizes = [(1, 1), (2, 2), (1, 7), (7, 1), (3, 3), (3, 17), (17, 3), (4, 5), (31, 64), (64, 31), (127, 200), (240, 416),
             (301, 257)]
    out = []
    for H, W in sizes:
        out.append((f"random{H}x{W}", rng.integers(0, 256, (H, W, 3), dtype=np.uint8)))
        out.append((f"flat{H}x{W}", np.clip(127 + rng.integers(-2, 3, (H, W, 3)), 0, 255).astype(np.uint8)))
        out.append((f"saturated{H}x{W}", np.where(rng.random((H, W, 3)) < 0.5, 0, 255).astype(np.uint8)))
    out.append(("black", np.zeros((9, 11, 3), np.uint8)))
    out.append(("white", np.full((9, 11, 3), 255, np.uint8)))
    return out


SWEEP = sweep_frames()


def test_smooth_weights_are_the_pillow_filter():
    size, divisor, offset, kernel = ImageFilter.SMOOTH.filterargs
    assert size == (3, 3) and offset == 0
    assert np.array_equal(P.SMOOTH_W, np.array(kernel, np.float32) / np.float32(divisor))
    # Pillow divides its float32 kernel by the double divisor; both quotients round to the same floats
    assert np.array_equal(P.SMOOTH_W, np.array([np.float32(k / divisor) for k in kernel], np.float32))


@pytest.mark.parametrize("name,frame", SWEEP, ids=[n for n, _ in SWEEP])
def test_oracle_matches_pillow_bitwise(name, frame):
    im = Image.fromarray(frame)
    assert P.luma_sum(frame) == int(sum(i * h for i, h in enumerate(im.convert("L").histogram())))
    assert np.array_equal(P.smooth(frame), np.asarray(im.filter(ImageFilter.SMOOTH)))
    for rate in RATES:
        assert np.array_equal(P.contrast(frame, rate), np.asarray(ImageEnhance.Contrast(im).enhance(rate))), rate
        assert np.array_equal(P.sharpness(frame, rate), np.asarray(ImageEnhance.Sharpness(im).enhance(rate))), rate


# ------------------------------------------------------------------------------------------- oracle vs reference
def test_golden_weights_are_the_synth_weights(golden, sd):
    assert S.weight_checksum(sd) == pytest.approx(float(golden["checksum"]), rel=1e-12)


@pytest.mark.parametrize("interpolate,tag", [(True, "rife_interp"), (False, "rife_avg")])
def test_rife_oracle_matches_reference_processor(golden, sd, interpolate, tag):
    with torch.no_grad():
        got = P.rife_smooth(sd, golden["frames"], batch_size=2, interpolate=interpolate)
    assert got.shape == golden[tag].shape
    assert np.array_equal(got[[0, -1]], golden["frames"][[0, -1]])
    assert np.abs(got.astype(int) - golden[tag].astype(int)).max() <= 1


def test_editor_chain_oracle_matches_reference(golden):
    got = np.stack([P.sharpness(P.contrast(f, 1.7), 2.3) for f in golden["chain_frames"]])
    assert np.array_equal(got, golden["chain"])


# ------------------------------------------------------------------------------------------- dispatch and chaining
class _Manager:
    device = "cpu"

    def __init__(self, model=None):
        self.model = model

    def fetch_model(self, name, *args, **kwargs):
        assert name == "rife"
        return self.model


def test_auto_processor_dispatch_and_error():
    from diffsynth.processors.FastBlend import FastBlendSmoother
    from diffsynth.processors.PILEditor import ContrastEditor, SharpnessEditor
    from diffsynth.processors.RIFE import RIFESmoother
    from diffsynth.processors.sequencial_processor import AutoVideoProcessor
    m = _Manager(model="ifnet")
    fb = AutoVideoProcessor.from_model_manager(m, "FastBlend", inference_mode="balanced", window_size=3)
    assert isinstance(fb, FastBlendSmoother) and fb.inference_mode == "balanced" and fb.window_size == 3
    c = AutoVideoProcessor.from_model_manager(m, "Contrast", rate=0.7)
    s = AutoVideoProcessor.from_model_manager(m, "Sharpness")
    assert isinstance(c, ContrastEditor) and c.rate == 0.7 and isinstance(s, SharpnessEditor) and s.rate == 1.5
    r = AutoVideoProcessor.from_model_manager(m, "RIFE", scale=0.5, batch_size=2, interpolate=False)
    assert isinstance(r, RIFESmoother) and r.model == "ifnet" and r.device == "cpu"
    assert (r.scale, r.batch_size, r.interpolate) == (0.5, 2, False)
    with pytest.raises(ValueError, match="invalid processor_type: ESRGAN"):
        AutoVideoProcessor.from_model_manager(m, "ESRGAN")


def test_sequencial_processor_from_configs_passes_kwargs_to_each():
    from diffsynth.processors.base import VideoProcessor
    from diffsynth.processors.sequencial_processor import SequencialProcessor
    chain = SequencialProcessor.from_model_manager(_Manager(), [
        {"processor_type": "Contrast", "config": {"rate": 1.2}},
        {"processor_type": "FastBlend", "config": {"inference_mode": "fast", "window_size": 5}},
        {"processor_type": "Sharpness", "config": {}}])
    assert [type(p).__name__ for p in chain.processors] == ["ContrastEditor", "FastBlendSmoother", "SharpnessEditor"]
    calls = []

    class Tag(VideoProcessor):
        def __init__(self, tag):
            self.tag = tag

        def __call__(self, frames, **kwargs):
            calls.append((self.tag, kwargs))
            return frames + [self.tag]

    out = SequencialProcessor([Tag("a"), Tag("b")])(["x"], original_frames="guide", extra=3)
    assert out == ["x", "a", "b"]
    assert calls == [("a", dict(original_frames="guide", extra=3)), ("b", dict(original_frames="guide", extra=3))]


# ------------------------------------------------------------------------------------------- on the stand-ins
def _rife_model(sd):
    from diffsynth.extensions.RIFE import IFNet
    m = IFNet().eval()
    m.load_state_dict(sd)
    return m


def _editors(device="cpu"):
    from diffsynth.processors.PILEditor import ContrastEditor, SharpnessEditor
    c, s = ContrastEditor(rate=1.7), SharpnessEditor(rate=2.3)
    c.device = s.device = device
    return c, s


def test_editors_on_stand_ins_match_reference_chain(monkeypatch, golden):
    from diffsynth.processors.sequencial_processor import SequencialProcessor
    emu.install(monkeypatch)
    c, s = _editors()
    frames = golden["chain_frames"]
    assert np.array_equal(_u8(SequencialProcessor([c, s])(_pil(frames))), golden["chain"])
    assert np.array_equal(_u8(s(c(_pil(frames)))), golden["chain"])
    t = torch.from_numpy(frames.copy())
    out = SequencialProcessor([c, s])(t)
    assert torch.is_tensor(out) and np.array_equal(out.numpy(), golden["chain"]) and np.array_equal(t.numpy(), frames)


@pytest.mark.parametrize("interpolate", [True, False])
def test_rife_processor_on_stand_ins(monkeypatch, golden, sd, interpolate):
    from diffsynth.processors.RIFE import RIFESmoother
    emu.install(monkeypatch)
    frames = golden["frames"]
    r = RIFESmoother(_rife_model(sd), device="cpu", batch_size=2, interpolate=interpolate)
    got = _u8(r(_pil(frames)))
    with torch.no_grad():
        ref = P.rife_smooth(sd, frames, batch_size=2, interpolate=interpolate, rnd=lambda t: t.to(torch.bfloat16).float())
    d = np.abs(got.astype(int) - ref.astype(int))
    assert np.array_equal(got[[0, -1]], frames[[0, -1]]) and d.mean() <= 0.5 and (d <= 2).mean() >= 0.99
    t = torch.from_numpy(frames.copy())
    assert np.array_equal(r(t).numpy(), got) and np.array_equal(t.numpy(), frames)
    r.batch_size = 1
    assert np.array_equal(_u8(r(_pil(frames))), got)


@pytest.mark.slow
def test_four_processor_chain_on_stand_ins(monkeypatch, golden, sd):
    """[FastBlend fast, RIFE, Contrast, Sharpness]: PIL in = one by one through PIL = a tensor in; an outside processor
    between them gets PIL frames"""
    from diffsynth.processors.FastBlend import FastBlendSmoother
    from diffsynth.processors.RIFE import RIFESmoother
    from diffsynth.processors.base import VideoProcessor
    from diffsynth.processors.sequencial_processor import SequencialProcessor
    emu.install(monkeypatch)
    frames = S.make_frames(5, 32, 64, seed=4)
    guide = S.make_frames(5, 32, 64, seed=9)
    fb = FastBlendSmoother(inference_mode="fast", batch_size=2, window_size=2)
    r = RIFESmoother(_rife_model(sd), device="cpu", batch_size=2, interpolate=False)
    c, s = _editors()
    seen = []

    class Outside(VideoProcessor):
        def __call__(self, frames, **kwargs):
            seen.append(type(frames))
            assert all(isinstance(f, Image.Image) for f in frames)
            return frames

    one_by_one = frames
    for p in (fb, r, c, s):
        one_by_one = p(one_by_one, original_frames=guide)
    ref = _u8(one_by_one)
    chained = SequencialProcessor([fb, r, c, s])(frames, original_frames=guide)
    assert all(isinstance(f, Image.Image) for f in chained) and np.array_equal(_u8(chained), ref)
    t = torch.from_numpy(np.stack([np.asarray(f) for f in frames]))
    assert np.array_equal(SequencialProcessor([fb, r, c, s])(t, original_frames=guide).numpy(), ref)
    assert np.array_equal(_u8(SequencialProcessor([fb, r, Outside(), c, s])(frames, original_frames=guide)), ref)
    assert seen == [list]


def test_chain_returns_the_kind_it_was_given(monkeypatch, golden):
    """a tensor in gives a tensor out on the same device, also when the last processor is from outside the package"""
    from diffsynth.processors.base import VideoProcessor
    from diffsynth.processors.sequencial_processor import SequencialProcessor
    emu.install(monkeypatch)
    c, s = _editors()

    class Outside(VideoProcessor):
        def __call__(self, frames, **kwargs):
            assert all(isinstance(f, Image.Image) for f in frames)
            return frames

    t = torch.from_numpy(golden["chain_frames"].copy())
    out = SequencialProcessor([c, s, Outside()])(t)
    assert torch.is_tensor(out) and out.device == t.device and np.array_equal(out.numpy(), golden["chain"])
    pil = SequencialProcessor([c, Outside(), s])(_pil(golden["chain_frames"]))
    assert all(isinstance(f, Image.Image) for f in pil) and np.array_equal(_u8(pil), golden["chain"])
    assert SequencialProcessor().processors == [] and SequencialProcessor()(t) is t
    with pytest.raises(ValueError, match="ContrastEditor: frames must be PIL images of mode RGB"):
        SequencialProcessor([c, s])([im.convert("L") for im in _pil(golden["chain_frames"])])


# ------------------------------------------------------------------------------------------- refused input
def test_processors_refuse_bad_frames_before_any_launch(monkeypatch, sd):
    from diffsynth import _native as nv
    from diffsynth.processors.RIFE import RIFESmoother
    emu.install(monkeypatch)
    for name in emu._NAMES + ("rife_stage_frames", "rife_block_input", "fastblend_stage_frames"):
        monkeypatch.setattr(nv, name, lambda *a, **k: pytest.fail("launched"))
    c, s = _editors()
    r = RIFESmoother(_rife_model(sd), device="cpu")
    small = S.make_frames(3, 32, 64)
    for p, who in ((c, "ContrastEditor"), (s, "SharpnessEditor"), (r, "RIFESmoother")):
        with pytest.raises(ValueError, match=f"{who}: every frame must have the size"):
            p(small[:2] + S.make_frames(1, 32, 48))
        with pytest.raises(ValueError, match=f"{who}: frames must be PIL images of mode RGB"):
            p(small[:2] + [small[2].convert("L")])
        with pytest.raises(ValueError, match=f"{who}: a frame tensor must be uint8"):
            p(torch.zeros(3, 32, 64, 4, dtype=torch.uint8))
        with pytest.raises(ValueError, match=f"{who}: no frames"):
            p([])
    with pytest.raises(ValueError, match="at least 3 frames"):
        r(small[:2])
    with pytest.raises(ValueError, match="multiple of 4"):
        r(S.make_frames(3, 40, 64))
    with pytest.raises(ValueError, match="rate must be a finite"):
        _editors()[0].__class__(rate=float("nan"))(small)
    assert not r.model._engines                       # refused before the RIFE weights were packed


# ------------------------------------------------------------------------------------------- C ABI
def _header_names():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))


def test_processors_header_is_plain_c():
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        HEADER], capture_output=True, text=True)
    assert r.returncode == 0 and not r.stdout and not r.stderr, r.stdout + r.stderr


def test_every_processors_entry_point_is_bound_exported_and_has_a_gpu_case():
    from diffsynth import _native as nv
    import test_processors_gpu as gpu
    names = _header_names()
    assert names == {"svi_luma_sum_u8", "svi_enhance_blend_u8", "svi_sharpen_u8", "svi_rife_average_u8"}
    assert names == set(nv.PROCESSORS_SIGNATURES)
    others = set()
    for table in (nv.SIGNATURES, nv.LORA_SIGNATURES, nv.RIFE_SIGNATURES, nv.ESRGAN_SIGNATURES, nv.FASTBLEND_SIGNATURES,
                  nv.FASTBLEND_MODES_SIGNATURES, nv.UNIANIMATE_SIGNATURES, nv.REPLACE_SIGNATURES, nv.QUALITY_SIGNATURES,
                  nv.REWARD_SIGNATURES):
        others |= set(table)
    assert not names & others
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)
