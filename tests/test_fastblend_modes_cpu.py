"""CPU: FastBlend's balanced and accurate modes and keyframe interpolation — the oracle against the reference runners'
golden outputs bit for bit (tests/golden/fastblend_modes_tiny.npz), the engine's runners on the torch stand-ins
(tests/nv_emulation_fastblend_modes.py) against the same golden, the in-memory processor against the runners, the C header
and its ctypes mirrors, and the inputs the runners refuse."""
import ctypes
import importlib.util
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from PIL import Image

import nv_emulation_fastblend_modes as emu
from oracle import fastblend_modes_oracle as M
from tools.synth_fastblend import digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "svi_b200_fastblend_modes.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "fastblend_modes_tiny.npz")


def _recipe():
    """the golden's recipe module: its cases and the inputs it feeds them"""
    spec = importlib.util.spec_from_file_location("make_golden_fastblend_modes",
                                                  os.path.join(ROOT, "tests", "golden", "make_golden_fastblend_modes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _recipe()
ORACLE = {"BalancedModeRunner": M.balanced, "AccurateModeRunner": M.accurate, "InterpolationModeRunner": M.interpolation,
          "InterpolationModeSingleFrameRunner": M.single_frame}


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _check(golden, name, frames):
    frames = np.asarray(frames)
    assert frames.shape == (G.N, G.H, G.W, 3) and frames.dtype == np.uint8
    if name in golden.files:
        assert np.array_equal(frames, golden[name]), f"{int((frames != golden[name]).sum())} bytes differ"
    assert digest(frames, np.uint8) == str(golden[f"{name}_sha256"]), (
        f"sum {int(frames.astype(np.int64).sum())}, reference {int(golden[f'{name}_sum'])}")


def _config(config):
    return dict(dict(minimum_patch_size=5, threads_per_block=8, num_iter=5, gpu_id=0, guide_weight=10.0,
                     initialize="identity", tracking_window_size=0), **config)


# ------------------------------------------------------------------------------------------- oracle vs reference
@pytest.mark.slow
@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_reference_runners_bitwise(golden, name):
    runner, kwargs, config = G.CASES[name]
    frames, draws = ORACLE[runner](**G.case_inputs(runner, kwargs), **config)
    _check(golden, name, frames)
    assert draws == int(golden[f"{name}_draws"])


def test_golden_cases_differ_where_their_options_do(golden):
    """batch size, tracking and the patch size each change the reference's bytes in these cases"""
    for a, b in [("balanced_b3", "balanced_b8"), ("accurate_t0", "accurate_t1"), ("interp_p5_t0", "interp_p5_t1"),
                 ("interp_p15_t0", "interp_p15_t1"), ("interp_p5_t0", "interp_p15_t0")]:
        assert str(golden[f"{a}_sha256"]) != str(golden[f"{b}_sha256"]), (a, b)


# ------------------------------------------------------------------------------------------- the engine on stand-ins
def _pil(frames):
    return [Image.fromarray(np.asarray(f)) for f in frames]


@pytest.mark.slow
@pytest.mark.parametrize("name", ["balanced_b3", "accurate_t1", "interp_p5_t1", "interp_p15_t0", "single_t1_b4"])
def test_engine_runners_match_reference_bytes(monkeypatch, tmp_path, golden, name):
    emu.install(monkeypatch)
    from diffsynth.extensions.FastBlend import runners
    runner, kwargs, config = G.CASES[name]
    args = G.case_inputs(runner, kwargs)
    args["frames_guide"], args["frames_style"] = _pil(args["frames_guide"]), _pil(args["frames_style"])
    out = getattr(runners, runner)().run(ebsynth_config=_config(config), save_path=str(tmp_path), **args)
    assert all(isinstance(f, Image.Image) for f in out)
    _check(golden, name, np.stack([np.asarray(f) for f in out]))
    saved = np.stack([np.asarray(Image.open(tmp_path / ("%05d.png" % i))) for i in range(G.N)])
    _check(golden, name, saved)


@pytest.mark.slow
def test_processor_matches_the_runners(monkeypatch, golden):
    """diffsynth.processors.FastBlend: the reference's in-memory API (PIL in, PIL out) on the same runners"""
    emu.install(monkeypatch)
    from diffsynth.processors.FastBlend import FastBlendSmoother
    from diffsynth.processors.base import VideoProcessor
    guide, style = G.inputs()
    p = FastBlendSmoother(inference_mode="balanced", batch_size=3, window_size=2)
    assert isinstance(p, VideoProcessor)
    out = p(_pil(style), original_frames=_pil(guide))
    _check(golden, "balanced_b3", np.stack([np.asarray(f) for f in out]))


def test_processor_defaults_and_modes():
    from diffsynth.processors.FastBlend import FastBlendSmoother
    p = FastBlendSmoother.from_model_manager(None)
    assert (p.inference_mode, p.batch_size, p.window_size) == ("fast", 8, 60)
    assert p.ebsynth_config == {"minimum_patch_size": 5, "threads_per_block": 8, "num_iter": 5, "gpu_id": 0,
                                "guide_weight": 10.0, "initialize": "identity", "tracking_window_size": 0}
    with pytest.raises(ValueError, match="inference_mode"):
        FastBlendSmoother(inference_mode="slow")(list(np.zeros((2, 64, 64, 3), np.uint8)))


def test_fast_mode_runner_is_the_smoother(monkeypatch):
    """FastModeRunner and FastBlendSmoother run one fast-mode implementation"""
    from diffsynth.extensions import FastBlend as FB
    from diffsynth.extensions.FastBlend import runners
    assert runners.fast_mode is FB.fast_mode
    calls = []
    fake = lambda *a: calls.append(a) or ["frame"]                       # noqa: E731
    monkeypatch.setattr(runners, "fast_mode", fake)
    monkeypatch.setattr(FB, "fast_mode", fake)
    frames = list(np.zeros((2, 64, 64, 3), np.uint8))
    config = {"tracking_window_size": 0}
    assert runners.FastModeRunner().run(frames, frames, 3, 4, config) == ["frame"]
    assert FB.FastBlendSmoother().run(frames, frames, 3, 4, config) == ["frame"]
    assert calls == [(frames, frames, 3, 4, config)] * 2


# ------------------------------------------------------------------------------------------- C ABI
def _header_names():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))


def test_fastblend_modes_header_is_plain_c():
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        HEADER], capture_output=True, text=True)
    assert r.returncode == 0 and not r.stdout and not r.stderr, r.stdout + r.stderr


@pytest.mark.parametrize("which", ["candidate", "select"])
def test_fastblend_modes_struct_mirrors_match_the_c_layout(tmp_path, which):
    from diffsynth import _native as nv
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    st, cname = {"candidate": (nv.FastblendCandidateDesc, "svi_fastblend_candidate_desc"),
                 "select": (nv.FastblendSelectDesc, "svi_fastblend_select_desc")}[which]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "svi_b200_fastblend_modes.h"', 'int main(void) {',
             f'  printf("sizeof %zu\\n", sizeof({cname}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in st._fields_]
    lines += ['  return 0;', '}']
    (tmp_path / "probe.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(tmp_path / "probe.c"), "-o",
                    str(tmp_path / "probe")], check=True)
    got = dict(line.split() for line in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                                       text=True).stdout.split("\n") if line)
    assert int(got.pop("sizeof")) == ctypes.sizeof(st)
    assert {f: int(v) for f, v in got.items()} == {f: getattr(st, f).offset for f, _ in st._fields_}


def test_fastblend_modes_constants_match_the_header():
    from diffsynth import _native as nv
    defs = dict(re.findall(r"^#define SVI_FASTBLEND_(\w+) (\d+)", open(HEADER).read(), re.M))
    assert int(defs["TRACK"]) == nv.FB_TRACK
    assert nv.FB_TRACK not in (nv.FB_CURRENT, nv.FB_NEIGHBOUR, nv.FB_RANDOM)


def test_every_fastblend_modes_entry_point_is_bound_exported_and_has_a_gpu_case():
    from diffsynth import _native as nv
    import test_fastblend_modes_gpu as gpu
    names = _header_names()
    assert names == {"svi_fastblend_candidate", "svi_fastblend_select", "svi_fastblend_batch_mean",
                     "svi_fastblend_running_mean", "svi_fastblend_to_u8"}
    assert names == set(nv.FASTBLEND_MODES_SIGNATURES)
    assert not names & (set(nv.SIGNATURES) | set(nv.FASTBLEND_SIGNATURES))
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)


# ------------------------------------------------------------------------------------------- refused input
def _frames(n, H=64, W=64):
    return list(np.zeros((n, H, W, 3), np.uint8))


def test_runners_refuse_what_the_reference_would_crash_on_or_drop(monkeypatch):
    emu.install(monkeypatch)
    from diffsynth.extensions.FastBlend import runners
    cfg = _config({})
    with pytest.raises(ValueError, match="at least 2 frames"):
        runners.BalancedModeRunner().run(_frames(1), _frames(1), 8, 2, cfg)
    with pytest.raises(ValueError, match="window_size"):
        runners.BalancedModeRunner().run(_frames(3), _frames(3), 8, 0, cfg)
    interp = runners.InterpolationModeRunner()
    with pytest.raises(ValueError, match="keyframe indices"):
        interp.run(_frames(5), _frames(2), [0, 5], 8, cfg)                  # out of range
    with pytest.raises(ValueError, match="keyframe indices"):
        interp.run(_frames(5), _frames(2), [-1, 3], 8, cfg)
    with pytest.raises(ValueError, match="keyframe indices"):
        interp.run(_frames(5), _frames(2), [1, 1], 8, cfg)                  # not distinct
    with pytest.raises(ValueError, match="2 keyframe indices for 3 keyframes"):
        interp.run(_frames(5), _frames(3), [0, 4], 8, cfg)                  # not matching frames_style
    single = runners.InterpolationModeSingleFrameRunner()
    with pytest.raises(ValueError, match="track_window_size"):
        single.run(_frames(5), _frames(1), [0], 4, _config(dict(tracking_window_size=2)))
    with pytest.raises(ValueError, match="keyframe indices"):
        single.run(_frames(5), _frames(1), [7], 8, cfg)


def test_matcher_accepts_the_three_options_and_still_refuses_random_init(monkeypatch):
    emu.install(monkeypatch)
    from diffsynth.extensions.FastBlend import PyramidPatchMatcher
    m = PyramidPatchMatcher(64, 64, 3, 5, use_mean_target_style=True, use_pairwise_patch_error=True,
                            tracking_window_size=2)
    assert (m.use_mean_target_style, m.use_pairwise_patch_error, m.tracking_window_size) == (True, True, 2)
    x = np.zeros((3, 64, 64, 3), np.uint8)
    with pytest.raises(ValueError, match="odd"):
        m.estimate_nnf(x, x, x)
    with pytest.raises(ValueError, match="initialize"):
        PyramidPatchMatcher(64, 64, 3, 5, initialize="random")
