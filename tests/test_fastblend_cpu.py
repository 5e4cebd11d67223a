"""CPU: FastBlend deflickering — the oracle against the reference's golden outputs bit for bit (PatchMatch at levels that
divide exactly and at one that does not, both batch sizes, the tables, the whole fast mode), the box filter against cv2,
the random stream's pinned values, the C header and its ctypes mirrors, and the engine's host logic on the torch
stand-ins (tests/nv_emulation_fastblend.py) against the oracle, with every rejected option."""
import ctypes
import os
import re
import shutil
import subprocess

import cv2
import numpy as np
import pytest
import torch

import nv_emulation_fastblend as emu
from oracle import fastblend_oracle as O
from tools.synth_fastblend import digest, make_frames, nnf_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "svi_b200_fastblend.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "fastblend_tiny.npz")
CASES = [("a", 8), ("a", 3), ("b", 8), ("b", 3)]       # a: 64x96 (levels divide exactly), b: 57x83 (they do not)
SIZES = {"a": (64, 96), "b": (57, 83)}                  # the inputs of tests/golden/make_golden_fastblend.py


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _t(x):
    return torch.from_numpy(np.asarray(x, np.float32))


def _inputs(tag, B):
    return nnf_inputs(*SIZES[tag], B, seed=B)


def _run_frames():
    return make_frames(9, 56, 72, seed=11)


def _check_estimate(golden, tag, B, nnf, ts):
    """bit-for-bit against the reference: the digests of the field (int32) and of target_style (f32); the statistics
    and the whole batch-3 fields only locate a mismatch"""
    if f"{tag}{B}_nnf" in golden.files:
        assert np.array_equal(nnf, golden[f"{tag}{B}_nnf"].astype(np.int32))
    assert digest(nnf, np.int32) == str(golden[f"{tag}{B}_nnf_sha256"])
    assert digest(ts, np.float32) == str(golden[f"{tag}{B}_ts_sha256"]), (
        f"target_style sum {ts.astype(np.float64).sum()!r} max {ts.max()!r}, reference "
        f"{float(golden[f'{tag}{B}_ts_sum'])!r} {float(golden[f'{tag}{B}_ts_max'])!r}")


# ------------------------------------------------------------------------------------------- oracle vs reference
@pytest.mark.parametrize("tag,B", CASES)
def test_oracle_estimate_nnf_matches_reference_bitwise(golden, tag, B):
    H, W = SIZES[tag]
    sg, tg, ss = _inputs(tag, B)
    m = O.PyramidPatchMatcher(H, W)
    nnf, ts = m.estimate_nnf(_t(sg), _t(tg), _t(ss))
    _check_estimate(golden, tag, B, nnf.numpy(), ts.numpy())
    assert m.draws == int(golden[f"{tag}{B}_draws"])


def test_oracle_tables_match_reference(golden):
    for n in (1, 2, 5, 9, 16, 17):
        got = np.array([[t["source"], t["target"], t["level"]] for t in O.task_list(n)], np.int64).reshape(-1, 3)
        assert np.array_equal(got, golden[f"tasks{n}"]), n
    got = [O.tree_query(int(l), int(r)) for l, r in golden["tree_lr"]]
    assert np.array_equal([len(g) for g in got], golden["tree_nodes"])
    assert np.array_equal([v for g in got for node in g for v in node], golden["tree_flat"])


@pytest.mark.parametrize("B", [8, 3])
def test_oracle_run_matches_reference_bytes(golden, B):
    frames = list(_run_frames())
    out = O.run(frames, frames, batch_size=B, window_size=4)
    if B == 3:
        assert np.array_equal(out, golden["run3"])
    assert digest(out, np.uint8) == str(golden[f"run{B}_sha256"])


def test_batch_size_changes_the_reference_output(golden):
    """the odd-index-below-batch +1 of the NNF upscale is live: batch 3 and batch 8 differ"""
    assert int(golden["run_differ"]) > 0 and str(golden["run8_sha256"]) != str(golden["run3_sha256"])


@pytest.mark.parametrize("k", [2, 4, 8, 16])
def test_box_filter_is_cv2_inter_area(k):
    rng = np.random.default_rng(k)
    img = (rng.random((480, 832, 3)) * 255).astype(np.float32)
    want = cv2.resize(img, (832 // k, 480 // k), interpolation=cv2.INTER_AREA)
    got = O.box_down(torch.from_numpy(img)[None], k)[0].numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_resample_takes_cv2_off_integer_ratios():
    img = (np.random.default_rng(0).random((1, 57, 83, 3)) * 255).astype(np.float32)
    assert O.integer_ratio(57, 83, 28, 41) is None and O.integer_ratio(480, 832, 30, 52) == 16
    want = cv2.resize(img[0], (41, 28), interpolation=cv2.INTER_AREA)
    assert np.array_equal(O.resample(torch.from_numpy(img), 28, 41)[0].numpy(), want)


# ------------------------------------------------------------------------------------------- the random stream
PINNED_U = {(0, 0): 2926543089, (0, 1): 2692512407, (1, 0): 2385989600, (7, 12345): 939238334,
            (4096, 2 ** 31 + 5): 3052316619}
PINNED_PERM = [[1, 2, 3, 0], [1, 2, 0, 3], [0, 1, 3, 2], [3, 1, 0, 2], [0, 2, 3, 1], [2, 1, 3, 0], [0, 1, 3, 2],
               [2, 3, 1, 0], [3, 2, 1, 0], [1, 2, 0, 3], [2, 0, 1, 3], [2, 3, 1, 0], [1, 0, 3, 2], [3, 1, 2, 0],
               [3, 0, 2, 1], [1, 0, 3, 2], [3, 1, 0, 2], [2, 0, 3, 1], [1, 2, 0, 3], [1, 2, 0, 3], [2, 3, 0, 1],
               [3, 1, 2, 0], [1, 0, 3, 2], [2, 0, 3, 1]]


def test_stream_pinned_values():
    from diffsynth.extensions import FastBlend as FB
    for (k, i), v in PINNED_U.items():
        assert int(O.stream_u(k, i)) == v and FB.stream_u(k, i) == v
    assert [O.permutation4(k) for k in range(24)] == PINNED_PERM
    m = FB.PyramidPatchMatcher(64, 96, 3, 5)
    assert [m._permutation4() for _ in range(24)] == PINNED_PERM
    assert O.randint(3, -4, 5, (2, 2)).tolist() == [[-4 + int(O.stream_u(3, i)) % 9 for i in (0, 1)],
                                                    [-4 + int(O.stream_u(3, i)) % 9 for i in (2, 3)]]


# ------------------------------------------------------------------------------------------- C ABI
def _header_names():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))


def test_fastblend_header_is_plain_c():
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        HEADER], capture_output=True, text=True)
    assert r.returncode == 0 and not r.stdout and not r.stderr, r.stdout + r.stderr


@pytest.mark.parametrize("which", ["step", "table"])
def test_fastblend_struct_mirrors_match_the_c_layout(tmp_path, which):
    from diffsynth import _native as nv
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    st, cname = {"step": (nv.FastblendStepDesc, "svi_fastblend_step_desc"),
                 "table": (nv.FastblendTableDesc, "svi_fastblend_table_desc")}[which]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "svi_b200_fastblend.h"', 'int main(void) {',
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


def test_fastblend_constants_match_the_header():
    from diffsynth import _native as nv
    from diffsynth.extensions import FastBlend as FB
    defs = dict(re.findall(r"^#define SVI_FASTBLEND_(\w+) (\d+)", open(HEADER).read(), re.M))
    assert int(defs["MAX_PATCH"]) == FB.MAX_PATCH
    assert (int(defs["CURRENT"]), int(defs["NEIGHBOUR"]), int(defs["RANDOM"])) == (nv.FB_CURRENT, nv.FB_NEIGHBOUR, nv.FB_RANDOM)
    assert (int(defs["U8"]), int(defs["F32"]), int(defs["F64"])) == (nv.FB_U8, nv.FB_F32, nv.FB_F64)
    assert (int(defs["MEAN"]), int(defs["HALF"]), int(defs["WSUM"])) == (nv.FB_MEAN, nv.FB_HALF, nv.FB_WSUM)


def test_every_fastblend_entry_point_is_bound_exported_and_has_a_gpu_case():
    from diffsynth import _native as nv
    import test_fastblend_gpu as gpu
    names = _header_names()
    assert names == {"svi_fastblend_stage_frames", "svi_fastblend_downsample", "svi_fastblend_nnf_identity",
                     "svi_fastblend_nnf_upscale", "svi_fastblend_remap", "svi_fastblend_step", "svi_fastblend_table"}
    assert names == set(nv.FASTBLEND_SIGNATURES), "include/svi_b200_fastblend.h and FASTBLEND_SIGNATURES disagree"
    assert not names & (set(nv.SIGNATURES) | set(nv.LORA_SIGNATURES) | set(nv.RIFE_SIGNATURES) | set(nv.ESRGAN_SIGNATURES))
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)


# ------------------------------------------------------------------------------------------- the engine on stand-ins
@pytest.mark.parametrize("tag,B", [("a", 8), ("b", 3)])
def test_engine_estimate_nnf_matches_oracle(monkeypatch, golden, tag, B):
    emu.install(monkeypatch)
    from diffsynth.extensions.FastBlend import PyramidPatchMatcher
    H, W = SIZES[tag]
    m = PyramidPatchMatcher(H, W, 3, 5)
    nnf, ts = m.estimate_nnf(*_inputs(tag, B))
    assert nnf.dtype == np.int32 and ts.dtype == np.float32 and ts.shape == (B, H, W, 3)
    _check_estimate(golden, tag, B, nnf, ts)
    assert m.draws == int(golden[f"{tag}{B}_draws"])


@pytest.mark.slow
def test_engine_smoother_matches_reference_bytes_and_self_guides(monkeypatch, golden):
    emu.install(monkeypatch)
    from PIL import Image
    from diffsynth.extensions.FastBlend import FastBlendSmoother
    frames = [Image.fromarray(f) for f in _run_frames()]
    s = FastBlendSmoother.from_model_manager(None)
    s.window_size, s.batch_size = 4, 3
    out = s(frames)
    assert all(isinstance(f, Image.Image) for f in out)
    assert np.array_equal(np.stack([np.asarray(f) for f in out]), golden["run3"])
    guided = s(frames, original_frames=[f.copy() for f in frames])
    assert np.array_equal(np.stack([np.asarray(f) for f in guided]), golden["run3"])


def test_smoother_defaults_are_the_reference_config():
    from diffsynth.extensions.FastBlend import FastBlendSmoother
    s = FastBlendSmoother()
    assert (s.batch_size, s.window_size) == (8, 64)
    assert s.ebsynth_config == {"minimum_patch_size": 5, "threads_per_block": 8, "num_iter": 5, "gpu_id": 0,
                                "guide_weight": 10.0, "initialize": "identity", "tracking_window_size": 0}


@pytest.mark.parametrize("option,value", [("use_mean_target_style", True), ("use_pairwise_patch_error", True),
                                          ("tracking_window_size", 2), ("initialize", "random")])
def test_rejected_options_raise_through_the_smoother(monkeypatch, option, value):
    emu.install(monkeypatch)
    from diffsynth.extensions.FastBlend import FastBlendSmoother
    s = FastBlendSmoother()
    s.ebsynth_config = dict(s.ebsynth_config, **{option: value})
    frames = list(np.zeros((2, 64, 64, 3), np.uint8))
    with pytest.raises(ValueError, match=option):
        s(frames)


def test_too_small_frames_and_too_large_batches_raise(monkeypatch):
    emu.install(monkeypatch)
    from diffsynth.extensions.FastBlend import FastBlendSmoother, PyramidPatchMatcher
    with pytest.raises(ValueError, match="too small"):
        FastBlendSmoother()(list(np.zeros((2, 25, 64, 3), np.uint8)))            # min side < 2 x 13
    m = PyramidPatchMatcher(52, 52, 3, 5)                                        # levels 26x26, 52x52
    x = np.zeros((54, 52, 52, 3), np.uint8)                                      # odd index 53 >= 52
    with pytest.raises(ValueError, match="batch_size 54"):
        m.estimate_nnf(x, x, x)
    m.check_batch(53)                                                            # largest odd index 51: fine
    s = FastBlendSmoother()
    s.batch_size = 54
    with pytest.raises(ValueError, match="batch_size 54"):
        s(list(np.zeros((60, 52, 52, 3), np.uint8)))
