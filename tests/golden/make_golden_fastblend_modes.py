"""Generate tests/golden/fastblend_modes_tiny.npz by running the REAL reference FastBlend runners (balanced, accurate,
keyframe interpolation) on the CPU.

The numpy stand-in for CuPy is tests/golden/make_golden_fastblend.py's, plus what these runners reach beyond the fast
mode: `zeros_like`, and the `pairwise_patch_error` kernel as a literal numpy restatement of its CUDA source (each square
and each addition rounded on its own, as the native kernels do).  The stream counter is reset before each runner call,
and the frames the runners save as PNGs are read back.  Nothing from the reference is copied into this repository; the
committed output pins oracle/fastblend_modes_oracle.py to the reference's host logic (tests/test_fastblend_modes_cpu.py).

usage:  python tests/golden/make_golden_fastblend_modes.py [--ref /root/reference]
"""
import argparse
import importlib
import os
import sys
import tempfile

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_fastblend import ROOT, _w, load_reference  # noqa: E402
from tools.synth_fastblend import digest, make_frames  # noqa: E402

sys.path.insert(0, ROOT)

N, H, W, SEED = 9, 56, 72, 11      # 2 pyramid levels at min patch 5, 1 level at min patch 15
KEYS = [2, 6]                       # a first, a middle and a last segment
CASES = {
    # name: (runner, kwargs of its run(), ebsynth_config)
    "balanced_b3": ("BalancedModeRunner", dict(batch_size=3, window_size=2), dict(minimum_patch_size=5)),
    "balanced_b8": ("BalancedModeRunner", dict(batch_size=8, window_size=2), dict(minimum_patch_size=5)),
    "accurate_t0": ("AccurateModeRunner", dict(batch_size=3, window_size=2), dict(minimum_patch_size=5)),
    "accurate_t1": ("AccurateModeRunner", dict(batch_size=3, window_size=2),
                    dict(minimum_patch_size=5, tracking_window_size=1)),
    "interp_p5_t0": ("InterpolationModeRunner", dict(batch_size=3), dict(minimum_patch_size=5)),
    "interp_p5_t1": ("InterpolationModeRunner", dict(batch_size=3), dict(minimum_patch_size=5, tracking_window_size=1)),
    "interp_p15_t0": ("InterpolationModeRunner", dict(batch_size=3), dict(minimum_patch_size=15)),
    "interp_p15_t1": ("InterpolationModeRunner", dict(batch_size=3), dict(minimum_patch_size=15, tracking_window_size=1)),
    "single_t1_b4": ("InterpolationModeSingleFrameRunner", dict(batch_size=4),
                     dict(minimum_patch_size=5, tracking_window_size=1)),
}
KEEP_WHOLE = ("interp_p5_t1",)      # one case kept whole, to locate a mismatch; the others are pinned by digest


def inputs():
    """(guide frames, style frames): the guide is the synthetic clip, the style a recoloured, brightened copy of it"""
    guide = make_frames(N, H, W, seed=SEED)
    style = make_frames(N, H, W, seed=SEED + 1)[..., ::-1] // 2 + guide // 2
    return list(guide), list(np.ascontiguousarray(style))


def case_inputs(runner, kwargs):
    guide, style = inputs()
    if runner == "InterpolationModeRunner":
        return dict(frames_guide=guide, frames_style=[style[k] for k in KEYS], index_style=list(KEYS), **kwargs)
    if runner == "InterpolationModeSingleFrameRunner":
        return dict(frames_guide=guide, frames_style=[style[4]], index_style=[4], **kwargs)
    return dict(frames_guide=guide, frames_style=style, **kwargs)


def _pairwise_patch_error(height, width, channel, patch_size, pad_size, source_a, nnf_a, source_b, nnf_b, error):
    """pairwise_patch_error: e += (source_a[nnf_a + (px, py)] - source_b[nnf_b + (px, py)])^2, px, py, c order"""
    r = (patch_size - 1) // 2
    B = source_a.shape[0]
    b = np.arange(B).reshape(B, 1, 1)
    na, nb = np.asarray(nnf_a), np.asarray(nnf_b)
    sa, sb = np.asarray(source_a), np.asarray(source_b)
    e = np.zeros((B, height, width), np.float32)
    for px in range(-r, r + 1):
        for py in range(-r, r + 1):
            a = sa[b, na[..., 0] + pad_size + px, na[..., 1] + pad_size + py]
            s = sb[b, nb[..., 0] + pad_size + px, nb[..., 1] + pad_size + py]
            for c in range(channel):
                d = a[..., c] - s[..., c]
                e = e + d * d
    error[...] = e


def load(ref_root):
    ref, cp = load_reference(ref_root)
    cp.zeros_like = lambda *a, **k: _w(np.zeros_like(*a, **k))
    pm = sys.modules["_ref_fastblend.patch_match"]
    pm.pairwise_patch_error_kernel = lambda grid, block, args: _pairwise_patch_error(*args)
    return importlib.import_module("_ref_fastblend.runners"), cp


def golden(ref_root):
    runners, cp = load(ref_root)
    out = {}
    for name, (runner, kwargs, config) in CASES.items():
        ebsynth_config = dict(dict(minimum_patch_size=5, threads_per_block=8, num_iter=5, gpu_id=0, guide_weight=10.0,
                                   initialize="identity", tracking_window_size=0), **config)
        with tempfile.TemporaryDirectory() as d:
            cp.random.k = 0
            getattr(runners, runner)().run(ebsynth_config=ebsynth_config, save_path=d, **case_inputs(runner, kwargs))
            files = sorted(os.listdir(d))
            assert files == ["%05d.png" % i for i in range(N)], files
            frames = np.stack([np.asarray(Image.open(os.path.join(d, f))) for f in files])
        out[f"{name}_sha256"], out[f"{name}_sum"] = digest(frames, np.uint8), np.int64(frames.astype(np.int64).sum())
        out[f"{name}_draws"] = np.int64(cp.random.k)
        if name in KEEP_WHOLE:
            out[name] = frames
        print(name, "draws", int(cp.random.k), "sum", int(out[f"{name}_sum"]))
    np.savez_compressed(os.path.join(HERE, "fastblend_modes_tiny.npz"), **out)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    golden(ap.parse_args().ref)
