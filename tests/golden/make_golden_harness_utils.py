"""Generate tests/golden/harness_utils_tiny.npz by running the REAL reference helpers of utils/image_process.py,
utils/video_process.py and utils/project_utils.py on the CPU.

Runs only where the reference tree exists; its output is committed and pins stable-video-infinity_b200/utils to the
reference's behaviour (tests/test_harness_utils_cpu.py).  The reference modules are loaded by file path with
`matplotlib` stubbed (imported, never used) and `imageio` replaced by a recorder whose writer keeps the uint8 frames
handed to `append_data` and the `get_writer` arguments; nothing from them is copied into this repository.

Every case stores its inputs (`<case>.in*`) next to the reference's output (`<case>.out`, or `<case>.raises` holding
the exception's type name), so the test needs nothing but this file.

usage:  python tests/golden/make_golden_harness_utils.py --ref <reference checkout>
"""
import argparse
import contextlib
import importlib.util
import io
import os
import sys
import tempfile
import types

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))

# resize_and_pad_to_target: (input [B,3,h,w], target (th, tw)); the scales min(th/h, tw/w) are not integers, and the
# cases include up- and downscaling with the odd pixel of padding on either axis
RESIZE_CASES = [((2, 3, 7, 11), (16, 24)), ((1, 3, 13, 5), (32, 16)), ((1, 3, 21, 30), (9, 10)),
                ((2, 3, 24, 18), (20, 30)), ((1, 3, 5, 9), (26, 22))]
# save_dwpose_as_mp4: input shapes (dim 0 == 3 is read as [C,T,H,W])
DWPOSE_SHAPES = [(3, 4, 6, 5), (4, 1, 6, 5), (4, 2, 6, 5), (4, 3, 6, 5), (4, 4, 6, 5), (2, 5, 3, 4)]
# save_tensor_as_image: shapes whose channel axis is first, middle, last, single, or ambiguous
IMAGE_SHAPES = [(3, 9, 7), (9, 7, 3), (1, 9, 7), (9, 1, 7), (4, 3, 5), (9, 7, 4)]
# update_experiment_path: (train_architecture, short, exp_prefix, pretrained_lora_path)
EXPERIMENT_CASES = [("lora", False, "", None), ("lora", True, "run", "x.pt"), ("full", False, "exp", "x.pt"),
                    ("full", True, None, "")]


def experiment_args(case, output_path):
    arch, short, prefix, pretrained = case
    return types.SimpleNamespace(train_architecture=arch, lora_rank=32, pose_cfg=0.5, mouth_cfg=1.5, pose_relax=True,
                                 pose_relax_num=3, exp_prefix=prefix, pretrained_lora_path=pretrained,
                                 output_path=output_path), short


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


class _Writer:
    def __init__(self, log, path, **kw):
        self.frames = []
        log.append((path, kw, self.frames))

    def append_data(self, frame):
        self.frames.append(np.array(frame, copy=True))

    def close(self):
        pass


def reference_utils(ref_root, writers):
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    iio = types.ModuleType("imageio")
    iio.get_writer = lambda path, **kw: _Writer(writers, path, **kw)
    sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": mpl.pyplot, "imageio": iio})
    try:
        import cv2  # noqa: F401
    except ImportError:                                    # imported, never used by the helpers recorded here
        sys.modules["cv2"] = types.ModuleType("cv2")
    d = os.path.join(ref_root, "utils")
    return (_load("_ref_image_process", os.path.join(d, "image_process.py")),
            _load("_ref_video_process", os.path.join(d, "video_process.py")),
            _load("_ref_project_utils", os.path.join(d, "project_utils.py")))


def _call(out, key, fn, *a, **kw):
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            res = fn(*a, **kw)
    except Exception as e:  # noqa: BLE001
        out[key + ".raises"] = np.array(type(e).__name__)
        return None
    return res


def _pil(im):
    return np.array(im), np.array(im.mode)


def golden(ref_root):
    writers = []
    IP, VP, PU = reference_utils(ref_root, writers)
    rng = np.random.default_rng(0)
    out = {}

    for i, (shape, target) in enumerate(RESIZE_CASES):
        u8 = rng.integers(0, 256, shape, dtype=np.uint8)
        f32 = rng.standard_normal(shape).astype(np.float32)
        for kind, x in (("u8", u8), ("f32", f32)):
            for pad in (0, 7):
                k = f"resize.{i}.{kind}.pad{pad}"
                out[k + ".in"] = x
                out[k + ".target"] = np.array(target)
                out[k + ".pad"] = np.array(pad)
                out[k + ".out"] = IP.resize_and_pad_to_target(torch.from_numpy(x), target, pad_value=pad).numpy()

    t2p = {
        "chw3_u8": rng.integers(0, 256, (3, 6, 5), dtype=np.uint8),
        "chw3_f32": rng.uniform(-0.5, 1.5, (3, 6, 5)).astype(np.float32),
        "hwc3_u8": rng.integers(0, 256, (6, 5, 3), dtype=np.uint8),
        "hwc3_f32": rng.uniform(-0.5, 1.5, (6, 5, 3)).astype(np.float32),
        "hwc3_f64": rng.uniform(-0.5, 1.5, (6, 5, 3)),
        "chw1_u8": rng.integers(0, 256, (1, 6, 5), dtype=np.uint8),
        "chw1_f32": rng.uniform(-0.5, 1.5, (1, 6, 5)).astype(np.float32),
        "hwc1_f32": rng.uniform(-0.5, 1.5, (6, 5, 1)).astype(np.float32),
        "hw_u8": rng.integers(0, 256, (6, 5), dtype=np.uint8),
        "hw_f32": rng.uniform(-0.5, 1.5, (6, 5)).astype(np.float32),
        "hwc3_pose_u8": rng.integers(0, 256, (3, 3, 3), dtype=np.uint8),   # H == 3: read as CHW
    }
    for name, x in t2p.items():
        k = f"tensor2pil.{name}"
        out[k + ".in"] = x
        im = _call(out, k, IP.tensor2pil, torch.from_numpy(x))
        if im is not None:
            out[k + ".out"], out[k + ".mode"] = _pil(im)
    for mode in ("RGBA", "L", "RGB"):
        k = f"tensor2pil.pil_{mode}"
        src = rng.integers(0, 256, (6, 5, len(mode)), dtype=np.uint8)
        out[k + ".in"] = src
        out[k + ".out"], out[k + ".mode"] = _pil(IP.tensor2pil(Image.fromarray(src.squeeze(-1) if mode == "L" else src, mode)))
    for k, bad in (("tensor2pil.ndarray", np.zeros((3, 4, 4), np.uint8)), ("tensor2pil.list", [1, 2])):
        _call(out, k, IP.tensor2pil, bad)

    for name, (h0, w0, h1, w1) in {"equal": (8, 6, 8, 5), "taller": (8, 6, 11, 4), "shorter": (8, 6, 5, 7)}.items():
        k = f"compose.{name}"
        a = rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
        b = rng.integers(0, 256, (h1, w1, 3), dtype=np.uint8)
        out[k + ".in0"], out[k + ".in1"] = a, b
        out[k + ".out"], _ = _pil(VP.image_compose_width(Image.fromarray(a), Image.fromarray(b)))

    for shape in DWPOSE_SHAPES:
        for normalize in (True, False):
            for src in ("torch", "numpy"):
                k = f"dwpose.{'x'.join(map(str, shape))}.norm{int(normalize)}.{src}"
                x = rng.uniform(-2.0, 3.0, shape).astype(np.float32) if normalize else rng.uniform(0, 1, shape).astype(np.float32)
                out[k + ".in"] = x
                del writers[:]
                with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                    VP.save_dwpose_as_mp4(torch.from_numpy(x) if src == "torch" else x, "pose.mp4", fps=12, quality=7,
                                          normalize=normalize, ffmpeg_params=["-crf", "18"])
                (path, kw, frames), = writers
                assert path == "pose.mp4" and kw == dict(fps=12, quality=7, ffmpeg_params=["-crf", "18"]), kw
                out[k + ".out"] = np.stack(frames)
    k = "dwpose.u8.norm0"                                 # uint8 data multiplied by 255 without normalising wraps
    out[k + ".in"] = rng.integers(0, 256, (4, 3, 6, 5), dtype=np.uint8)
    del writers[:]
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        VP.save_dwpose_as_mp4(torch.from_numpy(out[k + ".in"]), "pose.mp4", normalize=False)
    assert writers[0][1] == dict(fps=30, quality=9, ffmpeg_params=None), writers[0][1]
    out[k + ".out"] = np.stack(writers[0][2])

    with tempfile.TemporaryDirectory() as tmp:
        for i, shape in enumerate(IMAGE_SHAPES):
            for kind in ("f32", "u8", "const"):
                k = f"save_image.{i}.{kind}"
                x = {"f32": lambda: rng.standard_normal(shape).astype(np.float32),
                     "u8": lambda: rng.integers(0, 256, shape, dtype=np.uint8),
                     "const": lambda: np.full(shape, 0.5, np.float32)}[kind]()
                out[k + ".in"] = x
                path = os.path.join(tmp, f"{i}_{kind}.png")
                _call(out, k, IP.save_tensor_as_image, torch.from_numpy(x), path)
                if k + ".raises" not in out:
                    if os.path.exists(path):
                        out[k + ".out"], out[k + ".mode"] = _pil(Image.open(path))
                    else:
                        out[k + ".none"] = np.array(True)
        k = "save_image.hw.noauto"
        out[k + ".in"] = rng.standard_normal((9, 7)).astype(np.float32)
        path = os.path.join(tmp, "noauto.png")
        _call(out, k, IP.save_tensor_as_image, torch.from_numpy(out[k + ".in"]), path, auto_detect_channels=False)
        out[k + ".out"], out[k + ".mode"] = _pil(Image.open(path))

        x = rng.uniform(-10, 300, (4, 5)).astype(np.float32)
        out["normalized.in"] = x
        out["normalized.to"] = IP.to_normalized(x)
        out["normalized.from"] = IP.from_normalized(x)

        for i, case in enumerate(EXPERIMENT_CASES):
            args, short = experiment_args(case, tmp)
            with contextlib.redirect_stdout(io.StringIO()):
                res = PU.update_experiment_path(args, short=short)
            assert res is args and os.path.isdir(args.output_path)
            out[f"experiment_path.{i}.out"] = np.array(os.path.relpath(args.output_path, tmp))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="reference checkout")
    ap.add_argument("--out", default=os.path.join(HERE, "harness_utils_tiny.npz"))
    a = ap.parse_args()
    torch.manual_seed(0)
    out = golden(a.ref)
    np.savez_compressed(a.out, **out)
    print(f"wrote {a.out}: {len(out)} arrays")


if __name__ == "__main__":
    main()
