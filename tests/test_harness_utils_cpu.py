"""CPU: the host helpers the SVI-Talk and SVI-Dance scripts import (utils.video_process, utils.image_process,
utils.project_utils) against the reference's own helpers, recorded in tests/golden/harness_utils_tiny.npz by
tests/golden/make_golden_harness_utils.py; the names the scripts take from the three star imports; and
utils.video_process importing without imageio or matplotlib."""
import builtins
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "harness_utils_tiny.npz"))
PKG = os.path.join(os.path.dirname(HERE), "stable-video-infinity_b200")


def _cases(prefix):
    return sorted({k[len(prefix):].rsplit(".", 1)[0] for k in GOLD.files if k.startswith(prefix) and k.endswith(".in")})


def _generator():
    spec = importlib.util.spec_from_file_location("_make_golden_harness_utils",
                                                  os.path.join(HERE, "golden", "make_golden_harness_utils.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _same_image(im, key):
    assert im.mode == str(GOLD[key + ".mode"])
    want = GOLD[key + ".out"]
    got = np.array(im)
    assert got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("case", _cases("resize."))
def test_resize_and_pad_to_target_matches_reference(case):
    from utils.image_process import resize_and_pad_to_target
    k = "resize." + case
    x = torch.from_numpy(GOLD[k + ".in"])
    got = resize_and_pad_to_target(x, tuple(int(v) for v in GOLD[k + ".target"]), pad_value=int(GOLD[k + ".pad"]))
    want = GOLD[k + ".out"]
    assert got.dtype == x.dtype and got.shape == want.shape
    assert got.numpy().tobytes() == want.tobytes()


@pytest.mark.parametrize("case", _cases("tensor2pil."))
def test_tensor2pil_matches_reference(case):
    from utils.image_process import tensor2pil
    k = "tensor2pil." + case
    x = GOLD[k + ".in"]
    if case.startswith("pil_"):
        mode = case[len("pil_"):]
        x = Image.fromarray(x.squeeze(-1) if mode == "L" else x, mode)
    else:
        x = torch.from_numpy(x)
    if k + ".raises" in GOLD.files:
        with pytest.raises(getattr(builtins, str(GOLD[k + ".raises"]))):
            tensor2pil(x)
    else:
        _same_image(tensor2pil(x), k)


def test_tensor2pil_rejects_other_inputs():
    from utils.image_process import tensor2pil
    for k, bad in (("tensor2pil.ndarray", np.zeros((3, 4, 4), np.uint8)), ("tensor2pil.list", [1, 2])):
        assert str(GOLD[k + ".raises"]) == "TypeError"
        with pytest.raises(TypeError):
            tensor2pil(bad)


@pytest.mark.parametrize("case", ["equal", "taller", "shorter"])
def test_image_compose_width_matches_reference(case):
    from utils.video_process import image_compose_width
    k = "compose." + case
    a, b = GOLD[k + ".in0"], GOLD[k + ".in1"]
    out = image_compose_width(Image.fromarray(a), Image.fromarray(b))
    assert out.mode == "RGB" and out.size == (a.shape[1] + b.shape[1], a.shape[0])
    got, want = np.array(out), GOLD[k + ".out"]
    assert got.shape == want.shape and got.tobytes() == want.tobytes()


class _Recorder:
    """Stands in for imageio: keeps the arguments of get_writer and the frames handed to append_data."""

    def __init__(self):
        self.calls = []

    def get_writer(self, path, **kw):
        frames, rec = [], self

        class W:
            def append_data(self, frame):
                frames.append(np.array(frame, copy=True))

            def close(self):
                rec.calls.append((path, kw, frames))
        return W()


@pytest.mark.parametrize("case", _cases("dwpose."))
def test_save_dwpose_as_mp4_matches_reference(case, monkeypatch):
    import utils.video_process as VP
    rec = _Recorder()
    monkeypatch.setattr(VP, "imageio", rec)
    k = "dwpose." + case
    x = GOLD[k + ".in"]
    if case == "u8.norm0":
        VP.save_dwpose_as_mp4(torch.from_numpy(x), "pose.mp4", normalize=False)
        kw = dict(fps=30, quality=9, ffmpeg_params=None)
    else:
        VP.save_dwpose_as_mp4(torch.from_numpy(x) if case.endswith(".torch") else x, "pose.mp4", fps=12, quality=7,
                              normalize=".norm1." in case, ffmpeg_params=["-crf", "18"])
        kw = dict(fps=12, quality=7, ffmpeg_params=["-crf", "18"])
    (path, got_kw, frames), = rec.calls
    assert path == "pose.mp4" and got_kw == kw
    got, want = np.stack(frames), GOLD[k + ".out"]
    assert got.dtype == np.uint8 and got.shape == want.shape and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("case", _cases("save_image."))
def test_save_tensor_as_image_matches_reference(case, tmp_path):
    from utils.image_process import save_tensor_as_image
    k = "save_image." + case
    path = str(tmp_path / "out.png")
    kw = {"auto_detect_channels": False} if case == "hw.noauto" else {}
    save_tensor_as_image(torch.from_numpy(GOLD[k + ".in"]), path, **kw)
    if k + ".none" in GOLD.files:
        assert not os.path.exists(path)
    else:
        _same_image(Image.open(path), k)


def test_normalized_round_trip_matches_reference():
    from utils.image_process import from_normalized, to_normalized
    x = GOLD["normalized.in"]
    assert to_normalized(x).tobytes() == GOLD["normalized.to"].tobytes()
    assert from_normalized(x).tobytes() == GOLD["normalized.from"].tobytes()
    t = torch.from_numpy(x)
    assert torch.equal(to_normalized(t), torch.from_numpy(GOLD["normalized.to"]))


def test_update_experiment_path_matches_reference(tmp_path):
    from utils.project_utils import update_experiment_path
    gen = _generator()
    for i, case in enumerate(gen.EXPERIMENT_CASES):
        args, short = gen.experiment_args(case, str(tmp_path))
        assert update_experiment_path(args, short=short) is args
        assert os.path.relpath(args.output_path, str(tmp_path)) == str(GOLD[f"experiment_path.{i}.out"])
        assert os.path.isdir(args.output_path)


def test_resize_and_pad_keeps_the_pose_video_dtype():
    """the dance script's use: a uint8 [N, 3, h, w] pose video fitted to the clip size, then [3, N, H, W]"""
    from utils.image_process import resize_and_pad_to_target
    pose = torch.randint(0, 256, (5, 3, 30, 20), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    out = resize_and_pad_to_target(pose, (64, 96), pad_value=0).permute(1, 0, 2, 3)
    assert out.dtype == torch.uint8 and out.shape == (3, 5, 64, 96)
    # scale min(64/30, 96/20) = 2.133 -> 64 x 42, centred: 27 columns left, 27 right
    assert out[..., :27].eq(0).all() and out[..., 27 + 42:].eq(0).all() and out[..., 27:27 + 42].ne(0).any()


def test_star_imports_give_the_scripts_their_names():
    ns = {}
    exec("from utils.video_process import *\nfrom utils.image_process import *\nfrom utils.project_utils import *", ns)
    for name in ("image_compose_width", "tensor2pil", "resize_and_pad_to_target", "calculate_dimensions",
                 "find_reference_image", "print_args", "update_experiment_path", "save_dwpose_as_mp4",
                 "tensor_to_pil", "imageio"):
        assert name in ns, name
    try:
        import imageio
    except ImportError:
        return
    assert ns["imageio"] is imageio


_NO_OPTIONAL = """
import sys
for m in ("imageio", "matplotlib", "matplotlib.pyplot", "cv2"):
    sys.modules[m] = None                       # any import of them raises ImportError
import numpy as np
import utils.video_process as VP
from utils.video_process import image_compose_width
try:
    VP.save_dwpose_as_mp4(np.zeros((4, 3, 2, 2), np.float32), "never.mp4")
except ImportError as e:
    assert "imageio" in str(e), e
    print("ImportError:", e)
else:
    raise SystemExit("save_dwpose_as_mp4 ran without imageio")
try:
    VP.imageio.get_reader("pose.mp4")
except ImportError as e:
    assert "imageio" in str(e), e
else:
    raise SystemExit("imageio.get_reader ran without imageio")
"""


def test_video_process_imports_without_imageio_matplotlib_or_cv2():
    env = dict(os.environ, PYTHONPATH=PKG + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", _NO_OPTIONAL], env=env, capture_output=True, text=True, cwd=HERE)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "ImportError:" in r.stdout and not os.path.exists(os.path.join(HERE, "never.mp4"))
