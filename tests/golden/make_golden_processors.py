"""Generate tests/golden/processors_tiny.npz by running the REAL reference video processors on the CPU.

Runs only where the reference tree exists; its output is committed and pins oracle/processors_oracle.py to the
reference's behaviour (tests/test_processors_cpu.py).  The reference's diffsynth/processors modules (base, PILEditor,
RIFE, sequencial_processor: torch, numpy and PIL only) and its extensions/RIFE IFNet are loaded by file path; nothing
from them is copied into this repository.

  - rife_interp / rife_avg: processors/RIFE.py RIFESmoother(interpolate=True / False, batch_size=2) on the tiny IFNet
    weights and the four 32x64 frames of rife_tiny.npz;
  - chain: SequencialProcessor.from_model_manager over [Contrast 1.7, Sharpness 2.3] on five small random frames.

usage:  python tests/golden/make_golden_processors.py --ref <reference checkout>
"""
import argparse
import importlib.util
import os
import sys
import types

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

H, W = 32, 64
CHAIN_CONFIGS = [{"processor_type": "Contrast", "config": {"rate": 1.7}},
                 {"processor_type": "Sharpness", "config": {"rate": 2.3}}]


def chain_frames():
    rng = np.random.default_rng(5)
    return rng.integers(0, 256, (5, 23, 37, 3), dtype=np.uint8)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def reference_processors(ref_root):
    """the reference's processors package, without its __init__ (which is empty) or FastBlend (which needs CuPy)"""
    pkg = types.ModuleType("_ref_processors")
    pkg.__path__ = [os.path.join(ref_root, "diffsynth", "processors")]
    sys.modules["_ref_processors"] = pkg
    mods = {}
    for m in ("base", "PILEditor", "RIFE", "sequencial_processor"):
        mods[m] = _load(f"_ref_processors.{m}", os.path.join(pkg.__path__[0], f"{m}.py"))
    return mods


def golden_processors(ref_root):
    from tools import synth_rife as S
    P = reference_processors(ref_root)
    R = _load("_ref_rife", os.path.join(ref_root, "diffsynth", "extensions", "RIFE", "__init__.py"))
    sd = S.make_state_dict(seed=0)
    model = R.IFNet().eval()
    model.load_state_dict(sd, strict=True)
    frames = S.make_frames(4, H, W, seed=0)
    out = {"frames": np.stack([np.asarray(f) for f in frames]), "checksum": np.float64(S.weight_checksum(sd))}
    for tag, interpolate in (("rife_interp", True), ("rife_avg", False)):
        smoother = P["RIFE"].RIFESmoother(model, device="cpu", batch_size=2, interpolate=interpolate)
        out[tag] = np.stack([np.asarray(f) for f in smoother(frames)])
    cf = chain_frames()
    chain = P["sequencial_processor"].SequencialProcessor.from_model_manager(None, CHAIN_CONFIGS)
    out["chain_frames"] = cf
    out["chain"] = np.stack([np.asarray(f) for f in chain([Image.fromarray(f) for f in cf])])
    np.savez_compressed(os.path.join(HERE, "processors_tiny.npz"), **out)
    print("processors: rife", out["rife_interp"].shape, "inner frames changed by the average:",
          int((out["rife_avg"][1:-1] != out["frames"][1:-1]).sum()), "chain", out["chain"].shape)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="a checkout of the reference repository")
    a = ap.parse_args()
    torch.manual_seed(0)
    golden_processors(a.ref)
