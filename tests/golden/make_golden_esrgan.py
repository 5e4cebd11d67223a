"""Generate tests/golden/esrgan_tiny.npz by running the REAL reference ESRGAN module on the CPU.

Runs only where the reference tree exists; its output is committed and pins oracle/esrgan_oracle.py to the reference's
behaviour (tests/test_esrgan_cpu.py).  The reference module (diffsynth/extensions/ESRGAN/__init__.py, which imports only
torch, einops, numpy and PIL) is loaded by file path; nothing from it is copied into this repository.

usage:  python tests/golden/make_golden_esrgan.py [--ref /root/reference]
"""
import argparse
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

SIZES_2 = ((13, 17), (9, 22), (16, 11))     # (H, W) with num_block = 2
SIZE_23 = (10, 12)                          # the default 23-block config
UPSCALE = (3, 13, 17)                       # frames, H, W for ESRGAN.upscale with num_block = 2


def golden_esrgan(ref_root):
    from tools import synth_esrgan as S
    from tools.synth_rife import make_frames
    spec = importlib.util.spec_from_file_location("_ref_esrgan", os.path.join(ref_root, "diffsynth", "extensions", "ESRGAN",
                                                                              "__init__.py"))
    R = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(R)
    out = {}
    for nb in (2, 23):
        sd = S.make_state_dict(nb, seed=0)
        model = R.RRDBNet(num_block=nb).eval()
        model.load_state_dict(sd, strict=True)
        out[f"checksum_nb{nb}"] = np.float64(S.weight_checksum(sd))
        esr = R.ESRGAN(model)
        with torch.no_grad():
            for i, (H, W) in enumerate(SIZES_2 if nb == 2 else (SIZE_23,)):
                x = esr.process_images(make_frames(2, H, W, seed=i))
                out[f"nb{nb}_x{i}"] = x.numpy()
                out[f"nb{nb}_y{i}"] = model(x).numpy()
        if nb == 2:
            F, H, W = UPSCALE
            frames = make_frames(F, H, W, seed=5)
            out["frames"] = np.stack([np.asarray(f) for f in frames])
            out["upscale"] = np.stack([np.asarray(f) for f in esr.upscale(frames, batch_size=2)])
    np.savez_compressed(os.path.join(HERE, "esrgan_tiny.npz"), **out)
    print("esrgan:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    torch.manual_seed(0)
    golden_esrgan(a.ref)
