"""Generate tests/golden/rife_tiny.npz by running the REAL reference RIFE module on the CPU.

Runs only where the reference tree exists; its output is committed and pins oracle/rife_oracle.py to the reference's
behaviour (tests/test_rife_cpu.py).  The reference module (diffsynth/extensions/RIFE/__init__.py, which imports only
torch, numpy and PIL) is loaded by file path; nothing from it is copied into this repository.

usage:  python tests/golden/make_golden_rife.py [--ref /root/reference]
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

H, W = 32, 64


def golden_rife(ref_root):
    from tools import synth_rife as S
    spec = importlib.util.spec_from_file_location("_ref_rife", os.path.join(ref_root, "diffsynth", "extensions", "RIFE",
                                                                            "__init__.py"))
    R = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(R)
    sd = S.make_state_dict(seed=0)
    model = R.IFNet().eval()
    model.load_state_dict(sd, strict=True)
    frames = S.make_frames(4, H, W, seed=0)
    interp = R.RIFEInterpolater(model, device="cpu")
    x = interp.process_images(frames)
    x = torch.cat((x[:-1], x[1:]), 1)                                       # 3 pairs
    out = {"x": x.numpy(), "frames": np.stack([np.asarray(f) for f in frames]), "checksum": np.float64(S.weight_checksum(sd)),
           "seed": np.int64(0)}
    with torch.no_grad():
        for tag, scale in (("s1", 1.0), ("s05", 0.5)):
            flows, mask, merged = model(x, [4 / scale, 2 / scale, 1 / scale])
            out[f"{tag}_flows"] = torch.stack(flows).numpy()
            out[f"{tag}_mask"] = mask.numpy()
            out[f"{tag}_merged"] = torch.stack(merged).numpy()
    out["interp2"] = np.stack([np.asarray(f) for f in interp.interpolate(frames[:3], batch_size=2, num_iter=2)])
    out["smooth"] = np.stack([np.asarray(f) for f in R.RIFESmoother(model, device="cpu")(frames, batch_size=2)])
    np.savez_compressed(os.path.join(HERE, "rife_tiny.npz"), **out)
    print("rife: flows", out["s1_flows"].shape, "interp2", out["interp2"].shape, "smooth", out["smooth"].shape,
          "flow |max| %.2f" % np.abs(out["s1_flows"][2]).max())


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    torch.manual_seed(0)
    golden_rife(a.ref)
