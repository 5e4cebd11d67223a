"""CPU: the ESRGAN bf16 rounding study (DESIGN.md §4).  Replays the fp32 oracle with bf16 rounding at exactly the native
engine's storage points (every conv input and weight; residual streams and epilogues f32), the same with the input image
kept exact (the two-term hi | lo operand of conv_first), and with only the input image rounded, against plain fp32.
tools/synth_esrgan.py weights (23 blocks), tools/synth_rife.py frames.

Per row: mean and max |d| of the output as a fraction of the fp32 output's std, and for the uint8 frames the mean |d| in
grey levels and the share within +-2 levels.

usage:  python tools/esrgan_rounding_study.py [--sizes 48x64,72x96] [--seeds 0,1]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import esrgan_oracle as O  # noqa: E402
from tools import synth_esrgan as S  # noqa: E402
from tools.synth_rife import make_frames  # noqa: E402


def bf16(t):
    return t.to(torch.bfloat16).float()


def compare(ref, got):
    d = (got - ref).abs()
    u = np.abs(O.to_uint8(got).astype(int) - O.to_uint8(ref).astype(int))
    return {"mean_rel_std": d.mean().item() / ref.std().item(), "max_rel_std": d.max().item() / ref.std().item(),
            "u8_mean": float(u.mean()), "u8_within2": float((u <= 2).mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="48x64,72x96")
    ap.add_argument("--seeds", default="0,1")
    ap.add_argument("--frames", type=int, default=2)
    a = ap.parse_args()
    for seed in [int(s) for s in a.seeds.split(",")]:
        sd = S.make_state_dict(23, seed=seed)
        for size in a.sizes.split(","):
            H, W = (int(v) for v in size.split("x"))
            x = O.to_tensor(np.stack([np.asarray(f) for f in make_frames(a.frames, H, W, seed=seed)]))
            with torch.no_grad():
                ref = O.rrdbnet(sd, x)
                full = O.rrdbnet(sd, x, rnd=bf16)
                hilo = O.rrdbnet(sd, x, rnd=bf16, rnd_first=O._ident)
                inp = O.rrdbnet(sd, x, rnd_first=bf16)
            print(json.dumps({"seed": seed, "size": f"{W}x{H}", "out_mean": round(ref.mean().item(), 4),
                              "out_std": round(ref.std().item(), 4),
                              "bf16_storage": {k: round(v, 6) for k, v in compare(ref, full).items()},
                              "bf16_storage_hilo_input": {k: round(v, 6) for k, v in compare(ref, hilo).items()},
                              "input_only": {k: round(v, 6) for k, v in compare(ref, inp).items()}}), flush=True)


if __name__ == "__main__":
    main()
