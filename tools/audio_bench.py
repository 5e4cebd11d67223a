"""wav2vec2 audio feature extractor timing on one GPU: base size (conv 512 x 7, 768 x 12 layers), random-init weights, on a
seeded 16 kHz waveform (61 s by default, the length of the reference's talk example).

    python tools/audio_bench.py [--seconds 61] [--no-cpu]

Prints one JSON line: warm milliseconds per extraction from CUDA events, split into the conv stack (feature encoder)
and the encoder (interpolation, projection, positional conv, 12 layers), algorithmic TFLOP/s, launches, the GPU name and
power limit, and the CPU oracle's time for the same input on the host cores (fp32, which is how the reference runs the
extractor, once per clip)."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    sys.path.insert(0, p)
from tools import synth_audio as SA  # noqa: E402


def flops(cfg, n_samples, T):
    """Multiply-adds x 2 of every product, from the shapes."""
    f, t, cin = 0, n_samples, 1
    for cd, k, s in zip(cfg["conv_dim"], cfg["conv_kernel"], cfg["conv_stride"]):
        t = (t - k) // s + 1
        f += 2 * t * cd * k * cin
        cin = cd
    conv = f
    d, L, ff = cfg["hidden_size"], cfg["num_hidden_layers"], cfg["intermediate_size"]
    proj = 2 * T * cin * d
    pos = 2 * T * d * (d // cfg["num_conv_pos_embedding_groups"]) * cfg["num_conv_pos_embeddings"]
    gemm = L * (2 * T * d * 3 * d + 2 * T * d * d + 2 * 2 * T * d * ff)
    attn = L * 4 * T * T * d
    return {"conv": conv, "proj": proj, "pos_conv": pos, "encoder_gemm": gemm, "attention": attn}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=61.0)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "audio_bench needs a GPU"
    from diffsynth.models.wav2vec2 import Wav2Vec2Model
    from oracle import wav2vec2_oracle as O
    cfg = SA.BASE
    sd = {k: v.to(torch.bfloat16).float() for k, v in SA.make_state_dict(cfg, seed=0).items()}
    m = Wav2Vec2Model(cfg).eval()
    m.load_state_dict(sd)
    speech = SA.make_waveform(a.seconds, seed=0)
    iv = torch.from_numpy(O.normalize(speech)).cuda()
    T = O.seq_len_for(len(speech))
    eng = m.engine("cuda")
    feats = eng.features(iv)
    eng.encode(feats, T)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    conv_ms, enc_ms = [], []
    l0 = eng.launches
    for _ in range(a.iters):
        ev[0].record()
        feats = eng.features(iv)
        ev[1].record()
        eng.encode(feats, T)
        ev[2].record()
        torch.cuda.synchronize()
        conv_ms.append(ev[0].elapsed_time(ev[1]))
        enc_ms.append(ev[1].elapsed_time(ev[2]))
    launches = (eng.launches - l0) // a.iters
    fl = flops(cfg, len(speech), T)
    total = sum(fl.values())
    conv, enc = sorted(conv_ms)[len(conv_ms) // 2], sorted(enc_ms)[len(enc_ms) // 2]
    res = {"seconds_of_audio": a.seconds, "T_frames": T, "conv_frames": int(feats.shape[0]), "ms": conv + enc,
           "conv_stack_ms": conv, "encoder_ms": enc, "ms_all_iters": [c + e for c, e in zip(conv_ms, enc_ms)],
           "algorithmic_gflop": {k: v / 1e9 for k, v in fl.items()}, "tflops": total / (conv + enc) / 1e9,
           "conv_stack_tflops": fl["conv"] / conv / 1e9, "encoder_tflops": (total - fl["conv"]) / enc / 1e9,
           "launches": launches}
    res.update(gpu_info())
    if not a.no_cpu:
        torch.set_num_threads(os.cpu_count())
        t0 = time.perf_counter()
        O.embedding(sd, cfg, speech)
        res["cpu_oracle"] = {"cores": os.cpu_count(), "s": time.perf_counter() - t0, "dtype": "fp32"}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
