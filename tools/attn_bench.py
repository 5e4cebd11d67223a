"""The attention launches of the DiT at the bench shape and its neighbours, on one GPU, for A/B runs of kernel builds.

    python tools/attn_bench.py [--lib NAME=PATH ...] [--rounds 5]

Rows (seeded inputs; q, k, v are column slices of one [L, 3 * 1536] q|k|v buffer, as the engine holds them; 12 heads):
    self ws        L = 32760 self-attention with the engine's workspace (the last wave sliced: plan (3036, 7) on 132 SMs)
    self           the same without a workspace (every unit whole)
    self 8192      L = 8192
    cross qscale   attention_qscale, Lq 32760, Lk 512 (the text cross-attention; q's RMS factor in the softmax scale)
    audio 32       Lq 32760, Lk 32 (the SVI-Talk audio cross-attention)

Each build runs in processes of its own (tools/gemm_bench.py's alternating loop).  Per row: median ms over the rounds and
its spread, TFLOP/s (4 Lq Lk d per head), the K/V bytes the CTAs pull from L2 (64 KB per CTA and K/V tile) per second, the
launch plan, and a SHA-256 of the output bytes, so that two builds are compared bit for bit in the same call.  The card's
name, power limit and SM clocks are read in every process.
"""
import argparse
import hashlib
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gemm_bench import ROOT, alternate, card   # noqa: E402

D, H, HD = 1536, 12, 128
ROWS = [("self ws", 32760, 32760), ("self", 32760, 32760), ("self 8192", 8192, 8192), ("cross qscale", 32760, 512),
        ("audio 32", 32760, 32)]


def one_round(iters):
    import torch
    sys.path.insert(0, os.path.join(ROOT, "stable-video-infinity_b200"))
    from diffsynth import _native as nv
    if not torch.cuda.is_available():
        raise SystemExit("attn_bench.py measures on a CUDA device; none is visible")
    dev = "cuda"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"card_before": card()}
    for seed, (name, lq, lk) in enumerate(ROWS):
        g = torch.Generator(device=dev).manual_seed(seed)
        q = torch.randn(lq, 3 * D, generator=g, device=dev).to(torch.bfloat16)[:, :D]
        kv = torch.randn(lk, 3 * D, generator=g, device=dev).to(torch.bfloat16)
        k, v = kv[:, D:2 * D], kv[:, 2 * D:]
        out = torch.zeros(lq, D, device=dev, dtype=torch.bfloat16)
        ws = None
        if name == "self ws":
            ws = torch.empty(nv.attention_workspace_bytes(lq, lk, H), device=dev, dtype=torch.uint8)
        units, n_kv = -(-lq // 128) * H, -(-lk // 128)
        plan = nv.attention_plan(units, n_kv, sms, 0 if ws is None else ws.numel())
        if name == "cross qscale":
            ss = (torch.rand(lq, 1, D // 128, generator=g, device=dev) * 20 + 1)   # partials of q's row sum of squares
            fn = lambda: nv.attention_qscale(q, k, v, out, H, ss, D, 1e-6)
        else:
            fn = lambda: nv.attention(q, k, v, out, H, workspace=ws)
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        digest = hashlib.sha256(out.view(torch.int16).cpu().numpy().tobytes()).hexdigest()[:16]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        res[name] = {"ms": e0.elapsed_time(e1) / iters, "sha256": digest, "plan": list(plan),
                     "kv_bytes": 65536.0 * units * n_kv}
    res["card_after"] = card()
    return res


def summarize(rounds):
    out = {}
    for name, lq, lk in ROWS:
        ts = [r[name]["ms"] for r in rounds]
        t = statistics.median(ts)
        last = rounds[-1][name]
        out[name] = {"Lq": lq, "Lk": lk, "ms": round(t, 4), "spread_ms": round(max(ts) - min(ts), 4),
                     "tflops": round(4.0 * lq * lk * HD * H / t / 1e9, 1),
                     "kv_l2_tbps": round(last["kv_bytes"] / t / 1e9, 2), "plan": last["plan"],
                     "sha256": sorted({r[name]["sha256"] for r in rounds})}
    out["cards"] = sorted({r["card_before"] for r in rounds} | {r["card_after"] for r in rounds})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build of libsvi_b200.so to time (repeatable); default: the tree's build")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--one-round", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.one_round:
        print(json.dumps(one_round(a.iters)))
        return
    rounds = alternate(__file__, a.lib, a.rounds, ["--iters", str(a.iters)])
    builds = {name: summarize(rs) for name, rs in rounds.items()}
    res = {"rounds": a.rounds, "builds": builds}
    if len(builds) > 1:
        res["bit_identical"] = {row: len({json.dumps(b[row]["sha256"]) for b in builds.values()}) == 1
                                for row, _, _ in ROWS}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
