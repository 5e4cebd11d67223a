"""The DiT block's GEMMs with the epilogues the block gives them, next to the bare GEMM at the same shape, on one GPU.

    python tools/gemm_bench.py [--lib NAME=PATH ...] [--rounds 5]

Rows (M = 32760 tokens, the bench shape of Wan2.1-T2V-1.3B: d = 1536, ffn = 8960), each with the arguments
WanDiTEngine._block passes:
    qkv      N 4608  K 1536  bias + partial row sums of squares (q, k) -> bf16
    o        N 1536  K 1536  bias + gate + fp32 residual, in place
    cross q  N 1536  K 1536  bias + partial row sums -> bf16 columns [0, d) of the [M, 3d] qkv buffer
    cross o  N 1536  K 1536  bias + fp32 residual, in place
    ffn.0    N 8960  K 1536  bias + GELU-tanh -> bf16
    ffn.2    N 1536  K 8960  bias + gate + fp32 residual, in place
and the bare GEMM (bf16 out, no epilogue) at the four distinct shapes; every row in both weight formats (bf16 and e4m3).
The epilogue cost of a row is its time minus the bare time at its shape.

The library is picked when diffsynth._native is imported, so every --lib (default: the tree's build) runs in processes of
its own: one process per build and round, the builds alternating, the order flipped every round.  Each process warms
every case up, times it with CUDA events over --iters launches, and reads the card's name, power limit and SM clocks in
the same process.  Prints one JSON object: per build, per row the median over the rounds.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L, D, F = 32760, 1536, 8960
SHAPES = {"qkv": (3 * D, D), "o": (D, D), "ffn.0": (F, D), "ffn.2": (D, F)}   # bare GEMM shapes (N, K)
ROWS = [("qkv", "qkv"), ("o", "o"), ("cross q", "o"), ("cross o", "o"), ("ffn.0", "ffn.0"), ("ffn.2", "ffn.2")]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def one_round(iters):
    """Times every case once in this process (the library SVI_B200_LIB names, or the tree's)."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, "stable-video-infinity_b200"))
    from diffsynth import _native as nv
    if not torch.cuda.is_available():
        raise SystemExit("gemm_bench.py measures on a CUDA device; none is visible")
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s, sc=1.0: torch.randn(*s, generator=g, device=dev) * sc
    h, hf = rnd(L, D).to(torch.bfloat16), rnd(L, F).to(torch.bfloat16)
    x = rnd(L, D)
    gate2, gate5 = rnd(D, sc=0.05), rnd(D, sc=0.05)
    W = {k: rnd(n, kk, sc=kk ** -0.5).to(torch.bfloat16) for k, (n, kk) in SHAPES.items()}
    W["cross"] = rnd(D, D, sc=D ** -0.5).to(torch.bfloat16)
    W["cross o"] = rnd(D, D, sc=D ** -0.5).to(torch.bfloat16)
    W8 = {k: w.to(torch.float8_e4m3fn) for k, w in W.items()}
    b = {n: rnd(n, sc=0.1) for n in (3 * D, D, F)}
    qkv = torch.empty(L, 3 * D, device=dev, dtype=torch.bfloat16)
    ffn = torch.empty(L, F, device=dev, dtype=torch.bfloat16)
    P = D // 128
    ss = torch.empty(L, 2, P, device=dev)
    ss1 = torch.empty(L, 1, P, device=dev)
    bare_out = {k: torch.empty(L, n, device=dev, dtype=torch.bfloat16) for k, (n, _) in SHAPES.items()}

    def cases(ws):
        c = {}
        for k in SHAPES:
            a = hf if k == "ffn.2" else h
            c["bare " + k] = (lambda a=a, w=ws[k], o=bare_out[k]: nv.gemm(a, w, o))
        c["qkv"] = lambda: nv.gemm(h, ws["qkv"], qkv, bias=b[3 * D], sumsq=ss, sumsq_group_cols=D)
        c["o"] = lambda: nv.gemm(h, ws["o"], x, bias=b[D], gate=gate2, residual=x)
        c["cross q"] = lambda: nv.gemm(h, ws["cross"], qkv[:, :D], bias=b[D], sumsq=ss1, sumsq_group_cols=D)
        c["cross o"] = lambda: nv.gemm(h, ws["cross o"], x, bias=b[D], residual=x)
        c["ffn.0"] = lambda: nv.gemm(h, ws["ffn.0"], ffn, bias=b[F], act=nv.ACT_GELU_TANH)
        c["ffn.2"] = lambda: nv.gemm(hf, ws["ffn.2"], x, bias=b[D], gate=gate5, residual=x)
        return c

    res = {"card_before": card()}
    for fmt, ws in (("bf16", W), ("e4m3", W8)):
        for name, fn in cases(ws).items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            e1.synchronize()
            res[f"{fmt} {name}"] = e0.elapsed_time(e1) / iters
    res["card_after"] = card()
    return res


def summarize(rounds):
    out = {}
    for fmt in ("bf16", "e4m3"):
        rows = {}
        med = lambda key: statistics.median(r[f"{fmt} {key}"] for r in rounds)
        spread = lambda key: max(r[f"{fmt} {key}"] for r in rounds) - min(r[f"{fmt} {key}"] for r in rounds)
        for k, (n, kk) in SHAPES.items():
            t = med("bare " + k)
            rows["bare " + k] = {"N": n, "K": kk, "ms": round(t, 4), "spread_ms": round(spread("bare " + k), 4),
                                 "tflops": round(2.0 * L * n * kk / t / 1e9, 1)}
        for row, shape in ROWS:
            n, kk = SHAPES[shape]
            t, tb = med(row), med("bare " + shape)
            rows[row] = {"N": n, "K": kk, "ms": round(t, 4), "spread_ms": round(spread(row), 4),
                         "tflops": round(2.0 * L * n * kk / t / 1e9, 1), "epilogue_ms": round(t - tb, 4),
                         "over_bare": round(t / tb, 3)}
        out[fmt] = rows
    out["cards"] = sorted({r["card_before"] for r in rounds} | {r["card_after"] for r in rounds})
    return out


def alternate(script, lib_args, rounds, args):
    """Runs `script --one-round ARGS` once per build (--lib NAME=PATH, default the tree's) and round, the builds alternating
    and the order flipped every round; returns {name: [the JSON each round printed last]}."""
    libs = [s.split("=", 1) for s in lib_args] or [["tree", ""]]
    out = {name: [] for name, _ in libs}
    for r in range(rounds):
        for name, path in (libs if r % 2 == 0 else libs[::-1]):
            env = dict(os.environ)
            if path:
                env["SVI_B200_LIB"] = os.path.abspath(path)
            p = subprocess.run([sys.executable, os.path.abspath(script), "--one-round", *args],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"{os.path.basename(script)}: the {name} round failed:\n{p.stderr[-3000:]}")
            out[name].append(json.loads(p.stdout.strip().splitlines()[-1]))
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
    res = {"M": L, "rounds": a.rounds, "builds": {name: summarize(rs) for name, rs in rounds.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
