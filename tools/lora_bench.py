"""Cost of unmerged LoRA adapters on one GPU (svi_gemm_lora_bf16 + the down-projection GEMM in front of it), with the
card's name, power limit and SM clocks.  The variants of each comparison run alternately, round after round, and the
median per variant is reported.

    python tools/lora_bench.py [--sections gemm,step13,step14,switch] [--rounds 3]

gemm   : the block GEMMs of the 1.3B model at the bench's M = 32760 rows, plain vs a rank-128 segment plus its U GEMM,
         bf16 and e4m3 weights
step13 : the 1.3B model's CFG pair (two forwards, CUDA graphs) at the bench shape with 0, 1 and 2 rank-128 adapters
step14 : the 14B-I2V model's CFG pair at 480p (81 frames) with 0 and 1 rank-128 adapter, bf16 and e4m3 weights
switch : set_lora_adapters on the 1.3B model, then the first forward (eager) and the graph capture + replay after it
The algorithmic extra work of the adapters is 4 L R (6 d + ffn) FLOP per block and forward (``extra_flop_share``)."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
from tools import synth  # noqa: E402

E4M3 = torch.float8_e4m3fn
R = 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return q


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def alternate(variants, rounds, reps):
    """{name: median ms} of callables run alternately (forward order on even rounds, reversed on odd ones)."""
    times = {k: [] for k in variants}
    names = list(variants)
    for r in range(rounds):
        for k in names if r % 2 == 0 else names[::-1]:
            times[k].append(timed(variants[k], reps))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def extra_flop_share(cfg, L, n_txt):
    """extra FLOP of rank-R adapters on the ten block projections over the forward's algorithmic FLOP (oracle formula)."""
    from tools.flops import dit_forward_flops
    d, ffn = cfg["dim"], cfg["ffn_dim"]
    extra = cfg["num_layers"] * 4 * L * R * (6 * d + ffn)
    return extra / dit_forward_flops(cfg, L, n_txt), extra


def sec_gemm(rounds):
    from diffsynth import _native as nv
    d, ffn, M = 1536, 8960, 32760
    g = torch.Generator(device="cuda").manual_seed(0)
    h = torch.randn(M, d, device="cuda", generator=g).to(torch.bfloat16)
    hf = torch.randn(M, ffn, device="cuda", generator=g).to(torch.bfloat16)
    x = torch.randn(M, d, device="cuda", generator=g)
    gate = torch.ones(d, device="cuda")
    rows = []
    for name, a, N, groups, kw_of in (
            ("qkv", h, 3 * d, 3, lambda o: dict(bias=torch.zeros(3 * d, device="cuda"))),
            ("o", h, d, 1, lambda o: dict(bias=torch.zeros(d, device="cuda"), gate=gate, residual=o)),
            ("ffn.0", h, ffn, 1, lambda o: dict(bias=torch.zeros(ffn, device="cuda"), act=nv.ACT_GELU_TANH)),
            ("ffn.2", hf, d, 1, lambda o: dict(bias=torch.zeros(d, device="cuda"), gate=gate, residual=o))):
        K = a.shape[1]
        f32_out = name in ("o", "ffn.2")
        out = x if f32_out else torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        la = (torch.randn(groups * R, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
        lb = (torch.randn(N, R, device="cuda", generator=g) * 0.01).to(torch.bfloat16)
        lg = torch.ones(groups * R, device="cuda")
        u = torch.empty(M, groups * R, device="cuda", dtype=torch.bfloat16)
        for wdt in (torch.bfloat16, E4M3):
            w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(wdt)
            kw = kw_of(out)

            def plain():
                nv.gemm(a, w, out, **kw)

            def lora():
                nv.gemm(a, la, u, gate=lg)
                nv.gemm_lora(a, w, out, u, lb, R, N // groups if groups > 1 else 0, **kw)

            def seg_only():
                nv.gemm_lora(a, w, out, u, lb, R, N // groups if groups > 1 else 0, **kw)
            for f in (plain, lora, seg_only):
                f()
            t = alternate({"plain": plain, "lora": lora, "segment": seg_only}, rounds, 10)
            rows.append(dict(section="gemm", gemm=name, M=M, N=N, K=K, R=R, w="e4m3" if wdt == E4M3 else "bf16",
                             plain_ms=round(t["plain"], 4), with_lora_ms=round(t["lora"], 4),
                             segment_only_ms=round(t["segment"], 4), u_gemm_ms=round(t["lora"] - t["segment"], 4),
                             extra_pct=round(100 * (t["lora"] / t["plain"] - 1), 2),
                             extra_flop_pct=round(100 * R * (groups * K + N) / (K * N), 2)))
    return rows


def build_model(cfg, dtype):
    from diffsynth.models.wan_video_dit import WanModel, precompute_freqs_cis_3d
    with torch.device("meta"):
        m = WanModel(**cfg).to(torch.bfloat16)
    m.to_empty(device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if p.dim() >= 2 and "modulation" not in name:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * (1.0 / p[0].numel() ** 0.5)).to(p.dtype))
            elif name.endswith("bias"):
                p.zero_()
            elif "modulation" in name:
                p.copy_((torch.randn(p.shape, generator=g, device="cuda") * 0.02).to(p.dtype))
            else:
                p.fill_(1.0)
    m.freqs = precompute_freqs_cis_3d(cfg["dim"] // cfg["num_heads"])
    if dtype == E4M3:
        m.to(dtype=E4M3)
    return m.eval()


def cfg_pair(m, cfg, f, h, w):
    eng = m.engine("cuda")
    inp = synth.make_dit_inputs(cfg, f, h, w, seed=0, ctx_len=512)
    x = inp["x"].cuda().float()
    kw = {}
    clip = inp["clip_feature"].cuda() if "clip_feature" in inp else None
    if "y" in inp:
        kw["y"] = inp["y"].cuda()
    ctx_p, ctx_n = inp["context"].cuda(), torch.randn(inp["context"].shape, generator=torch.Generator().manual_seed(2)).cuda()
    v_c, v_u = torch.empty_like(x), torch.empty_like(x)

    def step():
        cp, cn = eng.context_state(ctx_p, clip), eng.context_state(ctx_n, clip)
        eng.forward(x, 500.0, cp, out=v_c, **kw)
        eng.forward(x, 500.0, cn, out=v_u, **kw)
    return step, f * (h // 2) * (w // 2)


def sec_step(cfg, f, h, w, dtypes, sets, rounds, tag):
    from test_lora_adapters_cpu import make_lora
    rows = []
    for dt in dtypes:
        m = build_model(cfg, dt)
        adapters = {}
        for j in range(max(len(s) for s in sets.values())):
            name = f"a{j}"
            m.add_lora_adapter(name, make_lora(cfg, j, rank=R, scale=0.05))
            adapters[name] = 1.0
        step, L = cfg_pair(m, cfg, f, h, w)
        times = {k: [] for k in sets}
        for r in range(rounds):
            for k in (list(sets) if r % 2 == 0 else list(sets)[::-1]):
                m.set_lora_adapters({n: 1.0 for n in sets[k]})
                for _ in range(3):                       # eager, capture, one replay
                    step()
                torch.cuda.synchronize()
                times[k].append(timed(step, 3))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        base = med[list(sets)[0]]
        share, extra = extra_flop_share(cfg, L, 512)
        rows.append(dict(section=tag, L=L, w="e4m3" if dt == E4M3 else "bf16", R=R,
                         ms_per_cfg_pair={k: round(v, 2) for k, v in med.items()},
                         extra_pct={k: round(100 * (v / base - 1), 2) for k, v in med.items()},
                         extra_flop_per_adapter_pct=round(100 * share, 2),
                         extra_gflop_per_forward_per_adapter=round(extra / 1e9, 1)))
        del m, step
        torch.cuda.empty_cache()
    return rows


def sec_switch(rounds):
    from test_lora_adapters_cpu import make_lora
    cfg = synth.CFG_T2V_1_3B
    m = build_model(cfg, torch.bfloat16)
    m.add_lora_adapter("shot", make_lora(cfg, 0, rank=R, scale=0.05))
    m.add_lora_adapter("film", make_lora(cfg, 1, rank=R, scale=0.05))
    eng = m.engine("cuda")
    inp = synth.make_dit_inputs(cfg, 21, 60, 104, seed=0, ctx_len=512)
    x, ctx = inp["x"].cuda().float(), inp["context"].cuda()
    out = torch.empty_like(x)
    rows = []
    for r in range(rounds):
        for name in ("shot", "film"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.set_lora_adapters({name: 1.0})
            cp = eng.context_state(ctx)
            eng.forward(x, 500.0, cp, out=out)                   # stacks built, context K|V projected, eager forward
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            eng.forward(x, 500.0, cp, out=out)                   # capture + replay
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            eng.forward(x, 500.0, cp, out=out)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            rows.append(dict(section="switch", to=name, set_and_first_forward_ms=round(1e3 * (t1 - t0), 1),
                             capture_ms=round(1e3 * (t2 - t1), 1), replay_ms=round(1e3 * (t3 - t2), 1)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", default="gemm,step13,step14,switch")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench: needs a CUDA device")
    print(json.dumps(dict(card=card())), flush=True)
    secs = a.sections.split(",")
    runs = {"gemm": lambda: sec_gemm(a.rounds),
            "step13": lambda: sec_step(synth.CFG_T2V_1_3B, 21, 60, 104, (torch.bfloat16,),
                                       {"0": [], "1": ["a0"], "2": ["a0", "a1"]}, a.rounds, "step13"),
            "step14": lambda: sec_step(synth.CFG_I2V_14B, 21, 60, 104, (torch.bfloat16, E4M3), {"0": [], "1": ["a0"]},
                                       a.rounds, "step14"),
            "switch": lambda: sec_switch(a.rounds)}
    for sec in secs:
        for r in runs[sec]():
            print(json.dumps(r), flush=True)
    print(json.dumps(dict(card_after=card())), flush=True)


if __name__ == "__main__":
    main()
