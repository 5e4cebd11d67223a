"""CPU: unmerged LoRA adapters of the Wan DiT — the C header and its ctypes mirror, key parsing, the stacked layout the
engine hands to svi_gemm_lora_bf16, and the engine's host logic on the torch stand-ins (tests/nv_emulation_lora.py)
against the oracle on fp32-merged weights, including the 2-rank gloo sequence-parallel split."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tools import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "svi_b200_lora.h")
TARGETS = ("self_attn.q", "self_attn.k", "self_attn.v", "self_attn.o", "cross_attn.q", "cross_attn.k", "cross_attn.v",
           "cross_attn.o", "ffn.0", "ffn.2")


def make_lora(cfg, seed, rank=16, targets=TARGETS, blocks=None, prefix="diffusion_model.", name=".default", scale=0.3):
    """A peft LoRA state dict on `targets` of every block (or `blocks`), bf16-representable factors, B A ~ scale * W."""
    shapes = synth.dit_param_shapes(cfg)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i in range(cfg["num_layers"]) if blocks is None else blocks:
        for t in targets:
            out_f, in_f = shapes[f"blocks.{i}.{t}.weight"]
            sd[f"{prefix}blocks.{i}.{t}.lora_A{name}.weight"] = (torch.randn(rank, in_f, generator=g) / in_f ** 0.5).to(torch.bfloat16)
            sd[f"{prefix}blocks.{i}.{t}.lora_B{name}.weight"] = (torch.randn(out_f, rank, generator=g) * scale / rank ** 0.5).to(torch.bfloat16)
    return sd


def merged(sd, loras):
    """fp32 state dict W + sum alpha B A over [(lora state dict, alpha)]: the oracle's weights."""
    out = dict(sd)
    for lsd, alpha in loras:
        for k, v in lsd.items():
            if ".lora_B." not in k:
                continue
            tgt = re.sub(r"^(diffusion_model\.|pipe\.dit\.)", "", k.split(".lora_B.")[0]) + ".weight"
            a = lsd[k.replace(".lora_B.", ".lora_A.")].float()
            out[tgt] = out[tgt] + alpha * (v.float() @ a)
    return out


def _model(cfg, sd):
    from diffsynth.models.wan_video_dit import WanModel
    m = WanModel(**cfg).eval()
    m.load_state_dict(sd)
    return m.to(torch.bfloat16)


def _stats(out, ref):
    err = (out - ref).abs()
    return (err <= 1e-3 + 1e-2 * ref.abs()).float().mean().item(), err.max().item(), err.mean().item() / ref.std().item()


# ------------------------------------------------------------------------------------------- C ABI
def test_lora_header_is_plain_c():
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    r = subprocess.run(["gcc", "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        HEADER], capture_output=True, text=True)
    assert r.returncode == 0 and not r.stdout and not r.stderr, r.stdout + r.stderr


def test_lora_struct_mirror_matches_the_c_layout(tmp_path):
    from diffsynth import _native as nv
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "svi_b200_lora.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(svi_gemm_lora));']
    lines += [f'  printf("{f} %zu\\n", offsetof(svi_gemm_lora, {f}));' for f, _ in nv.GemmLoRA._fields_]
    lines += ['  return 0;', '}']
    (tmp_path / "probe.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(tmp_path / "probe.c"), "-o", str(tmp_path / "probe")],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                                       text=True).stdout.split("\n") if line)
    assert int(got.pop("sizeof")) == ctypes.sizeof(nv.GemmLoRA)
    assert {f: int(v) for f, v in got.items()} == {f: getattr(nv.GemmLoRA, f).offset for f, _ in nv.GemmLoRA._fields_}


def lora_header_entry_points():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))


def test_every_lora_entry_point_is_bound_exported_and_has_a_gpu_case():
    from diffsynth import _native as nv
    import test_lora_adapters_gpu as gpu
    names = lora_header_entry_points()
    assert names == {"svi_gemm_lora_bf16"}
    assert names == set(nv.LORA_SIGNATURES), "include/svi_b200_lora.h and LORA_SIGNATURES disagree"
    assert not names & set(nv.SIGNATURES)
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        for n in names:
            assert hasattr(lib, n), f"{n} is not exported by {os.path.basename(nv.lib_path())}"


# ------------------------------------------------------------------------------------------- parsing
def test_adapter_key_parsing_prefixes_and_errors():
    from diffsynth.models.utils import hash_state_dict_keys
    cfg = synth.CFG_TINY_I2V
    m = _model(cfg, synth.make_dit_state_dict(cfg, seed=0))
    keys_before = hash_state_dict_keys(m.state_dict())
    names_before = [n for n, _ in m.named_parameters()]
    sig = m._param_signature()
    # diffusion_model. prefix + peft adapter name, and plain keys without adapter name
    m.add_lora_adapter("a", make_lora(cfg, 1, rank=8))
    m.add_lora_adapter("b", make_lora(cfg, 2, rank=4, prefix="", name="", targets=("ffn.2",), blocks=[1]))
    assert set(m._lora_adapters["a"][0]) == {(i, t) for i in range(cfg["num_layers"]) for t in TARGETS}
    a, b = m._lora_adapters["b"][0][(1, "ffn.2")]
    assert a.dtype == b.dtype == torch.bfloat16 and tuple(a.shape) == (4, cfg["ffn_dim"]) and tuple(b.shape) == (cfg["dim"], 4)
    # adapters are neither parameters nor buffers: the key set, the parameter list and the engine stamp stay
    assert hash_state_dict_keys(m.state_dict()) == keys_before
    assert [n for n, _ in m.named_parameters()] == names_before and not list(m.buffers())
    assert m._param_signature() == sig
    # unsupported targets and foreign keys point to the merge
    for bad in (make_lora(cfg, 3, targets=("cross_attn.k_img",), blocks=[0]),
                {"diffusion_model.head.head.lora_A.weight": torch.zeros(4, cfg["dim"]),
                 "diffusion_model.head.head.lora_B.weight": torch.zeros(64, 4)},
                dict(make_lora(cfg, 4, blocks=[0], targets=("ffn.0",)), **{"pipe.dwpose_embedding.0.weight": torch.zeros(3)})):
        with pytest.raises(ValueError, match="load_lora_v2"):
            m.add_lora_adapter("bad", bad)
    shape_bad = make_lora(cfg, 5, blocks=[0], targets=("self_attn.q",))
    k = "diffusion_model.blocks.0.self_attn.q.lora_A.default.weight"
    shape_bad[k] = shape_bad[k][:, :128]
    with pytest.raises(ValueError, match=r"blocks\.0\.self_attn\.q.*load_lora_v2"):
        m.add_lora_adapter("bad", shape_bad)
    assert "bad" not in m._lora_adapters
    with pytest.raises(ValueError, match="unknown"):
        m.set_lora_adapters({"nope": 1.0})


# ------------------------------------------------------------------------------------------- stacks
def test_stack_layout_groups_padding_and_alpha_columns(monkeypatch):
    import nv_emulation_lora
    nv_emulation_lora.install(monkeypatch)
    cfg = synth.CFG_TINY_T2V
    d = cfg["dim"]
    m = _model(cfg, synth.make_dit_state_dict(cfg, seed=0))
    la = make_lora(cfg, 1, rank=8)
    lb = make_lora(cfg, 2, rank=16, targets=("self_attn.k", "ffn.0"))
    m.add_lora_adapter("a", la)
    m.add_lora_adapter("b", lb)
    m.set_lora_adapters({"a": 0.7, "b": -0.3})
    eng = m.engine("cpu")
    eng._sync_lora()
    st = eng._lora[0]["qkv"]
    assert st.R == 64 and st.group_cols == d and tuple(st.a.shape) == (3 * 64, d) and tuple(st.b.shape) == (3 * d, 64)
    A = lambda lsd, t, f: lsd[f"diffusion_model.blocks.0.{t}.lora_{f}.default.weight"]
    for g, t in enumerate(("self_attn.q", "self_attn.k", "self_attn.v")):
        assert torch.equal(st.a[g * 64:g * 64 + 8], A(la, t, "A"))                  # adapter a: columns [0, 8) of each group
        assert torch.equal(st.b[g * d:(g + 1) * d, :8], A(la, t, "B"))
        if t == "self_attn.k":                                                        # adapter b: columns [8, 24)
            assert torch.equal(st.a[g * 64 + 8:g * 64 + 24], A(lb, t, "A"))
            assert torch.equal(st.b[g * d:(g + 1) * d, 8:24], A(lb, t, "B"))
        else:                                                                         # b has no q / v: zero rows / columns
            assert not st.a[g * 64 + 8:g * 64 + 24].any() and not st.b[g * d:(g + 1) * d, 8:24].any()
        assert not st.a[g * 64 + 24:(g + 1) * 64].any() and not st.b[g * d:(g + 1) * d, 24:].any()   # padding to 64
        want = torch.zeros(64)
        want[:8], want[8:24] = 0.7, -0.3
        assert torch.equal(st.gate[g * 64:(g + 1) * 64], want)
    assert eng._lora[0]["o"].R == 64 and eng._lora[0]["o"].group_cols == 0 and eng._lora[0]["ckv"].group_cols == d
    assert set(eng._lora[1]) == {"qkv", "o", "cq", "ckv", "co", "f0", "f2"}
    # an alpha change rewrites the gates in place and nothing else; the captured graphs stay
    eng._graphs["sentinel"] = {"graph": None}
    a_ptr, b_ptr, gate = st.a.data_ptr(), st.b.data_ptr(), st.gate
    m.set_lora_adapters({"a": 0.5, "b": 0.25})
    eng._sync_lora()
    st2 = eng._lora[0]["qkv"]
    assert st2 is st and st.a.data_ptr() == a_ptr and st.b.data_ptr() == b_ptr and st.gate is gate
    assert st.gate[:8].eq(0.5).all() and st.gate[8:24].eq(0.25).all() and "sentinel" in eng._graphs
    # a new set rebuilds the stacks and drops the graphs
    m.set_lora_adapters({"b": 1.0})
    eng._sync_lora()
    assert eng._lora[0]["qkv"] is not st and "sentinel" not in eng._graphs and set(eng._lora[0]) == {"qkv", "f0"}
    assert eng._lora[0]["qkv"].R == 64
    m.delete_lora_adapter("b")
    eng._sync_lora()
    assert eng._lora is None and m._lora_active == {}


# ------------------------------------------------------------------------------------------- engine vs oracle
@pytest.mark.parametrize("cfg,f,h,w,seed,n_adapters", [(synth.CFG_TINY_T2V, 3, 8, 12, 0, 1), (synth.CFG_TINY_I2V, 2, 6, 10, 1, 1),
                                                       (synth.CFG_TINY_T2V, 3, 8, 12, 2, 2), (synth.CFG_TINY_I2V, 2, 6, 10, 3, 2)])
def test_engine_with_adapters_matches_oracle_on_merged_weights(monkeypatch, cfg, f, h, w, seed, n_adapters):
    from oracle import wan_dit_oracle as O
    import nv_emulation_lora
    nv_emulation_lora.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    sd = {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=seed).items()}
    m = _model(cfg, sd)
    inp = synth.make_dit_inputs(cfg, f, h, w, seed=seed, ctx_len=24)
    kw = {k: inp[k] for k in ("clip_feature", "y") if k in inp}
    ts = torch.tensor([700.0])
    eng = m.engine("cpu")
    base = eng.forward(inp["x"], ts, inp["context"], **kw).clone()
    loras = [(make_lora(cfg, seed + 10, rank=16), 0.7 if n_adapters == 2 else 1.0)]
    if n_adapters == 2:
        loras.append((make_lora(cfg, seed + 20, rank=8, targets=TARGETS[::2]), -0.3))
    for j, (lsd, _) in enumerate(loras):
        m.add_lora_adapter(f"l{j}", lsd)
    m.set_lora_adapters({f"l{j}": a for j, (_, a) in enumerate(loras)})
    out = eng.forward(inp["x"], ts, inp["context"], **kw)
    ref = O.dit_forward(merged(sd, loras), cfg, inp["x"], ts, inp["context"], kw.get("clip_feature"), kw.get("y"))
    inside, mx, rel = _stats(out, ref)
    assert inside > 0.80 and rel < 4e-3, (inside, mx, rel)
    assert (out - base).abs().mean() > 10 * (out - ref).abs().mean()     # the adapters change the result well above the error
    m.set_lora_adapters({})
    assert torch.equal(eng.forward(inp["x"], ts, inp["context"], **kw), base)


def test_fold_env_takes_the_plain_path_with_adapters(monkeypatch):
    import nv_emulation_lora
    nv_emulation_lora.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    cfg = synth.CFG_TINY_T2V
    sd = {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=0).items()}
    inp = synth.make_dit_inputs(cfg, 3, 16, 24, seed=0, ctx_len=24)
    outs = []
    for fold in ("0", "1"):
        monkeypatch.setenv("SVI_LN_FOLD", fold)
        m = _model(cfg, sd)
        m.add_lora_adapter("a", make_lora(cfg, 1))
        m.set_lora_adapters(["a"])
        eng = m.engine("cpu")
        assert eng.use_fold == (fold == "1")
        outs.append(eng.forward(inp["x"], torch.tensor([500.0]), inp["context"]))
    assert torch.equal(outs[0], outs[1])


def test_context_cache_follows_adapters_and_time_cache_stays(monkeypatch):
    import nv_emulation_lora
    nv_emulation_lora.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    cfg = synth.CFG_TINY_T2V
    m = _model(cfg, synth.make_dit_state_dict(cfg, seed=0))
    m.add_lora_adapter("a", make_lora(cfg, 1))
    eng = m.engine("cpu")
    ctx = synth.make_dit_inputs(cfg, 1, 4, 4, seed=0, ctx_len=24)["context"]
    c0 = eng.context_state(ctx)
    assert eng.context_state(ctx) is c0
    t0 = eng.time_state(torch.tensor([500.0]))
    m.set_lora_adapters({"a": 1.0})
    c1 = eng.context_state(ctx)
    assert c1 is not c0 and not torch.equal(c1.kv_txt_all, c0.kv_txt_all)
    m.set_lora_adapters({"a": 0.5})
    c2 = eng.context_state(ctx)
    assert c2 is not c1 and not torch.equal(c2.kv_txt_all, c1.kv_txt_all)
    assert eng.context_state(ctx) is c2
    assert eng.time_state(torch.tensor([500.0])) is t0
    m.set_lora_adapters(None)
    assert torch.equal(eng.context_state(ctx).kv_txt_all, c0.kv_txt_all)


# ------------------------------------------------------------------------------------------- sequence parallel
def _sp_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      SVI_CUDA_GRAPHS="0")
    import sys
    for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import nv_emulation_lora
    nv_emulation_lora.install()
    from diffsynth.distributed.sequence_parallel import SequenceParallelGroup
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = {}
        for cfg, (f, h, w) in ((synth.CFG_TINY_T2V, (2, 8, 8)), (synth.CFG_TINY_I2V, (2, 4, 12))):
            sd = {k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=0).items()}
            m = _model(cfg, sd)
            m.add_lora_adapter("a", make_lora(cfg, 1))
            m.add_lora_adapter("b", make_lora(cfg, 2, rank=8, targets=("self_attn.k", "self_attn.v")))
            m.set_lora_adapters({"a": 0.7, "b": -0.3})
            eng = m.engine("cpu")
            inp = synth.make_dit_inputs(cfg, f, h, w, seed=0, ctx_len=24)
            kw = {k: inp[k] for k in ("clip_feature", "y") if k in inp}
            ref = eng.forward(inp["x"], 500.0, inp["context"], **kw).clone()
            sp = SequenceParallelGroup(world, rank, cfg_parallel=False)
            out = eng.forward(inp["x"], 500.0, inp["context"], sp=sp, **kw)
            res["i2v" if cfg["has_image_input"] else "t2v"] = (out - ref).abs().max().item()
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_sequence_parallel_two_ranks_with_adapters():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 90)
    procs = [ctx.Process(target=_sp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, res in got:
        assert len(res) == 2, res
        for name, err in res.items():
            assert err < 2e-2, (rank, name, err)


def test_stand_in_takes_the_arguments_of_the_binding():
    """The engine calls gemm_lora with the keyword arguments of gemm (ln / emit included, refused by the library when set):
    the stand-in the CPU tests run must accept exactly what the binding accepts."""
    import inspect
    import nv_emulation_lora
    from diffsynth import _native as nv
    assert list(inspect.signature(nv.gemm_lora).parameters) == list(inspect.signature(nv_emulation_lora.gemm_lora).parameters)
