"""CPU: e4m3 (float8_e4m3fn) model weights — the reference's weight-only FP8 mode — on the host side of the engines, with the
kernels replaced by the torch stand-ins of tests/nv_emulation.py.  A model cast to e4m3 must give the same engine outputs as
its bf16(e4m3(p)) twin, its engine must hold the GEMM matrices as e4m3 (about half the bytes), and the gemm binding must
refuse the formats the kernel does not take.  The kernel's bit-identity is checked on the GPU (test_fp8_weights_gpu.py)."""
import pytest
import torch

from tools import synth
from tools import synth_enc as SE

E4M3 = torch.float8_e4m3fn

DIT_BLOCK_MATS = ("w_qkv", "w_o", "w_cq", "w_ckv", "w_co", "w_f0", "w_f2")
DIT_ENGINE_MATS = ("w_patch", "w_te0", "w_te2", "w_t0", "w_t2", "w_tp", "w_head")
TEXT_MATS = ("w_qkv", "w_o", "w_gate", "w_fc1", "w_fc2")


def weight_bytes(*holders):
    """Bytes of the distinct tensor storages held as attributes (or dict values / tuple items) of the given objects."""
    seen, total = set(), 0

    def add(t):
        nonlocal total
        if isinstance(t, torch.Tensor):
            st = t.untyped_storage()
            if st.data_ptr() not in seen:
                seen.add(st.data_ptr())
                total += st.nbytes()
        elif isinstance(t, tuple):
            for x in t:
                add(x)

    for h in holders:
        for v in (h.values() if isinstance(h, dict) else vars(h).values()):
            add(v)
    return total


def dit_engine_bytes(eng):
    return weight_bytes(eng, *eng.blocks)


def _dit_pair(cfg, seed):
    from diffsynth.models.wan_video_dit import WanModel
    sd = synth.make_dit_state_dict(cfg, seed=seed)
    m8 = WanModel(**cfg).eval()
    m8.load_state_dict(sd)
    m8 = m8.to(E4M3)
    twin = WanModel(**cfg).eval()
    twin.load_state_dict({k: v.to(E4M3).to(torch.bfloat16) for k, v in sd.items()})
    twin = twin.to(torch.bfloat16)
    return m8, twin


@pytest.mark.parametrize("cfg,fold", [(synth.CFG_TINY_T2V, "0"), (synth.CFG_TINY_I2V, "0"), (synth.CFG_TINY_TALK, "0"),
                                      (synth.CFG_TINY_I2V, "1")])
def test_dit_engine_on_e4m3_weights_matches_upcast_twin(monkeypatch, cfg, fold):
    import nv_emulation
    nv_emulation.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    monkeypatch.setenv("SVI_LN_FOLD", fold)
    m8, twin = _dit_pair(cfg, seed=4)
    f, h, w = (3, 8, 8) if cfg.get("enable_multitalk") else (2, 20, 28)     # > 128 rows: the fold path engages
    inp = synth.make_dit_inputs(cfg, f, h, w, seed=4, ctx_len=24)
    kw = {k: inp[k] for k in ("clip_feature", "y") if k in inp}
    if cfg.get("enable_multitalk"):
        from diffsynth.pipelines.svi_video_talk import preprocess_audio
        kw["audio"] = preprocess_audio(synth.make_audio_embed(4 * (f - 1) + 1, seed=4).to(torch.bfloat16).float())
    e8, eb = m8.engine("cpu"), twin.engine("cpu")
    for name in DIT_BLOCK_MATS + (("w_ckv_img",) if cfg["has_image_input"] else ()) + \
            (("w_aq", "w_akv", "w_ap") if cfg.get("enable_multitalk") else ()):
        assert getattr(e8.blocks[0], name).dtype == E4M3, name
        assert torch.equal(getattr(e8.blocks[0], name).to(torch.bfloat16), getattr(eb.blocks[0], name)), name
    assert e8.blocks[1].w_q.dtype == E4M3 and e8.blocks[1].w_kv.dtype == E4M3          # sequence-parallel views
    for name in DIT_ENGINE_MATS + (("ie_w1", "ie_w3") if cfg["has_image_input"] else ()) + \
            (("ap_w1", "ap_w1v", "ap_w2", "ap_w3") if cfg.get("enable_multitalk") else ()):
        assert getattr(e8, name).dtype == E4M3, name
    assert e8.blocks[0].b_qkv.dtype == torch.float32 and e8.mod_table.dtype == torch.float32          # vectors: f32
    for ts in (700.0, 300.0):
        out8 = e8.forward(inp["x"], torch.tensor([ts]), inp["context"], **kw)
        outb = eb.forward(inp["x"], torch.tensor([ts]), inp["context"], **kw)
        assert torch.equal(out8, outb), (out8 - outb).abs().max()


@pytest.mark.parametrize("cfg", [synth.CFG_TINY_T2V, synth.CFG_TINY_I2V, synth.CFG_TINY_TALK])
def test_dit_engine_weight_bytes_halve(monkeypatch, cfg):
    import nv_emulation
    nv_emulation.install(monkeypatch)
    m8, twin = _dit_pair(cfg, seed=0)
    b8, bb = dit_engine_bytes(m8.engine("cpu")), dit_engine_bytes(twin.engine("cpu"))
    assert b8 <= 0.52 * bb, (b8, bb, b8 / bb)


def test_matrix_with_k_not_multiple_of_16_is_upcast():
    from diffsynth.models.wan_video_dit import _mat
    w = torch.randn(32, 40).to(E4M3)
    assert _mat(w, "cpu").dtype == torch.bfloat16 and torch.equal(_mat(w, "cpu"), w.to(torch.bfloat16))
    assert _mat(torch.randn(32, 48).to(E4M3), "cpu").dtype == E4M3
    assert _mat(torch.randn(32, 48), "cpu").dtype == torch.bfloat16


def _text_pair(cfg, seed):
    from diffsynth.models.wan_video_text_encoder import WanTextEncoder
    sd = SE.make_text_state_dict(cfg, seed=seed)
    m8 = WanTextEncoder(**cfg).eval()
    m8.load_state_dict(sd)
    m8 = m8.to(E4M3)
    twin = WanTextEncoder(**cfg).eval()
    twin.load_state_dict({k: v.to(E4M3).to(torch.bfloat16) for k, v in sd.items()})
    return m8, twin.to(torch.bfloat16)


def _install_text_standins(monkeypatch):
    """Torch stand-ins of the umT5 engine's non-GEMM kernels (both engines under comparison run the same ones)."""
    from diffsynth import _native as nv

    def embedding_gather(ids, table, out):
        return out.copy_(table[ids].float())

    def rmsnorm_affine(x, weight, eps, out):
        return out.copy_((x * torch.rsqrt(x.pow(2).mean(1, keepdim=True) + eps) * weight).to(out.dtype))

    def mul_bf16(a, b, out):
        return out.copy_(a.float() * b.float())

    def attention_small(q, k, v, out, num_heads, head_dim, scale, bias_table=None, bucket=None, key_mask=None):
        qf, kf, vf = (t.float().reshape(t.shape[0], num_heads, head_dim).transpose(0, 1) for t in (q, k, v))
        s = qf @ kf.transpose(1, 2) * scale
        if bias_table is not None:
            s = s + bias_table[bucket.long()].permute(2, 0, 1)
        if key_mask is not None:
            s = s.masked_fill(key_mask.view(1, 1, -1) == 0, float("-inf"))
        return out.copy_((torch.softmax(s, -1) @ vf).transpose(0, 1).reshape(out.shape))

    for name, fn in (("embedding_gather", embedding_gather), ("rmsnorm_affine", rmsnorm_affine), ("mul_bf16", mul_bf16),
                     ("attention_small", attention_small)):
        monkeypatch.setattr(nv, name, fn)


def test_text_engine_on_e4m3_weights_matches_upcast_twin(monkeypatch):
    import nv_emulation
    from diffsynth.models.wan_video_text_encoder import WanTextEncoderEngine
    nv_emulation.install(monkeypatch)
    _install_text_standins(monkeypatch)
    cfg = SE.TEXT_TINY
    m8, twin = _text_pair(cfg, seed=2)
    e8, eb = WanTextEncoderEngine(m8, "cpu"), WanTextEncoderEngine(twin, "cpu")
    for ly in e8.layers:
        for name in TEXT_MATS:
            assert ly[name].dtype == E4M3, name
    assert e8.table.dtype == torch.bfloat16 and torch.equal(e8.table, eb.table)
    ids, mask = SE.make_text_inputs(cfg, seq_len=24, valid=17, seed=2)
    assert torch.equal(e8.forward(ids, mask), eb.forward(ids, mask))
    # the module hands the prompter bf16, not e4m3-rounded embeddings (weight-only FP8 computes in bf16)
    out8 = m8(ids, mask)
    assert out8.dtype == torch.bfloat16 and torch.equal(out8, twin(ids, mask))
    # the umT5 engine keeps the embedding table in bf16 (the gather reads bf16); the tiny vocabulary keeps it small
    b8 = weight_bytes(e8, *e8.layers)
    bb = weight_bytes(eb, *eb.layers)
    assert b8 <= 0.52 * bb, (b8, bb, b8 / bb)


def test_gemm_binding_refuses_unsupported_formats():
    from diffsynth import _native as nv
    a = torch.zeros(4, 32, dtype=torch.bfloat16)
    out = torch.zeros(4, 16, dtype=torch.float32)
    with pytest.raises(RuntimeError, match="bf16 or float8_e4m3fn"):
        nv.gemm(a, torch.zeros(16, 32, dtype=torch.float8_e5m2), out)
    with pytest.raises(RuntimeError, match="a must be bf16"):
        nv.gemm(a.to(E4M3), torch.zeros(16, 32, dtype=E4M3), out)
    with pytest.raises(RuntimeError, match="multiples of 16"):
        nv.gemm(torch.zeros(4, 40, dtype=torch.bfloat16), torch.zeros(16, 40, dtype=E4M3), out)
    with pytest.raises(RuntimeError, match="a_next must be bf16"):
        nv.gemm(a, torch.zeros(16, 32, dtype=E4M3), out,
                emit=(torch.zeros(4, 16, dtype=E4M3), torch.zeros(16), torch.zeros(4, 2)))


def test_epilogue_mirror_has_the_weight_format_field():
    from diffsynth import _native as nv
    ep = nv.GemmEpilogue()
    assert nv.GemmEpilogue._fields_[-1][0] == "w_e4m3" and ep.w_e4m3 == 0
