"""CPU: dropping a WanModel frees it and its native engine at once (by reference count), without waiting for Python's cyclic
garbage collector.  The model caches its engine, and the engine holds the kernel-ready copies of every weight on the device;
a reference from the engine back to the model would keep all of that alive after the caller drops the model, until the
collector happened to run."""
import gc
import weakref

import torch

from tools import synth


def test_model_and_engine_die_with_the_last_reference(monkeypatch):
    import nv_emulation_lora
    from diffsynth.models.wan_video_dit import WanModel
    nv_emulation_lora.install(monkeypatch)
    monkeypatch.setenv("SVI_CUDA_GRAPHS", "0")
    cfg = synth.CFG_TINY_I2V
    gc.collect()
    gc.disable()
    try:
        m = WanModel(**cfg).eval()
        m.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in synth.make_dit_state_dict(cfg, seed=1).items()})
        lora = {}
        for t in ("self_attn.q", "ffn.2"):
            out_f, in_f = m.state_dict()[f"blocks.0.{t}.weight"].shape
            lora[f"blocks.0.{t}.lora_A.default.weight"] = torch.randn(4, in_f) * 0.01
            lora[f"blocks.0.{t}.lora_B.default.weight"] = torch.randn(out_f, 4) * 0.01
        m.add_lora_adapter("a", lora)
        m.set_lora_adapters({"a": 0.5})
        eng = m.engine("cpu")
        inp = synth.make_dit_inputs(cfg, 2, 4, 6, seed=1, ctx_len=8)
        eng.forward(inp["x"], 500.0, inp["context"], inp["clip_feature"], inp["y"])
        wm, we = weakref.ref(m), weakref.ref(eng)
        del m, eng
        assert wm() is None and we() is None
    finally:
        gc.enable()
