"""CPU: the quality-metric scorers (diffsynth.extensions.ImageQualityMetric).

* the oracle, the BPE tokenizer and the host preprocessing against the real reference modules
  (tests/golden/quality_tiny.npz): token ids and host-prepared pixels exactly, features and scores to fp32 tolerance;
* strict loading of both checkpoint formats and the aesthetic MLP, its fold, and config rejection naming the field;
* include/svi_b200_quality.h against QUALITY_SIGNATURES;
* every scorer end to end on the kernel stand-ins (nv_emulation_quality) against the oracle, a batch split into chunks,
  and load_preference_model's names.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import nv_emulation_quality as emu
from oracle import quality_oracle as O
from tools import synth_quality as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "quality_tiny.npz")
HEADER = os.path.join(ROOT, "include", "svi_b200_quality.h")
SIZES = [(40, 70), (71, 33), (56, 56), (97, 120)]      # as tests/golden/make_golden_quality.py


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    return S.write_tiny_checkpoints(str(tmp_path_factory.mktemp("quality")))


def _frames():
    return [S.frames(1, h, w, seed=i)[0] for i, (h, w) in enumerate(SIZES)]


# ------------------------------------------------------------------------------------------------ against the reference
def test_bpe_tokenizer_matches_reference_ids(gold, tiny):
    from diffsynth.extensions.ImageQualityMetric import SimpleTokenizer
    paths, _ = tiny
    ids = SimpleTokenizer(paths["open_clip_bpe"])(S.PROMPTS)
    assert torch.equal(ids, torch.from_numpy(gold["openclip_ids"]))
    assert ids[4, -1] == ids.max() and (ids[4] != 0).all(), "the over-long prompt keeps its end-of-text id"
    assert ids[3, :2].tolist() == [ids.max() - 1, ids.max()] and (ids[3, 2:] == 0).all()


def test_hf_processor_ids_and_pixels(gold, tiny):
    from transformers import AutoProcessor

    from diffsynth.extensions.ImageQualityMetric import towers as T
    paths, _ = tiny
    proc = AutoProcessor.from_pretrained(paths["clip"])
    for i, p in enumerate(S.PROMPTS):
        got = proc(text=p, padding=True, truncation=True, max_length=77, return_tensors="pt")["input_ids"]
        assert np.array_equal(got.numpy(), gold[f"hf_ids_{i}"])
    px = torch.stack([T.hf_pixels(proc, f) for f in _frames()])
    assert torch.equal(px, torch.from_numpy(gold["hf_pixels"]))


def test_openclip_pixels_match_reference_exactly(gold):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    px = torch.stack([T.openclip_pixels(f, 56) for f in _frames()])
    assert torch.equal(px, torch.from_numpy(gold["openclip_pixels"]))


def test_oracle_matches_reference_features_and_scores(gold, tiny):
    _, ref = tiny
    cfg, sd = ref["open_clip"]
    px = O.normalize(torch.from_numpy(gold["openclip_pixels"]))
    ids = torch.from_numpy(gold["openclip_ids"])
    img, txt = O.openclip_image(sd, cfg, px), O.openclip_text(sd, cfg, ids)
    tol = dict(rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(img, torch.from_numpy(gold["openclip_image_features"]), **tol)
    torch.testing.assert_close(txt, torch.from_numpy(gold["openclip_text_features"]), **tol)
    torch.testing.assert_close(O.cosine(img, txt[:1])[:, 0], torch.from_numpy(gold["openclip_scores"]), **tol)
    mean, std = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
    hpx = O.normalize(torch.from_numpy(gold["hf_pixels"]), mean, std)
    hids = torch.from_numpy(gold["hf_ids_0"])
    for name, key in (("pick", "pickscore"), ("large", "clip-large")):
        conf, hsd = ref[key]
        img, txt = O.hf_image(hsd, conf, hpx), O.hf_text(hsd, conf, hids)
        torch.testing.assert_close(img, torch.from_numpy(gold[f"{name}_image_features"]), **tol)
        torch.testing.assert_close(txt, torch.from_numpy(gold[f"{name}_text_features"]), **tol)
        torch.testing.assert_close(O.cosine(img, txt)[:, 0], torch.from_numpy(gold[f"{name}_scores"]), **tol)
    aes = O.aesthetic(ref["aesthetic_predictor"][1], torch.from_numpy(gold["large_image_features"]))
    torch.testing.assert_close(aes, torch.from_numpy(gold["aesthetic_scores"]), **tol)


def test_aesthetic_fold_equals_the_five_layers():
    from diffsynth.extensions.ImageQualityMetric.towers import AestheticMLP
    m = AestheticMLP(768).eval()
    m.load_state_dict(S.aesthetic_state_dict(seed=4), strict=True)
    w, b = m.folded()
    x = torch.randn(9, 768, dtype=torch.float64)
    with torch.no_grad():
        want = m.double().layers(x)[:, 0]
    torch.testing.assert_close(x @ w.double() + b, want, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------ loading and configs
def test_strict_loading_of_both_formats(tiny):
    from diffsynth.extensions.ImageQualityMetric.towers import HFCLIPModel, OpenCLIP
    paths, ref = tiny
    cfg, sd = ref["open_clip"]
    m = OpenCLIP(**cfg)
    m.load_state_dict(sd, strict=True)
    with pytest.raises(RuntimeError, match="Missing"):
        m.load_state_dict({k: v for k, v in sd.items() if k != "visual.proj"}, strict=True)
    h = HFCLIPModel.from_pretrained(paths["pickscore"])
    torch.testing.assert_close(h.visual_projection.weight, ref["pickscore"][1]["visual_projection.weight"])
    assert set(h.state_dict()) == set(ref["pickscore"][1])


def test_full_size_key_sets():
    from diffsynth.extensions.ImageQualityMetric import scorers
    from diffsynth.extensions.ImageQualityMetric.towers import VIT_H_14, HFCLIPModel, OpenCLIP
    with torch.device("meta"):
        m = OpenCLIP(**VIT_H_14)
        h = HFCLIPModel(S.HF_FULL_LARGE)
    sd = m.state_dict()
    assert len(sd) == (4 + 4 + 32 * 12) + (4 + 2 + 24 * 12) and sd["visual.proj"].shape == (1280, 1024)
    assert scorers.openclip_config({k: v for k, v in sd.items()}) == VIT_H_14
    assert h.state_dict()["vision_model.embeddings.position_embedding.weight"].shape == (257, 1024)


@pytest.mark.parametrize("kw,field", [
    (dict(vision_cfg=dict(head_width=96)), "vision_cfg.head_width"),
    (dict(text_cfg=dict(heads=4)), "text_cfg.heads"),
    (dict(vision_cfg=dict(image_size=336, patch_size=14)), "vision_cfg.image_size"),
    (dict(text_cfg=dict(context_length=400)), "text_cfg.context_length"),
    (dict(vision_cfg=dict(global_average_pool=True)), "vision_cfg.global_average_pool"),
])
def test_openclip_config_rejected_with_field(kw, field):
    from diffsynth.extensions.ImageQualityMetric.towers import VIT_H_14, OpenCLIP
    cfg = dict(embed_dim=1024, vision_cfg=dict(VIT_H_14["vision_cfg"], **kw.get("vision_cfg", {})),
               text_cfg=dict(VIT_H_14["text_cfg"], **kw.get("text_cfg", {})))
    with torch.device("meta"), pytest.raises(ValueError, match=re.escape(field)):
        OpenCLIP(**cfg)


@pytest.mark.parametrize("tower,key,value,field", [
    ("vision_config", "hidden_act", "relu", "vision_config.hidden_act"),
    ("text_config", "hidden_act", "gelu_new", "text_config.hidden_act"),
    ("vision_config", "num_attention_heads", 10, "vision_config.num_attention_heads"),
    ("text_config", "max_position_embeddings", 512, "text_config.max_position_embeddings"),
])
def test_hf_config_rejected_with_field(tower, key, value, field):
    from diffsynth.extensions.ImageQualityMetric.towers import HFCLIPModel
    conf = {k: (dict(v) if isinstance(v, dict) else v) for k, v in S.hf_tiny_pick(644).items()}
    conf[tower][key] = value
    with pytest.raises(ValueError, match=re.escape(field)):
        HFCLIPModel(conf)


# ------------------------------------------------------------------------------------------------ header
def test_header_matches_signatures_and_gpu_cases():
    from diffsynth import _native as nv
    import test_quality_gpu as gpu
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))
    assert names == set(nv.QUALITY_SIGNATURES)
    for other in (nv.SIGNATURES, nv.RIFE_SIGNATURES, nv.ESRGAN_SIGNATURES, nv.FASTBLEND_SIGNATURES, nv.REPLACE_SIGNATURES):
        assert not names & set(other)
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    import test_quality_fp64_gpu as fp64
    assert set(fp64.COVERED) <= names | set(nv.REWARD_SIGNATURES), "the fp64 module names an undeclared entry point"
    for entry, cases in fp64.COVERED.items():
        if entry in names:
            assert cases and all(callable(getattr(fp64, c, None)) and c.startswith("test_") for c in cases), entry
    for macro, value in (("SVI_QUALITY_MAX_L", nv.QUALITY_MAX_L), ("SVI_POOL_FIRST", nv.POOL_FIRST),
                         ("SVI_POOL_ARGMAX", nv.POOL_ARGMAX), ("SVI_POOL_EOS", nv.POOL_EOS)):
        assert re.search(rf"#define {macro} {value}\b", src), macro
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)


# ------------------------------------------------------------------------------------------------ engines on stand-ins
@pytest.mark.parametrize("name", ["CLIP", "HPSv2", "HPSv2.1", "PickScore", "Aesthetic"])
def test_scorers_on_standins_match_oracle(name, tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    emu.install(monkeypatch)
    paths, ref = tiny
    model = load_preference_model(name, device="cpu", path=paths)
    frames = _frames()
    got = model.score(frames, S.PROMPTS[1])
    want = S.oracle_scores(name, paths, ref, frames, S.PROMPTS[1])
    assert len(got) == 4 and all(isinstance(v, float) for v in got)
    assert np.abs(np.array(got) - np.array(want)).max() < 5e-3


def test_chunked_batch_equals_one_batch(tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import CLIPScore
    emu.install(monkeypatch)
    paths, _ = tiny
    model = CLIPScore(device="cpu", path=paths)
    frames = _frames() * 2
    whole = model.score(frames, "a photo of a cat")
    eng = model.model.engine("cpu")
    eng.vision.chunk = 3
    launches = eng.vision.launches
    assert model.score(frames, "a photo of a cat") == whole
    assert eng.vision.launches - launches == 3 * (3 + 7 * 2 + 3)      # three chunks of 3 + 3 + 2 images


def test_pickscore_softmax_is_one_and_errors_are_wrapped(tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import PickScore
    emu.install(monkeypatch)
    paths, _ = tiny
    model = PickScore(device="cpu", path=paths)
    assert model.score(_frames(), "a dog", softmax=True) == [1.0] * 4
    with pytest.raises(RuntimeError, match="Error in scoring images"):
        model.score(42, "a dog")


def test_load_preference_model_names(tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import (AestheticScore, CLIPScore, HPScore_v2, MODEL_PATHS, PickScore,
                                                         get_model_path, load_preference_model)
    emu.install(monkeypatch)
    paths, _ = tiny
    for name, cls in (("CLIP", CLIPScore), ("HPSv2", HPScore_v2), ("HPSv2.1", HPScore_v2), ("PickScore", PickScore),
                      ("Aesthetic", AestheticScore)):
        assert isinstance(load_preference_model(name, device="cpu", path=paths), cls)
    for name in ("ImageReward", "MPS"):
        with pytest.raises(ValueError, match=name):
            load_preference_model(name, device="cpu", path=paths)
    assert MODEL_PATHS["hpsv2"] == get_model_path("HPS_v2/HPS_v2_compressed.safetensors")
    assert MODEL_PATHS["pickscore"].endswith(os.path.join("models", "QualityMetric", "PickScore_v1"))
    with pytest.raises(ValueError, match="model version"):
        HPScore_v2(device="cpu", path=paths, model_version="v3")


def test_no_cpu_path_without_standins(tiny):
    from diffsynth.extensions.ImageQualityMetric import CLIPScore
    paths, _ = tiny
    with pytest.raises(RuntimeError, match="CUDA"):
        CLIPScore(device="cpu", path=paths)
