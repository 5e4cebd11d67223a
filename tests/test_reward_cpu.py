"""CPU: the cross-attention scorers (ImageRewardScore, MPScore of diffsynth.extensions.ImageQualityMetric).

* the oracle, the tokenizers and the host preprocessing against the real reference modules (tests/golden/reward_tiny.npz):
  token ids and host pixels exactly, image states, [CLS] rows, MPS's rows, mask, cross features and scores to fp32
  tolerance;
* strict loading, the keys skipped by name, config rejection naming the field, missing path entries;
* include/svi_b200_reward.h against REWARD_SIGNATURES and the GPU test file's COVERED table;
* both scorers end to end on the kernel stand-ins (nv_emulation_reward) against the oracle, and all seven
  load_preference_model names.
"""
import ctypes
import hashlib
import os
import re

import numpy as np
import pytest
import torch

import nv_emulation_reward as emu
from oracle import reward_oracle as O
from tools import synth_quality as SQ
from tools import synth_reward as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "reward_tiny.npz")
HEADER = os.path.join(ROOT, "include", "svi_b200_reward.h")
TOL = dict(rtol=1e-4, atol=1e-5)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    return R.write_reward_checkpoints(str(tmp_path_factory.mktemp("reward")))


def _t(a):
    return torch.from_numpy(np.asarray(a))


# ------------------------------------------------------------------------------------------------ against the reference
def test_tokenizers_match_reference_ids(gold, tiny):
    from transformers import AutoTokenizer

    from diffsynth.extensions.ImageQualityMetric.reward import MPS_CONDITIONS, ImageRewardScore, bert_tokenizer
    paths, _ = tiny
    scorer = ImageRewardScore.__new__(ImageRewardScore)
    scorer.tokenizer = bert_tokenizer(paths["bert_model_path"])
    for i, p in enumerate(R.PROMPTS):
        ids, mask = scorer.tokenize(p)
        assert np.array_equal(ids.numpy(), gold[f"bert_ids_{i}"]) and np.array_equal(mask.numpy(), gold[f"bert_mask_{i}"])
    assert gold["bert_mask_1"].all(), "the long prompt is truncated to 35 word pieces"
    assert gold["bert_mask_0"].sum() < 35, "the short prompt is padded"
    tok = AutoTokenizer.from_pretrained(paths["clip"])
    enc = lambda c: tok(c, max_length=tok.model_max_length, padding="max_length", truncation=True, return_tensors="pt").input_ids
    for i, p in enumerate(R.PROMPTS):
        assert np.array_equal(enc(p).numpy(), gold[f"clip_ids_{i}"])
    for c in ("overall", "semantic"):
        assert np.array_equal(enc(MPS_CONDITIONS[c]).numpy(), gold[f"clip_cond_ids_{c}"])


def test_host_pixels_match_reference_exactly(gold, tiny):
    from transformers import CLIPImageProcessor

    from diffsynth.extensions.ImageQualityMetric import towers as T
    paths, _ = tiny
    px = torch.stack([T.blip_pixels(f, 224) for f in R.frames()])
    assert hashlib.sha256(px.numpy().tobytes()).hexdigest() == str(gold["blip_pixels_sha256"])
    assert hashlib.sha256(O.Q.normalize(px).numpy().tobytes()).hexdigest() == str(gold["blip_inputs_sha256"])
    proc = CLIPImageProcessor.from_pretrained(paths["clip"])
    assert torch.equal(torch.stack([T.hf_pixels(proc, f) for f in R.frames()]), _t(gold["mps_pixels"]))
    with pytest.raises(ValueError, match="RGBA"):
        T.blip_pixels(R.frames()[0].convert("RGBA"), 224)


def test_oracle_matches_reference_imagereward(gold, tiny):
    _, ref = tiny
    from diffsynth.extensions.ImageQualityMetric import towers as T
    med, sd = ref["imagereward"]
    px = O.Q.normalize(torch.stack([T.blip_pixels(f, 224) for f in R.frames()]))      # the reference's inputs (sha256 above)
    img = O.blip_image_states(sd, px, R.TINY_VISION["layers"])
    torch.testing.assert_close(img[:, [0, 1, 98, 196]], _t(gold["blip_image_states"]), **TOL)
    for i in (0, 1):
        ids, mask = _t(gold[f"bert_ids_{i}"]), _t(gold[f"bert_mask_{i}"])
        cls = O.bert_cls(sd, med, ids, mask, img)
        torch.testing.assert_close(cls, _t(gold[f"bert_cls_{i}"]), **TOL)
        torch.testing.assert_close(O.reward_head(sd, cls), _t(gold[f"imagereward_scores_{i}"]), **TOL)


@pytest.mark.parametrize("cond", ["overall", "semantic"])
def test_oracle_matches_reference_mps(gold, tiny, cond):
    _, ref = tiny
    conf, sd = ref["mps"]
    r = O.mps(sd, conf, 2, 2, _t(gold["mps_inputs"]), _t(gold["clip_ids_2"]), _t(gold[f"clip_cond_ids_{cond}"]))
    for k in ("text_f", "cond_f", "text_eos", "ratio", "cross"):
        torch.testing.assert_close(r[k], _t(gold[f"mps_{k}_{cond}"]), **TOL)
    torch.testing.assert_close(r["image_rows"], _t(gold["mps_image_rows"]), **TOL)
    assert torch.equal(r["keep"], _t(gold[f"mps_keep_{cond}"]))
    torch.testing.assert_close(r["scores"], _t(gold[f"mps_scores_{cond}"]), rtol=1e-4, atol=1e-4)
    if cond == "overall":
        assert 0 < int(r["keep"].sum()) < r["keep"].numel(), "the fixture's mask keeps and drops keys"


# ------------------------------------------------------------------------------------------------ loading and configs
def test_strict_loading_and_skipped_keys(tiny):
    from safetensors.torch import load_file

    from diffsynth.extensions.ImageQualityMetric.reward import ImageRewardModel, MPSModel, _ignored
    paths, ref = tiny
    m = ImageRewardModel.from_files(paths["imagereward"], paths["med_config"])
    skipped = {k for k in load_file(paths["imagereward"]) if _ignored(k)}
    assert skipped == {"blip.vision_proj.weight", "blip.vision_proj.bias", "blip.text_proj.weight", "blip.text_proj.bias",
                       "blip.text_encoder.embeddings.position_ids"}
    assert set(m.state_dict()) == set(ref["imagereward"][1]) - skipped
    mm = MPSModel.from_files(paths["mps"], paths["clip"])
    assert {k for k in load_file(paths["mps"]) if _ignored(k)} == {f"cross_model.layers.{i}.1.fn.rotary_emb.inv_freq" for i in range(2)}
    assert torch.equal(mm.cross_model.layers[0][0].fn.norm.bias, torch.zeros(64))
    sd = {k: v for k, v in ref["imagereward"][1].items() if not _ignored(k) and k != "blip.visual_encoder.norm.bias"}
    with pytest.raises(RuntimeError, match="Missing"):
        m.load_state_dict(sd, strict=True)


@pytest.mark.parametrize("key,value,field", [
    ("hidden_act", "gelu_new", "hidden_act"),
    ("position_embedding_type", "relative_key", "position_embedding_type"),
    ("add_cross_attention", False, "add_cross_attention"),
    ("num_attention_heads", 4, "num_attention_heads"),
    ("max_position_embeddings", 20, "max_position_embeddings"),
])
def test_med_config_rejected_with_field(key, value, field):
    from diffsynth.extensions.ImageQualityMetric.reward import BertCrossModel
    conf = dict(R.FULL_MED, **{key: value})
    with torch.device("meta"), pytest.raises(ValueError, match=re.escape(field)):
        BertCrossModel(conf, 1024)


def test_mps_cross_sizes_from_weights_and_rejections(tiny):
    from diffsynth.extensions.ImageQualityMetric.reward import CrossModel, MPSModel
    _, ref = tiny
    conf, sd = ref["mps"]
    assert CrossModel.sizes(sd) == (64, 2, 64, 256, 2)
    full = {k: torch.empty(v.shape, device="meta") for k, v in R.cross_state_dict(1024, 16, 4).items()}
    assert CrossModel.sizes(full) == (1024, 16, 64, 4096, 4)
    bad = dict(sd, **{"cross_model.layers.0.0.fn.to_kv.weight": torch.empty(160, 64)})
    with pytest.raises(ValueError, match="dim_head"):
        CrossModel.sizes(bad)
    with pytest.raises(ValueError, match="projection_dim"):
        MPSModel(dict(conf, projection_dim=128), CrossModel.sizes(sd))


def test_missing_paths_name_the_model_and_key(tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import ImageRewardScore, MPScore
    emu.install(monkeypatch)
    paths, _ = tiny
    for cls, name, key in ((ImageRewardScore, "ImageReward", "bert_model_path"), (ImageRewardScore, "ImageReward", "med_config"),
                           (MPScore, "MPS", "mps")):
        with pytest.raises(ValueError, match=rf"{name}.*{key}"):
            cls(device="cpu", path={k: v for k, v in paths.items() if k != key})
    with pytest.raises(ValueError, match="imagereward"):
        ImageRewardScore(device="cpu", path=dict(paths, imagereward="/nonexistent/ImageReward.safetensors"))


def test_full_size_key_sets():
    from diffsynth.extensions.ImageQualityMetric.reward import ImageRewardModel
    with torch.device("meta"):
        m = ImageRewardModel(R.FULL_MED, **R.FULL_VISION)
    sd = m.state_dict()
    assert len([k for k in sd if k.startswith("blip.visual_encoder.")]) == 4 + 24 * 12 + 2
    assert len([k for k in sd if k.startswith("blip.text_encoder.")]) == 4 + 12 * 26
    assert ImageRewardModel.vision_sizes({k: v for k, v in sd.items()}) == tuple(R.FULL_VISION.values())


# ------------------------------------------------------------------------------------------------ header
def test_header_matches_signatures_and_gpu_cases():
    from diffsynth import _native as nv
    import test_reward_gpu as gpu
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = set(re.findall(r"^(?:int|size_t|void|const char\*)\s+(svi_\w+)\s*\(", src, re.M))
    assert names == set(nv.REWARD_SIGNATURES)
    for other in (nv.SIGNATURES, nv.LORA_SIGNATURES, nv.RIFE_SIGNATURES, nv.ESRGAN_SIGNATURES, nv.FASTBLEND_SIGNATURES,
                  nv.UNIANIMATE_SIGNATURES, nv.REPLACE_SIGNATURES, nv.QUALITY_SIGNATURES):
        assert not names & set(other)
    assert set(gpu.COVERED) == names
    for entry, cases in gpu.COVERED.items():
        assert cases and all(callable(getattr(gpu, c, None)) and c.startswith("test_") for c in cases), entry
    import test_quality_fp64_gpu as fp64
    for entry, cases in fp64.COVERED.items():
        if entry in names:
            assert cases and all(callable(getattr(fp64, c, None)) and c.startswith("test_") for c in cases), entry
    if os.path.exists(nv.lib_path()):
        lib = ctypes.CDLL(nv.lib_path())
        assert all(hasattr(lib, n) for n in names)


# ------------------------------------------------------------------------------------------------ engines on stand-ins
def _oracle_imagereward(paths, ref, frames, prompt):
    from diffsynth.extensions.ImageQualityMetric import towers as T
    from diffsynth.extensions.ImageQualityMetric.reward import bert_tokenizer
    med, sd = ref["imagereward"]
    t = bert_tokenizer(paths["bert_model_path"])(prompt, padding="max_length", truncation=True, max_length=35,
                                                  return_tensors="pt")
    px = O.Q.normalize(torch.stack([T.blip_pixels(f, 224) for f in frames]))
    return O.imagereward(sd, med, R.TINY_VISION["layers"], px, t.input_ids, t.attention_mask)[2].tolist()


def _oracle_mps(paths, ref, frames, prompt, cond="overall"):
    from transformers import AutoTokenizer, CLIPImageProcessor

    from diffsynth.extensions.ImageQualityMetric import towers as T
    from diffsynth.extensions.ImageQualityMetric.reward import MPS_CONDITIONS
    conf, sd = ref["mps"]
    proc, tok = CLIPImageProcessor.from_pretrained(paths["clip"]), AutoTokenizer.from_pretrained(paths["clip"])
    enc = lambda c: tok(c, max_length=77, padding="max_length", truncation=True, return_tensors="pt").input_ids
    px = O.Q.normalize(torch.stack([T.hf_pixels(proc, f) for f in frames]), *T.hf_mean_std(proc))
    return O.mps(sd, conf, 2, 2, px, enc(prompt), enc(MPS_CONDITIONS[cond]))["scores"].tolist()


@pytest.mark.parametrize("prompt", [R.PROMPTS[0], R.PROMPTS[1]])
def test_imagereward_on_standins_matches_oracle(prompt, tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import load_preference_model
    emu.install(monkeypatch)
    paths, ref = tiny
    model = load_preference_model("ImageReward", device="cpu", path=paths)
    frames = R.frames()
    got = model.score(frames, prompt)
    want = _oracle_imagereward(paths, ref, frames, prompt)
    assert len(got) == 4 and all(isinstance(v, float) for v in got)
    assert np.abs(np.array(got) - np.array(want)).max() < 3e-2 * max(1.0, np.abs(want).max())
    eng = model.engine()
    eng.chunk = eng.vision.chunk = 3
    assert model.score(frames, prompt) == got
    assert model.score(frames[1], prompt) == got[1:2]
    assert model.score([], prompt) == []
    with pytest.raises(TypeError, match="illegal"):
        model.score(42, prompt)
    with pytest.raises(TypeError, match="illegal"):
        model.score([frames[0], 42], prompt)


def test_mps_on_standins_matches_oracle(tiny, monkeypatch):
    from diffsynth.extensions.ImageQualityMetric import MPScore, load_preference_model
    emu.install(monkeypatch)
    paths, ref = tiny
    model = load_preference_model("MPS", device="cpu", path=paths)
    frames = R.frames()
    got = model.score(frames, R.PROMPTS[2])
    want = _oracle_mps(paths, ref, frames, R.PROMPTS[2])
    assert len(got) == 4 and all(isinstance(v, float) for v in got)
    assert np.abs(np.array(got) - np.array(want)).max() < 3e-2 * max(1.0, np.abs(want).max())
    eng = model.engine()
    eng.chunk = eng.vision.chunk = 3
    assert model.score(frames, R.PROMPTS[2]) == got
    bad = MPScore(device="cpu", path=paths, condition="style")          # accepted at construction, as in the reference
    with pytest.raises(ValueError, match="Unsupported condition: style"):
        bad.score(frames, R.PROMPTS[2])
    with pytest.raises(TypeError, match="illegal"):
        model.score(3.5, R.PROMPTS[2])


def test_project_then_pool_equals_pool_then_project_on_standins(monkeypatch, tiny):
    from diffsynth.extensions.ImageQualityMetric.reward import MPSModel
    emu.install(monkeypatch)
    paths, _ = tiny
    eng = MPSModel.from_files(paths["mps"], paths["clip"]).model.engine("cpu")
    ids = torch.randint(1, 600, (3, 77), generator=torch.Generator().manual_seed(0))
    ids[:, 30] = 643
    rows, pooled = eng.text.encode_text_rows(ids)
    torch.testing.assert_close(pooled, eng.text.encode_text(ids), rtol=1e-6, atol=1e-6)


def test_load_preference_model_builds_all_seven_names(tiny, monkeypatch, tmp_path):
    from diffsynth.extensions.ImageQualityMetric import (MODEL_PATHS, AestheticScore, CLIPScore, HPScore_v2,
                                                         ImageRewardScore, MPScore, PickScore, get_model_path,
                                                         load_preference_model)
    emu.install(monkeypatch)
    quality_paths, _ = SQ.write_tiny_checkpoints(str(tmp_path))
    paths = dict(quality_paths, **tiny[0])
    for name, cls in (("CLIP", CLIPScore), ("HPSv2", HPScore_v2), ("HPSv2.1", HPScore_v2), ("PickScore", PickScore),
                      ("Aesthetic", AestheticScore), ("ImageReward", ImageRewardScore), ("MPS", MPScore)):
        assert isinstance(load_preference_model(name, device="cpu", path=paths), cls)
    assert MODEL_PATHS["bert_model_path"] == get_model_path("bert-base-uncased")
    with pytest.raises(ValueError, match="unknown model"):
        load_preference_model("BLIP", device="cpu", path=paths)


def test_no_cpu_path_without_standins(tiny):
    from diffsynth.extensions.ImageQualityMetric import ImageRewardScore
    paths, _ = tiny
    with pytest.raises(RuntimeError, match="CUDA"):
        ImageRewardScore(device="cpu", path=paths)
