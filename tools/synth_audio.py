"""Deterministic synthetic weights, waveforms and checkpoint directories of the wav2vec2 audio feature extractor.

Shared by tests/golden/make_golden_audio.py, the tests and tools/audio_bench.py.  Keys and shapes follow the Hugging Face
`Wav2Vec2Model` state dict the reference loads (utils/src/audio_analysis/wav2vec2.py subclasses it), with the positional
conv's weight norm in the current `parametrizations.weight.original0/1` naming.
"""
import json
import os

import numpy as np
import torch

# the "base" config (chinese-wav2vec2-base / wav2vec2-base) and a tiny one with the same structure
BASE = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, conv_dim=[512] * 7,
            conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2, 2, 2], num_conv_pos_embeddings=128,
            num_conv_pos_embedding_groups=16, layer_norm_eps=1e-5, feat_extract_norm="group", do_stable_layer_norm=False,
            hidden_act="gelu", feat_extract_activation="gelu", conv_bias=False)
TINY = dict(BASE, hidden_size=48, num_hidden_layers=2, num_attention_heads=4, intermediate_size=96, conv_dim=[32] * 7,
            num_conv_pos_embeddings=16, num_conv_pos_embedding_groups=4)
# the tiny structure with a positional-conv group width of 16: the native engine needs hidden_size / groups % 8 == 0 (the
# GEMM's N granularity; 48 in BASE), which TINY's 12 is not
TINY_ENGINE = dict(TINY, hidden_size=64, intermediate_size=128)
PREPROCESSOR = dict(do_normalize=True, feature_size=1, padding_side="right", padding_value=0.0, return_attention_mask=False,
                    sampling_rate=16000)
POS_G, POS_V = "encoder.pos_conv_embed.conv.parametrizations.weight.original0", "encoder.pos_conv_embed.conv.parametrizations.weight.original1"


def param_shapes(cfg):
    d, f, cd = cfg["hidden_size"], cfg["intermediate_size"], cfg["conv_dim"]
    k, groups = cfg["num_conv_pos_embeddings"], cfg["num_conv_pos_embedding_groups"]
    sh = {"masked_spec_embed": (d,)}
    for i, (c, kk) in enumerate(zip(cd, cfg["conv_kernel"])):
        sh[f"feature_extractor.conv_layers.{i}.conv.weight"] = (c, 1 if i == 0 else cd[i - 1], kk)
    sh["feature_extractor.conv_layers.0.layer_norm.weight"] = (cd[0],)
    sh["feature_extractor.conv_layers.0.layer_norm.bias"] = (cd[0],)
    sh.update({"feature_projection.layer_norm.weight": (cd[-1],), "feature_projection.layer_norm.bias": (cd[-1],),
               "feature_projection.projection.weight": (d, cd[-1]), "feature_projection.projection.bias": (d,),
               "encoder.pos_conv_embed.conv.bias": (d,), POS_G: (1, 1, k), POS_V: (d, d // groups, k),
               "encoder.layer_norm.weight": (d,), "encoder.layer_norm.bias": (d,)})
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layers.{i}."
        for n in ("q", "k", "v", "out"):
            sh[p + f"attention.{n}_proj.weight"] = (d, d)
            sh[p + f"attention.{n}_proj.bias"] = (d,)
        sh.update({p + "layer_norm.weight": (d,), p + "layer_norm.bias": (d,),
                   p + "feed_forward.intermediate_dense.weight": (f, d), p + "feed_forward.intermediate_dense.bias": (f,),
                   p + "feed_forward.output_dense.weight": (d, f), p + "feed_forward.output_dense.bias": (d,),
                   p + "final_layer_norm.weight": (d,), p + "final_layer_norm.bias": (d,)})
    return sh


def make_state_dict(cfg, seed=0):
    """Seeded weights at the scale of a trained model: fan-in scaled products, norm gains near 1, small biases."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in param_shapes(cfg).items():
        if name.endswith("norm.weight"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif name == POS_G:
            t = 1.0 + 0.2 * torch.rand(shape, generator=g)
        elif name.endswith(".bias") or name == "masked_spec_embed":
            t = 0.05 * torch.randn(shape, generator=g)
        else:
            fan_in = int(np.prod(shape[1:]))
            t = torch.randn(shape, generator=g) * (1.5 / fan_in) ** 0.5
        sd[name] = t.float()
    return sd


def make_waveform(seconds, sr=16000, seed=0, channels=1):
    """Speech-like test signal in [-1, 1): a few gliding harmonics under a syllable-rate envelope plus noise,
    float32 [n] (channels == 1) or [n, channels]."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * sr))
    t = np.arange(n) / sr
    f0 = 120 + 40 * np.sin(2 * np.pi * 0.7 * t + rng.uniform(0, 6))
    phase = 2 * np.pi * np.cumsum(f0) / sr
    voiced = sum((0.5 / h) * np.sin(h * phase + rng.uniform(0, 6)) for h in range(1, 6))
    env = 0.5 + 0.5 * np.sin(2 * np.pi * 4.0 * t + rng.uniform(0, 6)) ** 2
    x = 0.3 * env * voiced + 0.02 * rng.standard_normal(n)
    if channels > 1:
        x = np.stack([x * (1.0 - 0.1 * c) + 0.005 * rng.standard_normal(n) for c in range(channels)], axis=1)
    return np.clip(x, -1.0, 0.999).astype(np.float32)


def write_checkpoint(path, cfg, sd, fmt="safetensors", weight_norm="parametrizations", prefix="", extra_keys=False,
                     config_overrides=None):
    """A Hugging Face style directory: config.json, preprocessor_config.json and model.safetensors / pytorch_model.bin.
    weight_norm="legacy" stores the positional conv as weight_g / weight_v; prefix="wav2vec2." and extra_keys=True give the
    layout of a pretraining checkpoint (Wav2Vec2ForPreTraining: quantizer / project_* heads next to the encoder)."""
    os.makedirs(path, exist_ok=True)
    out = {}
    for k, v in sd.items():
        if weight_norm == "legacy" and k == POS_G:
            k = "encoder.pos_conv_embed.conv.weight_g"
        elif weight_norm == "legacy" and k == POS_V:
            k = "encoder.pos_conv_embed.conv.weight_v"
        out[prefix + k] = v.contiguous()
    if extra_keys:
        d = cfg["hidden_size"]
        out["quantizer.codevectors"] = torch.zeros(1, 8, 16)
        out["quantizer.weight_proj.weight"] = torch.zeros(8, cfg["conv_dim"][-1])
        out["project_hid.weight"] = torch.zeros(16, d)
        out["project_q.weight"] = torch.zeros(16, 16)
    conf = dict(cfg, model_type="wav2vec2", architectures=["Wav2Vec2Model"])
    conf.update(config_overrides or {})
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(conf, f, indent=1)
    with open(os.path.join(path, "preprocessor_config.json"), "w") as f:
        json.dump(dict(PREPROCESSOR, feature_extractor_type="Wav2Vec2FeatureExtractor"), f, indent=1)
    if fmt == "safetensors":
        from safetensors.torch import save_file
        save_file(out, os.path.join(path, "model.safetensors"))
    else:
        torch.save(out, os.path.join(path, "pytorch_model.bin"))
    return path


def write_wav(path, x, sr, dtype="int16"):
    """x float [n] or [n, channels] in [-1, 1) -> WAV: PCM int16 / int24 / int32 or IEEE float32 (scipy.io.wavfile
    writes no 24-bit PCM, so that one is written by write_wav24)."""
    from scipy.io import wavfile
    if dtype == "float32":
        wavfile.write(path, sr, x.astype(np.float32))
    elif dtype == "int16":
        wavfile.write(path, sr, np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.int16))
    elif dtype == "int32":
        wavfile.write(path, sr, np.clip(np.round(x * 2.0 ** 31), -2 ** 31, 2 ** 31 - 1).astype(np.int32))
    elif dtype == "int24":
        write_wav24(path, x, sr)
    else:
        raise ValueError(dtype)
    return path


def write_wav24(path, x, sr):
    """24-bit PCM WAV written by hand (RIFF header + little-endian 3-byte samples)."""
    import struct
    x = x.reshape(len(x), -1)
    ch = x.shape[1]
    q = np.clip(np.round(x * 2.0 ** 23), -2 ** 23, 2 ** 23 - 1).astype(np.int32).reshape(-1)
    b = q.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    hdr = b"RIFF" + struct.pack("<I", 36 + len(b)) + b"WAVE" + b"fmt " + struct.pack("<IHHIIHH", 16, 1, ch, sr, sr * ch * 3, ch * 3, 24)
    with open(path, "wb") as f:
        f.write(hdr + b"data" + struct.pack("<I", len(b)) + b)
    return path
