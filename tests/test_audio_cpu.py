"""CPU: the wav2vec2 audio feature extractor of SVI-Talk — the oracle against the reference module (tests/golden/
wav2vec_tiny.npz), checkpoint loading, WAV reading / resampling / loudness, and the engine's host logic on the torch
stand-ins of its kernels (tests/nv_emulation_audio.py)."""
import json
import os

import numpy as np
import pytest
import torch

from tools import synth_audio as SA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "wav2vec_tiny.npz")


def _bf(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def test_oracle_matches_reference_golden():
    """The oracle restates the reference's Wav2Vec2Model subclass, linear_interpolation, get_embedding and
    get_audio_embedding to fp32 round-off (measured: input values and conv stack bit-equal, hidden states <= 1.3e-6)."""
    from oracle import wav2vec2_oracle as O
    z = np.load(GOLDEN)
    cfg, sd = SA.TINY, SA.make_state_dict(SA.TINY, seed=int(z["seed"]))
    speech = SA.make_waveform(float(z["seconds"]), seed=int(z["seed"]))
    iv = O.normalize(speech)
    assert np.abs(iv - z["input_values"]).max() < 1e-6
    conv = O.conv_stack(sd, cfg, z["input_values"])
    assert (conv - torch.from_numpy(z["conv_out"])).abs().max().item() < 1e-5
    assert (O.interpolate(conv, int(z["seq_len"])) - torch.from_numpy(z["interp"])).abs().max().item() < 1e-5
    hs = torch.stack(O.forward(sd, cfg, z["input_values"], int(z["seq_len"])))
    assert hs.shape == z["hidden_states"].shape
    assert (hs - torch.from_numpy(z["hidden_states"])).abs().max().item() < 2e-5
    emb = O.embedding(sd, cfg, z["input_values"] * 0 + speech)
    for i, s in enumerate(z["starts"]):
        w = O.windows(emb, int(z["num_frames"]), int(s))
        assert w.shape == z["windows"][i].shape
        assert (w - torch.from_numpy(z["windows"][i])).abs().max().item() < 2e-5


def test_model_keys_match_the_reference_state_dict():
    from diffsynth.models.wav2vec2 import Wav2Vec2Model
    z = np.load(GOLDEN)
    assert sorted(Wav2Vec2Model(SA.TINY).state_dict().keys()) == sorted(str(k) for k in z["keys"])


@pytest.mark.parametrize("fmt,weight_norm,prefix,extra", [("safetensors", "parametrizations", "", False),
                                                          ("safetensors", "legacy", "wav2vec2.", True),
                                                          ("bin", "legacy", "", False),
                                                          ("bin", "parametrizations", "wav2vec2.", True)])
def test_from_pretrained_checkpoint_layouts(tmp_path, fmt, weight_norm, prefix, extra):
    from diffsynth.models.wav2vec2 import Wav2Vec2FeatureExtractor, Wav2Vec2Model
    sd = SA.make_state_dict(SA.TINY, seed=3)
    d = SA.write_checkpoint(str(tmp_path / "w2v"), SA.TINY, sd, fmt=fmt, weight_norm=weight_norm, prefix=prefix, extra_keys=extra)
    m = Wav2Vec2Model.from_pretrained(d)
    got = m.state_dict()
    assert sorted(got) == sorted(sd)
    for k, v in sd.items():
        assert torch.equal(got[k], v), k
    assert m.config.hidden_size == 48 and m.config.num_conv_pos_embedding_groups == 4
    fe = Wav2Vec2FeatureExtractor.from_pretrained(d)
    assert fe.do_normalize and fe.sampling_rate == 16000


def test_from_pretrained_refuses_missing_weights_and_unsupported_configs(tmp_path):
    from diffsynth.models.wav2vec2 import Wav2Vec2Model
    sd = SA.make_state_dict(SA.TINY, seed=3)
    for field, value in (("feat_extract_norm", "layer"), ("do_stable_layer_norm", True), ("hidden_act", "relu"),
                         ("feat_extract_activation", "relu"), ("conv_bias", True)):
        d = SA.write_checkpoint(str(tmp_path / field), SA.TINY, sd, config_overrides={field: value})
        with pytest.raises(ValueError, match=field):
            Wav2Vec2Model.from_pretrained(d)
    sd.pop("encoder.layers.1.final_layer_norm.bias")
    d = SA.write_checkpoint(str(tmp_path / "partial"), SA.TINY, sd)
    with pytest.raises(KeyError, match="lacks"):
        Wav2Vec2Model.from_pretrained(d)
    with pytest.raises(FileNotFoundError):
        Wav2Vec2Model.from_pretrained(str(tmp_path / "absent"))


def test_feature_extractor_matches_the_reference_formula():
    from diffsynth.models.wav2vec2 import Wav2Vec2FeatureExtractor
    z = np.load(GOLDEN)
    speech = SA.make_waveform(float(z["seconds"]), seed=int(z["seed"]))
    iv = Wav2Vec2FeatureExtractor()(speech, sampling_rate=16000).input_values
    assert iv.shape == (1, len(speech)) and iv.dtype == np.float32
    assert np.array_equal(iv[0], z["input_values"])
    with pytest.raises(ValueError):
        Wav2Vec2FeatureExtractor()(speech, sampling_rate=44100)


@pytest.mark.parametrize("dtype,tol", [("int16", 2.0 ** -15), ("int24", 2.0 ** -23), ("int32", 2.0 ** -30), ("float32", 0.0)])
@pytest.mark.parametrize("channels", [1, 2])
def test_wav_reading_scales_to_unit_range(tmp_path, dtype, tol, channels):
    from utils.audio_process import read_wav
    x = SA.make_waveform(0.25, sr=22050, seed=4, channels=channels)
    p = SA.write_wav(str(tmp_path / f"a_{dtype}.wav"), x, 22050, dtype)
    y, sr = read_wav(p)
    assert sr == 22050 and y.dtype == np.float32 and y.shape == x.shape
    assert np.abs(y - x).max() <= tol + 1e-7


def test_prepare_single_mixes_to_mono_and_resamples_to_librosa_length(tmp_path):
    from utils.audio_process import audio_prepare_single, integrated_loudness, resample
    sr, n = 44100, 44100 * 2 + 37
    t = np.arange(n) / sr
    tone = (0.3 * np.sin(2 * np.pi * 440.0 * t)).astype(np.float32)
    y = resample(tone, sr, 16000)
    assert len(y) == int(np.ceil(n * 16000 / sr))
    spec = np.abs(np.fft.rfft(y[1000:-1000] * np.hanning(len(y) - 2000)))
    f_peak = np.argmax(spec) * 16000 / (len(y) - 2000)
    assert abs(f_peak - 440.0) < 1.0
    stereo = np.stack([tone, 0.5 * tone], axis=1)
    p = SA.write_wav(str(tmp_path / "st.wav"), stereo, sr, "float32")
    out = audio_prepare_single(p)
    assert out.ndim == 1 and len(out) == len(y)
    assert abs(integrated_loudness(out, 16000) + 23.0) < 0.05                  # normalised to -23 LUFS
    mono = resample(0.75 * tone, sr, 16000)
    assert np.corrcoef(out, mono)[0, 1] > 0.9999                                # channel mean, then the same resampling
    with pytest.raises(ValueError, match="WAV"):
        audio_prepare_single(str(tmp_path / "speech.mp3"))


def test_loudness_known_answers():
    """A 997 Hz sine at -20 dBFS RMS measures -20.07 LUFS at 16 kHz through the K-weighting filters (the +4 dB shelf adds
    a little at 997 Hz); silence is returned unchanged."""
    from utils.audio_process import integrated_loudness, loudness_norm
    sr = 16000
    t = np.arange(sr * 5) / sr
    amp = 10 ** (-20 / 20) * np.sqrt(2)
    x = (amp * np.sin(2 * np.pi * 997 * t)).astype(np.float32)
    assert abs(integrated_loudness(x, sr) - (-20.07)) < 0.1
    y = loudness_norm(x, sr)
    assert abs(integrated_loudness(y, sr) + 23.0) < 0.01
    z = np.zeros(sr * 2, dtype=np.float32)
    assert loudness_norm(z, sr) is z


def _engine_model(cfg, seed):
    from diffsynth.models.wav2vec2 import Wav2Vec2Model
    sd = _bf(SA.make_state_dict(cfg, seed=seed))
    m = Wav2Vec2Model(cfg).eval()
    m.load_state_dict(sd)
    return m, sd


def test_engine_orchestration_matches_oracle(monkeypatch):
    """Host logic of Wav2Vec2Engine on the emulated kernels: conv packing in (tap, channel) order, the in-place k = s = 2
    operand, the GroupNorm statistics, interpolation, the per-group positional conv with its folded weight norm, the fused
    q|k|v layout and the layer-major residual stream — against the oracle's bf16-point mode (which rounds where the
    kernels store bf16; conv 0's operand in its two-term form).  Measured: mean error 0.30 % of the std, 84 % of the
    elements within rtol 1e-2 / atol 1e-3 — as large as the bf16 rounding error itself (0.33 % against the fp32 oracle):
    at this width a different accumulation order flips bf16 roundings at every rounding point and the LayerNorms carry
    them on, so the bars are 0.6 % / 75 %, and the fp32 oracle's parity bar of 1.5 %."""
    import nv_emulation_audio
    from oracle import wav2vec2_oracle as O
    nv_emulation_audio.install(monkeypatch)
    cfg = SA.TINY_ENGINE
    m, sd = _engine_model(cfg, seed=1)
    speech = SA.make_waveform(3.3, seed=2)
    iv = O.normalize(speech)
    seq_len = O.seq_len_for(len(speech))
    out = m.engine("cpu").forward(torch.from_numpy(iv), seq_len)
    ref = torch.stack(O.forward(sd, cfg, iv, seq_len, bf16_points=True, split_conv0=True))
    got = torch.stack([h[0] for h in out.hidden_states])
    assert got.shape == ref.shape == (cfg["num_hidden_layers"] + 1, seq_len, cfg["hidden_size"])
    err = (got - ref).abs()
    assert err.mean().item() / ref.std().item() < 6e-3 and (err <= 1e-3 + 1e-2 * ref.abs()).float().mean().item() > 0.75
    assert torch.equal(out.last_hidden_state[0], got[-1])
    # the fp32 oracle: the parity statement's bar
    ref32 = torch.stack(O.forward(sd, cfg, iv, seq_len))
    assert (got - ref32).abs().mean().item() / ref32.std().item() < 1.5e-2


def test_pipeline_windows_and_cache_on_emulated_kernels(monkeypatch, tmp_path):
    """SVITalkVideoPipeline.get_audio_embedding: WAV -> mono 16 kHz -> loudness -> extractor -> windows clamped at both
    ends; the whole-file features are extracted once per file and reused by every clip."""
    import nv_emulation_audio
    from diffsynth import SVITalkVideoPipeline
    from oracle import wav2vec2_oracle as O
    from utils.audio_process import audio_prepare_single
    nv_emulation_audio.install(monkeypatch)
    cfg = SA.TINY_ENGINE
    m, sd = _engine_model(cfg, seed=1)
    ck = SA.write_checkpoint(str(tmp_path / "w2v"), cfg, m.state_dict())
    wav = SA.write_wav(str(tmp_path / "talk.wav"), SA.make_waveform(4.0, sr=44100, seed=5, channels=2), 44100, "int16")
    pipe = SVITalkVideoPipeline(device="cpu", torch_dtype=torch.bfloat16, wav2vec_path=ck)
    w0 = pipe.get_audio_embedding(wav, 33, audio_start_idx=0)
    w1 = pipe.get_audio_embedding(wav, 33, audio_start_idx=80)
    assert pipe.audio_extractions == 1
    assert w0.shape == (1, 33, 5, cfg["num_hidden_layers"], cfg["hidden_size"]) and w0.dtype == torch.float32
    speech = audio_prepare_single(wav)
    emb = O.embedding(sd, cfg, speech, bf16_points=True, split_conv0=True)
    assert emb.shape[0] == 100
    for w, s in ((w0, 0), (w1, 80)):
        ref = O.windows(emb, 33, s)
        assert (w - ref).abs().mean().item() / ref.std().item() < 6e-3          # measured 0.44 %
    assert torch.equal(w1[0, -1, -1], w1[0, -1, 0]) or w1.shape[1] + 80 - 1 > 99          # end clamp reached
    assert torch.equal(w0[0, 0, 0], w0[0, 0, 2])                                              # start clamp
    with pytest.raises(FileNotFoundError, match="not found"):
        SVITalkVideoPipeline(device="cpu", wav2vec_path=str(tmp_path / "nowhere")).get_audio_embedding(wav, 5)


def test_checkpoint_config_is_plain_json(tmp_path):
    d = SA.write_checkpoint(str(tmp_path / "w2v"), SA.TINY, SA.make_state_dict(SA.TINY, seed=0))
    with open(os.path.join(d, "config.json")) as f:
        c = json.load(f)
    assert c["feat_extract_norm"] == "group" and c["model_type"] == "wav2vec2"
