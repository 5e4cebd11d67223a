"""CPU oracle of the wav2vec2 audio feature extractor — TEST INFRASTRUCTURE ONLY.

Only tests/ and tools/ may import this module; the product path (stable-video-infinity_b200/) never does.  Plain torch
fp32 restatement of what the reference computes from a waveform (utils/audio_process.py:18-41 get_embedding,
utils/src/audio_analysis/wav2vec2.py Wav2Vec2Model.forward, torch_utils.py:16-19 linear_interpolation, and the
transformers Wav2Vec2 modules it builds on for feat_extract_norm="group", do_stable_layer_norm=False, gelu):

  Wav2Vec2FeatureExtractor   (x - mean) / sqrt(var + 1e-7)
  feature encoder            conv 0 -> GroupNorm(groups = channels) -> GELU, convs 1..6 -> GELU (no conv bias)
  linear_interpolation       50 Hz -> seq_len frames, F.interpolate(mode='linear', align_corners=True)
  feature projection         LayerNorm -> Linear
  encoder                    + GELU(grouped pos conv, weight norm over dim 2, last output dropped) -> LayerNorm ->
                             post-LN layers [attention -> + -> LayerNorm -> FFN(GELU) -> + -> LayerNorm]

Parity pinned: tests/golden/wav2vec_tiny.npz holds the outputs of the reference module itself on a seeded tiny config
(tests/golden/make_golden_audio.py); tests/test_audio_cpu.py holds this file to it.
"""
import numpy as np
import torch
import torch.nn.functional as F

POS_G, POS_V = "encoder.pos_conv_embed.conv.parametrizations.weight.original0", "encoder.pos_conv_embed.conv.parametrizations.weight.original1"


def _r(x, on):
    """Round to bf16 and back when `on`: the `bf16_points=True` mode applies it exactly where the native path stores a
    bf16 tensor (GEMM operands and bf16 GEMM outputs, attention output); conv outputs feeding a norm, statistics, the
    residual stream and every norm stay fp32."""
    return x.to(torch.bfloat16).float() if on else x


def normalize(speech):
    """Wav2Vec2FeatureExtractor with do_normalize=True on one float32 waveform (numpy, as transformers computes it)."""
    x = np.asarray(speech, dtype=np.float32)
    return (x - x.mean()) / np.sqrt(x.var() + 1e-7)


def seq_len_for(n_samples, sr=16000):
    """get_embedding :19-20,31: int(duration * 25), video frames at 25 fps."""
    return int(n_samples / sr * 25)


def pos_conv_weight(sd):
    """torch weight norm over dim 2: w[:, :, k] = g[k] * v[:, :, k] / ||v[:, :, k]||."""
    return torch._weight_norm(sd[POS_V].float(), sd[POS_G].float(), 2)


def conv_stack(sd, cfg, x, bf16_points=False, split_conv0=False):
    """Feature encoder on input values [n] -> channels-last features f32 [T, conv_dim[-1]].  split_conv0: conv 0's operand
    is kept in fp32 (the native two-term hi/lo form) instead of being rounded to bf16."""
    b = bf16_points
    h = torch.as_tensor(x).float().view(1, 1, -1)
    h = _r(h, b and not split_conv0)
    n = len(cfg["conv_dim"])
    for i in range(n):
        w = sd[f"feature_extractor.conv_layers.{i}.conv.weight"].float()
        h = F.conv1d(h, w, stride=cfg["conv_stride"][i])
        if i == 0:
            h = F.group_norm(h, cfg["conv_dim"][0], sd["feature_extractor.conv_layers.0.layer_norm.weight"].float(),
                             sd["feature_extractor.conv_layers.0.layer_norm.bias"].float(), eps=1e-5)
        h = F.gelu(h)
        if i < n - 1:
            h = _r(h, b)                       # the next conv's operand (GN output / bf16 GEMM output)
    return h[0].t().contiguous()


def interpolate(feat, seq_len):
    """torch_utils.linear_interpolation on channels-last [T_in, C] -> [seq_len, C]."""
    return F.interpolate(feat.t().unsqueeze(0), size=seq_len, align_corners=True, mode="linear")[0].t().contiguous()


def encode(sd, cfg, feat, bf16_points=False):
    """feature projection + encoder on interpolated features [T, C] -> list of num_hidden_layers + 1 hidden states [T, d]."""
    b = bf16_points
    g = lambda k: sd[k].float()
    d, H = cfg["hidden_size"], cfg["num_attention_heads"]
    eps = cfg["layer_norm_eps"]
    T = feat.shape[0]
    h = _r(F.layer_norm(feat, (feat.shape[1],), g("feature_projection.layer_norm.weight"), g("feature_projection.layer_norm.bias"), eps), b)
    h = h @ g("feature_projection.projection.weight").T + g("feature_projection.projection.bias")
    k = cfg["num_conv_pos_embeddings"]
    pos = F.conv1d(_r(h, b).t().unsqueeze(0), pos_conv_weight(sd), g("encoder.pos_conv_embed.conv.bias"), padding=k // 2,
                   groups=cfg["num_conv_pos_embedding_groups"])
    if k % 2 == 0:
        pos = pos[:, :, :-1]                                           # Wav2Vec2SamePadLayer
    h = h + F.gelu(pos)[0].t()
    h = F.layer_norm(h, (d,), g("encoder.layer_norm.weight"), g("encoder.layer_norm.bias"), eps)
    states = [h]
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layers.{i}."
        a = _r(h, b)
        q, kk, v = (_r(a @ g(p + f"attention.{n}_proj.weight").T + g(p + f"attention.{n}_proj.bias"), b).view(T, H, d // H).transpose(0, 1)
                    for n in ("q", "k", "v"))
        o = F.softmax(q @ kk.transpose(-1, -2) * (d // H) ** -0.5, dim=-1) @ v
        o = _r(o.transpose(0, 1).reshape(T, d), b)
        h = h + o @ g(p + "attention.out_proj.weight").T + g(p + "attention.out_proj.bias")
        h = F.layer_norm(h, (d,), g(p + "layer_norm.weight"), g(p + "layer_norm.bias"), eps)
        m = _r(F.gelu(_r(h, b) @ g(p + "feed_forward.intermediate_dense.weight").T + g(p + "feed_forward.intermediate_dense.bias")), b)
        h = h + m @ g(p + "feed_forward.output_dense.weight").T + g(p + "feed_forward.output_dense.bias")
        h = F.layer_norm(h, (d,), g(p + "final_layer_norm.weight"), g(p + "final_layer_norm.bias"), eps)
        states.append(h)
    return states


def forward(sd, cfg, input_values, seq_len, bf16_points=False, split_conv0=False):
    """Wav2Vec2Model.forward of the reference subclass: hidden states (list of [T, d]) for normalised input values [n]."""
    return encode(sd, cfg, interpolate(conv_stack(sd, cfg, input_values, bf16_points, split_conv0), seq_len), bf16_points)


def embedding(sd, cfg, speech, sr=16000, bf16_points=False, split_conv0=False):
    """get_embedding :18-41 on a 16 kHz waveform: [T, num_hidden_layers, d] (hidden_states[1:], frame-major)."""
    states = forward(sd, cfg, normalize(speech), seq_len_for(len(speech), sr), bf16_points, split_conv0)
    return torch.stack(states[1:], dim=1)


def windows(emb, num_frames, start):
    """SVITalkVideoPipeline.get_audio_embedding :412-430: 5-frame windows centred on start .. start + num_frames - 1,
    indices clamped to [0, T-1] -> [1, num_frames, 5, L, d]."""
    idx = torch.arange(start, start + num_frames).unsqueeze(1) + (torch.arange(5) - 2).unsqueeze(0)
    idx = idx.clamp(0, emb.shape[0] - 1)
    return emb[idx][None]
