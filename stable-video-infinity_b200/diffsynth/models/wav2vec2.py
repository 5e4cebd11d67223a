"""wav2vec2 audio feature extractor of SVI-Talk (the "base" Wav2Vec2Model the reference loads from
`./weights/chinese-wav2vec2-base/`) — host side.

Same parameter names as the Hugging Face ``Wav2Vec2Model`` that the reference subclasses
(utils/src/audio_analysis/wav2vec2.py), so its checkpoint directories load unchanged.  Supported: the configuration of the
base models — ``feat_extract_norm="group"`` (GroupNorm with groups = channels after the first conv only),
``do_stable_layer_norm=False`` (post-LN encoder), GELU activations, no conv bias.

``Wav2Vec2Engine`` runs the arithmetic on the kernel library, channels-last ([time, channels]):

  * each feature-encoder conv is an im2col operand (``svi_conv1d_gather``; the kernel-2 / stride-2 layers read the previous
    output in place as [T/2, 2C]) times the (tap, channel)-packed weight on ``svi_gemm_bf16`` with the GELU(erf) epilogue;
    conv 0's GroupNorm is ``svi_col_stats`` (reproducible fp64 column reduction) + ``svi_col_norm_act``;
  * the 50 Hz -> 25 Hz interpolation and the feature projection's LayerNorm are one ``svi_interp_layernorm``;
  * the positional conv is one gather + GEMM per group (bias, GELU and the residual add fused), its weight norm folded at
    build time;
  * every encoder layer is a fused q|k|v GEMM, ``svi_attn_small`` (head_dim 64, scale 1/8), GEMMs with bias / GELU /
    residual epilogues and two ``svi_layernorm_f32`` into the layer-major residual stream [L + 1, T, d], whose slab l is
    hidden state l.

No torch compute fallback.  Numerics: bf16 GEMM operands with fp32 accumulation; fp32 norms, statistics, interpolation
and residual stream (DESIGN.md §2).
"""
import json
import math
import os
import types

import numpy as np
import torch
import torch.nn as nn

from .. import _native as nv

_POS_G = "encoder.pos_conv_embed.conv.parametrizations.weight.original0"
_POS_V = "encoder.pos_conv_embed.conv.parametrizations.weight.original1"
_LEGACY = {"encoder.pos_conv_embed.conv.weight_g": _POS_G, "encoder.pos_conv_embed.conv.weight_v": _POS_V}

_DEFAULTS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, conv_dim=[512] * 7,
                 conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2, 2, 2], num_conv_pos_embeddings=128,
                 num_conv_pos_embedding_groups=16, layer_norm_eps=1e-5, feat_extract_norm="group", do_stable_layer_norm=False,
                 hidden_act="gelu", feat_extract_activation="gelu", conv_bias=False)

# conv 0's operand is the normalised waveform; its bf16 rounding is the largest single operand error of the extractor, and
# the GEMM (K = 10) is small, so it is fed in the two-term hi/lo form (DESIGN.md §2, rounding study of the extractor)
SPLIT_CONV0 = True


def check_config(cfg):
    """Full config dict (defaults filled in) of a supported model; ValueError naming the first unsupported field."""
    c = dict(_DEFAULTS)
    c.update({k: v for k, v in cfg.items() if k in _DEFAULTS})
    for field, want in (("feat_extract_norm", "group"), ("do_stable_layer_norm", False), ("hidden_act", "gelu"),
                        ("feat_extract_activation", "gelu"), ("conv_bias", False)):
        if c[field] != want:
            raise ValueError(f"wav2vec2: unsupported config {field}={c[field]!r} (only {want!r} is implemented: the base "
                             f"models with a GroupNorm feature encoder and a post-LN encoder)")
    if not (len(c["conv_dim"]) == len(c["conv_kernel"]) == len(c["conv_stride"])):
        raise ValueError("wav2vec2: conv_dim, conv_kernel and conv_stride must have the same length")
    if c["hidden_size"] % c["num_attention_heads"] or c["hidden_size"] % c["num_conv_pos_embedding_groups"]:
        raise ValueError("wav2vec2: hidden_size must divide by num_attention_heads and num_conv_pos_embedding_groups")
    return c


class _FeatureEncoder(nn.Module):
    def __init__(self, c):
        super().__init__()
        layers = []
        for i, (cd, k, s) in enumerate(zip(c["conv_dim"], c["conv_kernel"], c["conv_stride"])):
            m = nn.Module()
            m.conv = nn.Conv1d(1 if i == 0 else c["conv_dim"][i - 1], cd, k, stride=s, bias=False)
            if i == 0:
                m.layer_norm = nn.GroupNorm(cd, cd, affine=True)
            layers.append(m)
        self.conv_layers = nn.ModuleList(layers)


class _EncoderLayer(nn.Module):
    def __init__(self, d, f, eps):
        super().__init__()
        self.attention = nn.Module()
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            setattr(self.attention, n, nn.Linear(d, d))
        self.layer_norm = nn.LayerNorm(d, eps=eps)
        self.feed_forward = nn.Module()
        self.feed_forward.intermediate_dense = nn.Linear(d, f)
        self.feed_forward.output_dense = nn.Linear(f, d)
        self.final_layer_norm = nn.LayerNorm(d, eps=eps)


class Wav2Vec2Model(nn.Module):
    """Parameter container with the Hugging Face names; ``forward`` runs on the CUDA engine."""

    def __init__(self, config):
        super().__init__()
        c = check_config(config)
        self.config = types.SimpleNamespace(**c)
        d, eps = c["hidden_size"], c["layer_norm_eps"]
        self.feature_extractor = _FeatureEncoder(c)
        self.feature_projection = nn.Module()
        self.feature_projection.layer_norm = nn.LayerNorm(c["conv_dim"][-1], eps=eps)
        self.feature_projection.projection = nn.Linear(c["conv_dim"][-1], d)
        self.encoder = nn.Module()
        self.encoder.pos_conv_embed = nn.Module()
        k = c["num_conv_pos_embeddings"]
        conv = nn.Conv1d(d, d, k, padding=k // 2, groups=c["num_conv_pos_embedding_groups"])
        self.encoder.pos_conv_embed.conv = nn.utils.parametrizations.weight_norm(conv, name="weight", dim=2)
        self.encoder.layer_norm = nn.LayerNorm(d, eps=eps)
        self.encoder.layers = nn.ModuleList([_EncoderLayer(d, c["intermediate_size"], eps) for _ in range(c["num_hidden_layers"])])
        self.masked_spec_embed = nn.Parameter(torch.zeros(d))          # SpecAugment (training only); kept for the key set
        self._engine = None

    @staticmethod
    def from_pretrained(path, device="cpu"):
        """config.json + model.safetensors or pytorch_model.bin of a Wav2Vec2Model (bare keys or under `wav2vec2.`, as in
        a pretraining checkpoint whose quantizer / project_* heads are ignored); the positional conv's weight norm may be
        stored as weight_g / weight_v or parametrizations.weight.original0 / 1."""
        cfg_path = os.path.join(path, "config.json")
        if not os.path.isfile(cfg_path):
            raise FileNotFoundError(f"wav2vec2: no config.json in {path!r}")
        with open(cfg_path) as f:
            model = Wav2Vec2Model(json.load(f))
        st, bn = os.path.join(path, "model.safetensors"), os.path.join(path, "pytorch_model.bin")
        if os.path.isfile(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        elif os.path.isfile(bn):
            sd = torch.load(bn, map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"wav2vec2: neither model.safetensors nor pytorch_model.bin in {path!r}")
        model.load_state_dict(convert_state_dict(sd, model.state_dict().keys()))
        return model.to(device).eval()

    def engine(self, device=None):
        p = self.feature_extractor.conv_layers[0].conv.weight
        dev = torch.device(device) if device is not None else p.device
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        sig = (str(dev), p.data_ptr(), p._version, self.encoder.layers[-1].final_layer_norm.weight.data_ptr())
        if self._engine is None or self._engine[0] != sig:
            self._engine = (sig, Wav2Vec2Engine(self, dev))
        return self._engine[1]

    def forward(self, input_values, seq_len, output_hidden_states=True):
        """The reference subclass's forward (wav2vec2.py:13-64) without masks: normalised input values [1, n] -> an object
        with ``last_hidden_state`` [1, seq_len, d] and ``hidden_states`` (num_hidden_layers + 1 tensors [1, seq_len, d])."""
        return self.engine().forward(input_values, seq_len, output_hidden_states)


def convert_state_dict(sd, wanted):
    """Checkpoint keys -> this module's keys: strip a `wav2vec2.` prefix, rename the legacy weight-norm pair, drop keys the
    model does not have (pretraining heads).  Missing keys are an error (masked_spec_embed, training-only, defaults to 0)."""
    wanted = set(wanted)
    if any(k.startswith("wav2vec2.") for k in sd):
        sd = {k[len("wav2vec2."):]: v for k, v in sd.items() if k.startswith("wav2vec2.")}
    out = {_LEGACY.get(k, k): v for k, v in sd.items()}
    out = {k: v for k, v in out.items() if k in wanted}
    out.setdefault("masked_spec_embed", torch.zeros_like(out.get("encoder.layer_norm.bias", torch.zeros(1))))
    missing = sorted(wanted - set(out))
    if missing:
        raise KeyError(f"wav2vec2: checkpoint lacks {len(missing)} parameters, e.g. {missing[:4]}")
    return out


class Wav2Vec2FeatureExtractor:
    """The part of transformers' Wav2Vec2FeatureExtractor the reference uses (one unpadded waveform):
    float32 input values, normalised to (x - mean) / sqrt(var + 1e-7) when do_normalize."""

    def __init__(self, do_normalize=True, sampling_rate=16000):
        self.do_normalize, self.sampling_rate = bool(do_normalize), int(sampling_rate)

    @staticmethod
    def from_pretrained(path):
        p = os.path.join(path, "preprocessor_config.json")
        if not os.path.isfile(p):
            raise FileNotFoundError(f"wav2vec2: no preprocessor_config.json in {path!r}")
        with open(p) as f:
            c = json.load(f)
        return Wav2Vec2FeatureExtractor(c.get("do_normalize", True), c.get("sampling_rate", 16000))

    def __call__(self, speech, sampling_rate=None):
        if sampling_rate is not None and int(sampling_rate) != self.sampling_rate:
            raise ValueError(f"wav2vec2: the feature extractor expects {self.sampling_rate} Hz input, got {sampling_rate}")
        x = np.asarray(speech, dtype=np.float32).reshape(-1)
        if self.do_normalize:
            x = (x - x.mean()) / np.sqrt(x.var() + 1e-7)
        return types.SimpleNamespace(input_values=x[None])


class Wav2Vec2Output:
    """``last_hidden_state`` [1, T, d] and ``hidden_states`` (L + 1 views [1, T, d]) of the layer-major buffer ``stacked``."""

    def __init__(self, stacked, output_hidden_states):
        self.stacked = stacked
        self.last_hidden_state = stacked[-1].unsqueeze(0)
        self.hidden_states = tuple(s.unsqueeze(0) for s in stacked) if output_hidden_states else None

    def __len__(self):
        return 2 if self.hidden_states is not None else 1


def _ceil8(n):
    return (n + 7) // 8 * 8


def _conv_out_len(n, k, s, pad=0):
    return (n + 2 * pad - k) // s + 1


class Wav2Vec2Engine:
    def __init__(self, model: Wav2Vec2Model, device):
        nv.require_cuda(device, "the wav2vec2 audio encoder")
        self.device = torch.device(device)
        c = vars(model.config)
        self.cfg = c
        self.d, self.H = c["hidden_size"], c["num_attention_heads"]
        self.hd = self.d // self.H
        self.eps = c["layer_norm_eps"]
        self.groups = c["num_conv_pos_embedding_groups"]
        self.dg = self.d // self.groups
        if self.dg % 8:
            raise ValueError(f"wav2vec2 engine: hidden_size / num_conv_pos_embedding_groups = {self.dg} must be a multiple of 8 "
                             f"(the GEMM's N granularity; 48 for base, 64 for large models)")
        bf = lambda t: t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        fe = model.feature_extractor
        # conv weights [Cout, Cin, k] -> [Cout, Kpad] in (tap, channel) order, the column order of the im2col operand
        self.convs = []
        for i, layer in enumerate(fe.conv_layers):
            w = layer.conv.weight.detach().float().cpu()
            co, ci, k = w.shape
            kp = _ceil8(k * ci)
            wp = torch.zeros(co, kp)
            wp[:, :k * ci] = w.permute(0, 2, 1).reshape(co, k * ci)
            split = i == 0 and SPLIT_CONV0
            if split:
                wp = torch.cat([wp, wp], dim=1)                       # [W | W] against the operand's [hi | lo] columns
            self.convs.append(dict(w=bf(wp), k=k, s=layer.conv.stride[0], cin=ci, cout=co, kpad=kp, split=split))
        self.gn_w, self.gn_b = f32(fe.conv_layers[0].layer_norm.weight), f32(fe.conv_layers[0].layer_norm.bias)
        self.gn_eps = fe.conv_layers[0].layer_norm.eps
        fp = model.feature_projection
        self.fp_ln_w, self.fp_ln_b = f32(fp.layer_norm.weight), f32(fp.layer_norm.bias)
        self.w_proj, self.b_proj = bf(fp.projection.weight), f32(fp.projection.bias)
        # positional conv: weight norm folded (w = g * v / ||v|| over dims 0, 1 per tap), one packed weight per group
        pc = model.encoder.pos_conv_embed.conv
        with torch.no_grad():
            w = torch._weight_norm(pc.parametrizations.weight.original1.detach().float().cpu(),
                                   pc.parametrizations.weight.original0.detach().float().cpu(), 2)      # [d, dg, k]
        self.pos_k = w.shape[2]
        self.pos_kpad = _ceil8(self.pos_k * self.dg)
        wp = torch.zeros(self.d, self.pos_kpad)
        wp[:, :self.pos_k * self.dg] = w.permute(0, 2, 1).reshape(self.d, self.pos_k * self.dg)
        self.w_pos, self.b_pos = bf(wp), f32(pc.bias)
        self.enc_ln_w, self.enc_ln_b = f32(model.encoder.layer_norm.weight), f32(model.encoder.layer_norm.bias)
        self.layers = []
        for ly in model.encoder.layers:
            a = ly.attention
            self.layers.append(dict(
                w_qkv=bf(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)),
                b_qkv=f32(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0)),
                w_o=bf(a.out_proj.weight), b_o=f32(a.out_proj.bias),
                ln1_w=f32(ly.layer_norm.weight), ln1_b=f32(ly.layer_norm.bias),
                w_ff1=bf(ly.feed_forward.intermediate_dense.weight), b_ff1=f32(ly.feed_forward.intermediate_dense.bias),
                w_ff2=bf(ly.feed_forward.output_dense.weight), b_ff2=f32(ly.feed_forward.output_dense.bias),
                ln2_w=f32(ly.final_layer_norm.weight), ln2_b=f32(ly.final_layer_norm.bias)))
        self.ffn = self.layers[0]["w_ff1"].shape[0] if self.layers else 0
        self.launches = 0

    def feature_length(self, n_samples):
        """Frames at the feature encoder's output (50 Hz) for n input samples."""
        T = n_samples
        for cv in self.convs:
            T = _conv_out_len(T, cv["k"], cv["s"])
        return T

    def features(self, input_values):
        """Feature encoder: normalised input values (any shape with n elements) -> f32 [T, conv_dim[-1]] (GELU applied)."""
        dev = self.device
        x = torch.as_tensor(input_values).to(device=dev, dtype=torch.float32).reshape(-1, 1).contiguous()
        if self.feature_length(x.shape[0]) < 1:
            raise ValueError(f"wav2vec2: {x.shape[0]} samples are too short for the feature encoder")
        h, T = x, x.shape[0]
        last = len(self.convs) - 1
        for i, cv in enumerate(self.convs):
            k, s, C = cv["k"], cv["s"], cv["cin"]
            To = _conv_out_len(T, k, s)
            if i > 0 and k == s and k * C == cv["kpad"]:
                a = h[:To * k].view(To, k * C)                        # non-overlapping taps: the previous output read in place
            else:
                a = torch.empty(To, cv["kpad"] * (2 if cv["split"] else 1), device=dev, dtype=torch.bfloat16)
                nv.conv1d_gather(h, a, k, s, split=cv["split"])
                self.launches += 1
            if i == 0:
                y = torch.empty(To, cv["cout"], device=dev, dtype=torch.float32)
                nv.gemm(a, cv["w"], y)
                mean = torch.empty(cv["cout"], device=dev, dtype=torch.float32)
                var = torch.empty_like(mean)
                ws = torch.empty(nv.col_stats_workspace_bytes(To, cv["cout"]), device=dev, dtype=torch.uint8)
                nv.col_stats(y, mean, var, ws)
                h = torch.empty(To, cv["cout"], device=dev, dtype=torch.bfloat16)
                nv.col_norm_act(y, mean, var, self.gn_eps, self.gn_w, self.gn_b, nv.ACT_GELU_ERF, h)
                self.launches += 3
            else:
                h = torch.empty(To, cv["cout"], device=dev, dtype=torch.float32 if i == last else torch.bfloat16)
                nv.gemm(a, cv["w"], h, act=nv.ACT_GELU_ERF)
                self.launches += 1
            T = To
        return h

    def encode(self, feats, seq_len):
        """feature projection + encoder on the 50 Hz features f32 [T_in, C]: -> f32 [L + 1, seq_len, d], slab 0 the input
        of layer 0 (after the positional conv and LayerNorm), slab l the output of layer l."""
        dev, d, T = self.device, self.d, int(seq_len)
        if T < 1:
            raise ValueError(f"wav2vec2: seq_len must be >= 1, got {seq_len}")
        L = len(self.layers)
        a = torch.empty(T, feats.shape[1], device=dev, dtype=torch.bfloat16)
        nv.interp_layernorm(feats, T, self.fp_ln_w, self.fp_ln_b, self.eps, a)
        h0 = torch.empty(T, d, device=dev, dtype=torch.float32)
        nv.gemm(a, self.w_proj, h0, bias=self.b_proj)
        # positional conv (grouped, 'same' padding with the last output dropped): per group an im2col of its channel window
        # and a GEMM whose epilogue adds bias, applies GELU and adds the residual h0
        tmp = torch.empty(T, d, device=dev, dtype=torch.float32)
        cols = torch.empty(T, self.pos_kpad, device=dev, dtype=torch.bfloat16)
        pad = self.pos_k // 2
        for g in range(self.groups):
            c0, c1 = g * self.dg, (g + 1) * self.dg
            nv.conv1d_gather(h0, cols, self.pos_k, 1, pad, pad, col0=c0, C=self.dg)
            nv.gemm(cols, self.w_pos[c0:c1], tmp[:, c0:c1], bias=self.b_pos[c0:c1], act=nv.ACT_GELU_ERF, residual=h0[:, c0:c1])
        hs = torch.empty(L + 1, T, d, device=dev, dtype=torch.float32)
        nv.layernorm_f32(tmp, self.enc_ln_w, self.enc_ln_b, self.eps, hs[0])
        xb = torch.empty(T, d, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(T, 3 * d, device=dev, dtype=torch.bfloat16)
        att = torch.empty(T, d, device=dev, dtype=torch.bfloat16)
        mid = torch.empty(T, d, device=dev, dtype=torch.float32)
        m = torch.empty(T, self.ffn, device=dev, dtype=torch.bfloat16)
        scale = 1.0 / math.sqrt(self.hd)
        for i, ly in enumerate(self.layers):
            x = hs[i]
            nv.cast_f32_to_bf16(x, xb)
            nv.gemm(xb, ly["w_qkv"], qkv, bias=ly["b_qkv"])
            nv.attention_small(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], att, self.H, self.hd, scale)
            nv.gemm(att, ly["w_o"], tmp, bias=ly["b_o"], residual=x)
            nv.layernorm_f32(tmp, ly["ln1_w"], ly["ln1_b"], self.eps, mid)
            nv.cast_f32_to_bf16(mid, xb)
            nv.gemm(xb, ly["w_ff1"], m, bias=ly["b_ff1"], act=nv.ACT_GELU_ERF)
            nv.gemm(m, ly["w_ff2"], tmp, bias=ly["b_ff2"], residual=mid)
            nv.layernorm_f32(tmp, ly["ln2_w"], ly["ln2_b"], self.eps, hs[i + 1])
        self.launches += 4 + 2 * self.groups + 9 * L
        return hs

    def forward(self, input_values, seq_len, output_hidden_states=True):
        return Wav2Vec2Output(self.encode(self.features(input_values), seq_len), output_hidden_states)
