"""Regenerate tests/golden/reward_tiny.npz from the REAL reference modules (run on a machine with the reference tree):

    python tests/golden/make_golden_reward.py /path/to/reference

The reference's ImageQualityMetric directory is imported as a package under another name, so its ``__init__`` (which
imports modelscope) does not run.  Modules used as they are: ``BLIP/vit.VisionTransformer``, ``BLIP/med.BertModel``,
``BLIP/blip.init_tokenizer``, ``imagereward.MLP`` and ``_transform``, ``trainer/models/clip_model.XCLIPModel`` and
``CLIPModel``, ``trainer/models/cross_modeling.Cross_model``; the scores come from the reference's own
``ImageReward._calculate_score`` and ``MPScore._calculate_score``, called on objects made with ``__new__`` and given the
tiny parts (their constructors load fixed full-size files).

Import shims, none of which restates model math:
* ``timm`` is not installed; a stand-in package provides what BLIP imports: ``PatchEmbed`` (timm's: a Conv2d with bias,
  then flatten and transpose to [B, N, C]), ``DropPath`` (the identity, as in eval), ``trunc_normal_``
  (torch.nn.init.trunc_normal_), and no-op ``_cfg``, ``register_model``, ``named_apply``, ``adapt_input_conv``,
  ``download_cached_file`` (never called here);
* ``apply_chunking_to_forward`` and ``prune_linear_layer`` are taken from ``transformers.pytorch_utils`` into
  ``transformers.modeling_utils``, where med.py imports them from; ``find_pruneable_heads_and_indices`` is a no-op
  (pruning is never used);
* ``BertPreTrainedModel.init_weights`` is ``self.apply(self._init_weights)`` (every weight is overwritten by the seeded
  state dict afterwards), and ``BertModel.get_head_mask`` returns ``[None] * n`` (no head mask, as the reference's
  calls pass none);
* ``invert_attention_mask`` is added only when the installed transformers lacks it;
* ``transformers.CLIPFeatureExtractor`` (imported, never used by mps.py) is ``CLIPImageProcessor`` where missing;
* ``BertTokenizer.additional_special_tokens_ids``, which BLIP's ``init_tokenizer`` reads, is the ids of the tokenizer's
  ``extra_special_tokens`` where the installed transformers lacks the property.
Records: the BERT ids and masks (synthetic ``vocab.txt``), the CLIP ids of the prompts and conditions, the host pixels
(unnormalised; ImageReward's 224 x 224 ones and its normalised inputs as SHA-256 digests of their f32 bytes) and the
exact inputs MPS saw, four rows of each BLIP image state, the BERT [CLS] rows, MPS's text_f, cond_f, mask
ratio and keep, cross features and the scores.
"""
import hashlib
import importlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stable-video-infinity_b200")]
from tools import synth_reward as R  # noqa: E402

CONDITIONS = ("overall", "semantic")
STATE_ROWS = [0, 1, 98, 196]          # the rows of the BLIP image states kept in the fixture


def install_shims():
    import transformers
    import transformers.modeling_utils as mu
    import transformers.pytorch_utils as pu

    class PatchEmbed(torch.nn.Module):
        def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768):
            super().__init__()
            self.num_patches = (img_size // patch_size) ** 2
            self.proj = torch.nn.Conv2d(in_chans, embed_dim, patch_size, patch_size)

        def forward(self, x):
            return self.proj(x).flatten(2).transpose(1, 2)

    class DropPath(torch.nn.Identity):
        def __init__(self, *a, **k):
            super().__init__()

    noop = lambda *a, **k: None
    mods = {"timm": {}, "timm.models": {}, "timm.models.hub": dict(download_cached_file=noop),
            "timm.models.vision_transformer": dict(_cfg=noop, PatchEmbed=PatchEmbed),
            "timm.models.registry": dict(register_model=lambda f: f),
            "timm.models.layers": dict(trunc_normal_=torch.nn.init.trunc_normal_, DropPath=DropPath),
            "timm.models.helpers": dict(named_apply=noop, adapt_input_conv=noop)}
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    mu.apply_chunking_to_forward = pu.apply_chunking_to_forward
    mu.prune_linear_layer = pu.prune_linear_layer
    mu.find_pruneable_heads_and_indices = noop
    image_processor = transformers.CLIPImageProcessor
    tf_mod = sys.modules["transformers"]          # resolving a lazy name can replace the module object in sys.modules
    if "CLIPFeatureExtractor" not in dir(tf_mod):
        tf_mod.CLIPFeatureExtractor = image_processor
    from transformers import BertTokenizer
    if not hasattr(BertTokenizer, "additional_special_tokens_ids"):
        BertTokenizer.additional_special_tokens_ids = property(
            lambda self: self.convert_tokens_to_ids(list(self.extra_special_tokens)))


def load_reference(ref):
    install_shims()
    pkg = types.ModuleType("ref_iqm")
    pkg.__path__ = [os.path.join(ref, "diffsynth", "extensions", "ImageQualityMetric")]
    sys.modules["ref_iqm"] = pkg
    med = importlib.import_module("ref_iqm.BLIP.med")
    med.BertPreTrainedModel.init_weights = lambda self: self.apply(self._init_weights)
    med.BertModel.get_head_mask = lambda self, head_mask, n, *a, **k: [None] * n
    if not hasattr(med.BertModel, "invert_attention_mask"):
        def invert_attention_mask(self, m):
            return (1.0 - m[:, None, None, :].to(self.dtype)) * torch.finfo(self.dtype).min
        med.BertModel.invert_attention_mask = invert_attention_mask
    return (med, importlib.import_module("ref_iqm.BLIP.vit"), importlib.import_module("ref_iqm.BLIP.blip"),
            importlib.import_module("ref_iqm.imagereward"), importlib.import_module("ref_iqm.mps"),
            importlib.import_module("ref_iqm.trainer.models.clip_model"),
            importlib.import_module("ref_iqm.trainer.models.cross_modeling"))


def main(ref):
    med_m, vit_m, blip_m, ir_m, mps_m, clip_m, cross_m = load_reference(ref)
    from transformers import AutoTokenizer, CLIPConfig, CLIPImageProcessor
    from transformers.models.bert.configuration_bert import BertConfig
    torch.manual_seed(0)
    d = tempfile.mkdtemp()
    paths, tiny = R.write_reward_checkpoints(d)
    out = {}
    frames = R.frames()

    # ---------------------------------------------------------------------------------------------- ImageReward
    med, sd = tiny["imagereward"]
    v = R.TINY_VISION
    vis = vit_m.VisionTransformer(img_size=v["image_size"], patch_size=v["patch"], embed_dim=v["width"], depth=v["layers"],
                                  num_heads=v["width"] // 64, mlp_ratio=v["mlp_width"] / v["width"])
    vis.load_state_dict({k[len("blip.visual_encoder."):]: t for k, t in sd.items() if k.startswith("blip.visual_encoder.")})
    conf = BertConfig.from_json_file(paths["med_config"])
    conf.encoder_width = v["width"]
    bert = med_m.BertModel(config=conf, add_pooling_layer=False)
    bert.load_state_dict({k[len("blip.text_encoder."):]: t for k, t in sd.items() if k.startswith("blip.text_encoder.")})
    mlp = ir_m.MLP(med["hidden_size"])
    mlp.load_state_dict({k[len("mlp."):]: t for k, t in sd.items() if k.startswith("mlp.")})
    blip = torch.nn.Module()
    blip.visual_encoder, blip.text_encoder = vis.eval(), bert.eval()
    blip.tokenizer = blip_m.init_tokenizer(paths["bert_model_path"])
    model = ir_m.ImageReward.__new__(ir_m.ImageReward)
    torch.nn.Module.__init__(model)
    model.device, model.blip, model.mlp = torch.device("cpu"), blip, mlp.eval()
    model.mean, model.std = 0.16717362830052426, 1.0333394966054072
    tf = ir_m._transform(224)
    host = torch.stack([_compose(tf.transforms[:-1])(f) for f in frames]).numpy()
    out["blip_pixels_sha256"] = np.array(hashlib.sha256(host.tobytes()).hexdigest())     # the f32 bytes, [4, 3, 224, 224]
    px = torch.stack([tf(f) for f in frames])
    out["blip_inputs_sha256"] = np.array(hashlib.sha256(px.numpy().tobytes()).hexdigest())
    for i, p in enumerate(R.PROMPTS):
        t = blip.tokenizer(p, padding="max_length", truncation=True, max_length=35, return_tensors="pt")
        out[f"bert_ids_{i}"], out[f"bert_mask_{i}"] = t.input_ids.numpy(), t.attention_mask.numpy()
    with torch.no_grad():
        img = vis(px)
        out["blip_image_states"] = img[:, STATE_ROWS].numpy()
        for i in (0, 1):
            ids, mask = torch.from_numpy(out[f"bert_ids_{i}"]), torch.from_numpy(out[f"bert_mask_{i}"])
            o = bert(ids.expand(len(frames), -1), attention_mask=mask.expand(len(frames), -1), encoder_hidden_states=img,
                     encoder_attention_mask=torch.ones(img.shape[:-1], dtype=torch.long), return_dict=True)
            out[f"bert_cls_{i}"] = o.last_hidden_state[:, 0].numpy()
            out[f"imagereward_scores_{i}"] = np.array([model._calculate_score(R.PROMPTS[i], px[j:j + 1]).item()
                                                       for j in range(len(frames))], dtype=np.float32)

    # ---------------------------------------------------------------------------------------------- MPS
    cconf, msd = tiny["mps"]
    xclip = clip_m.XCLIPModel(CLIPConfig.from_dict(cconf))
    xclip.load_state_dict({k[len("model."):]: t for k, t in msd.items() if k.startswith("model.")})
    heads = max(cconf["projection_dim"] // 64, 2)
    cross = cross_m.Cross_model(dim=cconf["projection_dim"], layer_num=2, dim_head=64, heads=heads, ff_mult=4)
    cross.load_state_dict({k[len("cross_model."):]: t for k, t in msd.items() if k.startswith("cross_model.")}, strict=True)
    cm = clip_m.CLIPModel.__new__(clip_m.CLIPModel)
    torch.nn.Module.__init__(cm)
    cm.model, cm.cross_model = xclip.eval(), cross.eval()
    scorer = mps_m.MPScore.__new__(mps_m.MPScore)
    torch.nn.Module.__init__(scorer)
    scorer.device, scorer.model = torch.device("cpu"), cm
    scorer.image_processor = CLIPImageProcessor.from_pretrained(paths["clip"])
    scorer.tokenizer = AutoTokenizer.from_pretrained(paths["clip"])
    out["mps_pixels"] = torch.cat([scorer.image_processor(f, return_tensors="pt", do_normalize=False)["pixel_values"]
                                   for f in frames]).numpy()
    mpx = torch.cat([scorer.image_processor(f, return_tensors="pt")["pixel_values"] for f in frames])
    out["mps_inputs"] = mpx.half().float().numpy()             # what get_image_features(image.half()) computes on
    tok = lambda c: scorer.tokenizer(c, max_length=scorer.tokenizer.model_max_length, padding="max_length",
                                     truncation=True, return_tensors="pt").input_ids
    for i, p in enumerate(R.PROMPTS):
        out[f"clip_ids_{i}"] = tok(p).numpy()
    for c in CONDITIONS:
        scorer.condition = c
        cond = {"overall": "light, color, clarity, tone, style, ambiance, artistry, shape, face, hair, hands, limbs, "
                           "structure, instance, texture, quantity, attributes, position, number, location, word, things",
                "semantic": "quantity, attributes, position, number, location"}[c]
        out[f"clip_cond_ids_{c}"] = tok(cond).numpy()
        with torch.no_grad():
            ids = torch.from_numpy(out["clip_ids_2"])
            text_f, text_eos = xclip.get_text_features(ids)
            cond_f, _ = xclip.get_text_features(torch.from_numpy(out[f"clip_cond_ids_{c}"]))
            sim = torch.einsum("b i d, b j d -> b j i", text_f, cond_f).max(dim=1, keepdim=True)[0]
            ratio = (sim / sim.max())[0, 0]
            image_f = xclip.get_image_features(mpx.half())
            mask = torch.where(ratio > 0.3, 0, float("-inf"))[None, None].repeat(len(frames), image_f.shape[1], 1)
            feats = cross(image_f, text_f, mask.half())[:, 0]
            out[f"mps_text_f_{c}"], out[f"mps_cond_f_{c}"] = text_f[0].numpy(), cond_f[0].numpy()
            out[f"mps_text_eos_{c}"] = text_eos.numpy()
            out[f"mps_ratio_{c}"], out[f"mps_keep_{c}"] = ratio.numpy(), (ratio > 0.3).numpy()
            out[f"mps_cross_{c}"] = feats.numpy()
            out["mps_image_rows"] = image_f.numpy()
            out[f"mps_scores_{c}"] = np.array([scorer._calculate_score(mpx[j:j + 1], R.PROMPTS[2]) for j in range(len(frames))],
                                              dtype=np.float32)
        print(c, "keys kept", int((ratio > 0.3).sum()), "of", ratio.numel())
    path = os.path.join(ROOT, "tests", "golden", "reward_tiny.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


def _compose(ts):
    def run(x):
        for t in ts:
            x = t(x)
        return x
    return run


if __name__ == "__main__":
    main(sys.argv[1])
