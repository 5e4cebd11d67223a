"""The four scorers with the reference's names, arguments and return values (reference ``clip.py``, ``hps.py``,
``pickscore.py``, ``aesthetic.py``).

``score(images, prompt)`` takes a path, a PIL image or a list of either and returns one float per image.  Underneath,
every image of the call is preprocessed on the host, and the batch goes through the vision tower together (in chunks of
``TowerEngine.chunk``); the prompt is tokenised and encoded once per call.  The score kernel normalises both features
and takes their dot products (or applies the folded aesthetic head) in one launch.
"""
from typing import List, Union

import torch
from PIL import Image

from .config import MODEL_PATHS
from .tokenizer import SimpleTokenizer
from .towers import (AestheticMLP, HFCLIPModel, OpenCLIP, OPENAI_MEAN, OPENAI_STD, VIT_H_14, hf_mean_std, hf_pixels,
                     openclip_pixels)
from ... import _native as nv


def _as_list(images):
    if isinstance(images, (str, Image.Image)):
        return [images]
    if isinstance(images, list):
        return images
    raise TypeError("The type of parameter images is illegal.")


def _open(image):
    if isinstance(image, str):
        return Image.open(image)
    if isinstance(image, Image.Image):
        return image
    raise TypeError("The type of parameter images is illegal.")


def _device(device):
    dev = device if isinstance(device, torch.device) else torch.device(device)
    nv.require_cuda(dev, "ImageQualityMetric")
    return dev


def load_open_clip_state_dict(path):
    """open_clip's load_state_dict: a torch file (optionally {'state_dict': ...}, optionally 'module.'-prefixed) or
    safetensors"""
    if str(path).endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
        if isinstance(sd, dict) and "state_dict" in sd:
            sd = sd["state_dict"]
    if next(iter(sd)).startswith("module"):
        sd = {k[7:]: v for k, v in sd.items()}
    return sd


def openclip_config(sd):
    """open_clip's ViT-H-14 config (head width 80 in the vision tower, 64 in the text tower, GELU), with the sizes read
    from the checkpoint's shapes; a ViT-H-14 checkpoint gives VIT_H_14 itself"""
    n_layers = lambda prefix: len({k.split(".")[len(prefix.split(".")) + 1] for k in sd if k.startswith(prefix + ".resblocks.")})
    grid2 = sd["visual.positional_embedding"].shape[0] - 1
    P = sd["visual.conv1.weight"].shape[-1]
    tw = sd["positional_embedding"].shape[1]
    return dict(embed_dim=sd["text_projection"].shape[1],
                vision_cfg=dict(image_size=int(round(grid2 ** 0.5)) * P, layers=n_layers("visual.transformer"),
                                width=sd["visual.class_embedding"].shape[0], head_width=VIT_H_14["vision_cfg"]["head_width"],
                                patch_size=P),
                text_cfg=dict(context_length=sd["positional_embedding"].shape[0], vocab_size=sd["token_embedding.weight"].shape[0],
                              width=tw, heads=max(tw // 64, 1), layers=n_layers("transformer")))


class _OpenCLIPScorer(torch.nn.Module):
    """image-text cosine of an open_clip ViT-H-14: open_clip's preprocess_val (light augmentation), its BPE tokenizer"""

    def _setup(self, device, state_dict_path, bpe_path):
        self.device = _device(device)
        sd = load_open_clip_state_dict(state_dict_path)
        model = OpenCLIP(**openclip_config(sd)).eval()
        model.load_state_dict(sd, strict=True)
        self.model = model
        self.tokenizer = SimpleTokenizer(bpe_path)
        self.context_length = model.text_cfg["context_length"]

    def features(self, images, prompt):
        """(normalised-on-device) inputs -> (image features f32 [B, E], text features f32 [1, E]) on the device"""
        eng = self.model.engine(self.device, OPENAI_MEAN, OPENAI_STD)
        size = self.model.vision_cfg["image_size"]
        px = torch.stack([openclip_pixels(_open(im), size) for im in _as_list(images)])
        ids = self.tokenizer([prompt], self.context_length)
        with torch.no_grad():
            return eng.vision.encode_images(px), eng.text.encode_text(ids)

    def _score(self, images, prompt):
        img, txt = self.features(images, prompt)
        cos = torch.empty(img.shape[0], 1, device=self.device, dtype=torch.float32)
        nv.quality_score(img, txt, cos)
        return cos[:, 0].tolist()


class CLIPScore(_OpenCLIPScorer):
    """CLIP score of open_clip ViT-H-14 (laion2B-s32B-b79K): the cosine of image and prompt features.  Like the
    reference, errors are not wrapped."""

    def __init__(self, device: torch.device, path: dict = MODEL_PATHS):
        super().__init__()
        self._setup(device, path.get("open_clip"), path["open_clip_bpe"])

    @torch.no_grad()
    def score(self, images: Union[str, List[str], Image.Image, List[Image.Image]], prompt: str) -> List[float]:
        return self._score(images, prompt)


class HPScore_v2(_OpenCLIPScorer):
    """Human Preference Score v2 / v2.1: the cosine of an HPS-fine-tuned open_clip ViT-H-14."""

    def __init__(self, device: torch.device, path: dict = MODEL_PATHS, model_version: str = "v2"):
        super().__init__()
        if model_version == "v2":
            safetensors_path = path.get("hpsv2")
        elif model_version == "v21":
            safetensors_path = path.get("hpsv2.1")
        else:
            raise ValueError(f"Unsupported model version: {model_version}. Choose 'v2' or 'v21'.")
        try:
            self._setup(device, safetensors_path, path["open_clip_bpe"])
        except (RuntimeError, OSError, KeyError) as e:
            raise ValueError(f"Error loading model weights from {safetensors_path}: {e}")

    @torch.no_grad()
    def score(self, images: Union[str, List[str], Image.Image, List[Image.Image]], prompt: str) -> List[float]:
        try:
            return self._score(images, prompt)
        except Exception as e:
            raise RuntimeError(f"Error in scoring images: {e}")


class PickScore(torch.nn.Module):
    """PickScore_v1 (an HF CLIPModel ViT-H/14) with the CLIP-ViT-H-14 processor.  ``softmax=True`` is kept as the
    reference has it: the softmax runs over the one score of each image, so it returns 1.0 for every image."""

    def __init__(self, device: Union[str, torch.device], path: dict = MODEL_PATHS):
        super().__init__()
        from transformers import AutoProcessor
        self.device = _device(device)
        self.processor = AutoProcessor.from_pretrained(path.get("clip"))
        self.model = HFCLIPModel.from_pretrained(path.get("pickscore"))
        self.mean, self.std = hf_mean_std(self.processor)

    def features(self, images, prompt):
        eng = self.model.engine(self.device, self.mean, self.std)
        px = torch.stack([hf_pixels(self.processor, _open(im)) for im in _as_list(images)])
        ids = self.processor(text=prompt, padding=True, truncation=True, max_length=77, return_tensors="pt")["input_ids"]
        with torch.no_grad():
            return eng.vision.encode_images(px), eng.text.encode_text(ids)

    @torch.no_grad()
    def score(self, images: Union[str, List[str], Image.Image, List[Image.Image]], prompt: str,
              softmax: bool = False) -> List[float]:
        try:
            img, txt = self.features(images, prompt)
            cos = torch.empty(img.shape[0], 1, device=self.device, dtype=torch.float32)
            nv.quality_score(img, txt, cos)
            s = cos.cpu()
            if softmax:
                s = torch.softmax(self.model.logit_scale.detach().exp() * s, dim=-1)
            return s[:, 0].tolist()
        except Exception as e:
            raise RuntimeError(f"Error in scoring images: {e}")


class AestheticScore(torch.nn.Module):
    """LAION aesthetic predictor v2 (sac+logos+ava1-l14-linearMSE) on CLIP ViT-L/14 image features.  The head's five
    Linear layers are folded into one 768 -> 1 affine map at load time (fp64 on the host, rounded once)."""

    def __init__(self, device: torch.device, path: dict = MODEL_PATHS):
        super().__init__()
        from transformers import AutoProcessor
        self.device = _device(device)
        self.aes_model_path = path.get("aesthetic_predictor")
        self.mlp = AestheticMLP(768)
        try:
            if self.aes_model_path.endswith(".safetensors"):
                from safetensors.torch import load_file
                state_dict = load_file(self.aes_model_path)
            else:
                state_dict = torch.load(self.aes_model_path, map_location="cpu", weights_only=True)
            self.mlp.load_state_dict(state_dict, strict=True)
        except Exception as e:
            raise ValueError(f"Error loading model weights from {self.aes_model_path}: {e}")
        w, b = self.mlp.folded()
        self.head_w, self.head_b = w.to(self.device), b
        clip_model_name = path.get("clip-large")
        self.model2 = HFCLIPModel.from_pretrained(clip_model_name)
        if self.model2.projection_dim != 768:
            raise ValueError(f"ImageQualityMetric: unsupported CLIPModel config projection_dim={self.model2.projection_dim} "
                             f"(the aesthetic head takes 768 features)")
        self.processor = AutoProcessor.from_pretrained(clip_model_name)
        self.mean, self.std = hf_mean_std(self.processor)

    def features(self, images):
        eng = self.model2.engine(self.device, self.mean, self.std)
        px = torch.stack([hf_pixels(self.processor, _open(im)) for im in _as_list(images)])
        with torch.no_grad():
            return eng.vision.encode_images(px)

    @torch.no_grad()
    def score(self, images: Union[str, List[str], Image.Image, List[Image.Image]], prompt: str = "") -> List[float]:
        try:
            img = self.features(images)
            aes = torch.empty(img.shape[0], device=self.device, dtype=torch.float32)
            nv.quality_score(img, w=self.head_w, bias=self.head_b, aes=aes)
            return aes.tolist()
        except Exception as e:
            raise RuntimeError(f"Error in scoring images: {e}")
