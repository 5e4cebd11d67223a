"""ModelManager — checkpoint detection/loading boundary (reference diffsynth/models/model_manager.py).

Only the Wan rows of the reference's hash table are kept (model_config.py:117-125); the inherited
DiffSynth-Studio model zoo is out of scope (SURVEY.md §2 row 23), except the two post-processing models: RIFE's
flownet.pkl (model_config.py:100), which loads as diffsynth.extensions.RIFE.IFNet, and RealESRGAN_x4.pth
(model_config.py:101), which loads as diffsynth.extensions.ESRGAN.RRDBNet.  Detection is by the md5 of the sorted
'key[:shape]' list exactly as the reference does (models/utils.py:179-182), so real Wan2.1 checkpoints and
SVI LoRA files resolve to the same classes.
"""
import os
from typing import List

import torch

from .lora import get_lora_loaders
from .utils import hash_state_dict_keys, init_weights_on_device, load_state_dict
from .wan_video_dit import WanModel


def _loader_table():
    from ..extensions.ESRGAN import RRDBNet
    from ..extensions.RIFE import IFNet
    from .wan_video_image_encoder import WanImageEncoder
    from .wan_video_text_encoder import WanTextEncoder
    from .wan_video_vae import WanVideoVAE
    return [
        # (keys_hash, keys_hash_with_shape, model_names, model_classes, resource)  — model_config.py:117-125
        (None, "9269f8db9040a9d860eaca435be61814", ["wan_video_dit"], [WanModel], "civitai"),
        (None, "aafcfd9672c3a2456dc46e1cb6e52c70", ["wan_video_dit"], [WanModel], "civitai"),
        (None, "6bfcfb3b342cb286ce886889d519a77e", ["wan_video_dit"], [WanModel], "civitai"),
        (None, "b6caaaa1388107ec24d25592901ca489", ["wan_video_dit"], [WanModel], "civitai"),     # SVI-Talk (multitalk)
        (None, "cb104773c6c2cb6df4f9529ad5c60d0b", ["wan_video_dit"], [WanModel], "diffusers"),
        (None, "9c8818c2cbea55eca56c7b447df170da", ["wan_video_text_encoder"], [WanTextEncoder], "civitai"),
        (None, "5941c53e207d62f20f9025686193c40b", ["wan_video_image_encoder"], [WanImageEncoder], "civitai"),
        (None, "1378ea763357eea97acdef78e65d6d96", ["wan_video_vae"], [WanVideoVAE], "civitai"),
        (None, "ccc42284ea13e1ad04693284c7a09be6", ["wan_video_vae"], [WanVideoVAE], "civitai"),
        (None, "9b9313d104ac4df27991352fec013fd4", ["rife"], [IFNet], "civitai"),                # flownet.pkl, :100
        (None, "6b7116078c4170bfbeaedc8fe71f6649", ["esrgan"], [RRDBNet], "civitai"),            # RealESRGAN_x4.pth, :101
    ]


def load_model_from_single_file(state_dict, model_names, model_classes, model_resource, torch_dtype, device):
    """reference model_manager.py:57-105: converter -> construct on meta -> load_state_dict(assign=True)."""
    names, models = [], []
    for model_name, cls in zip(model_names, model_classes):
        print(f"    model_name: {model_name} model_class: {cls.__name__}")
        conv = cls.state_dict_converter()
        res = conv.from_civitai(state_dict) if model_resource == "civitai" else conv.from_diffusers(state_dict)
        sd, extra = res if isinstance(res, tuple) else (res, {})
        if extra:
            print(f"        This model is initialized with extra kwargs: {extra}")
        with init_weights_on_device():
            model = cls(**extra)
        model = model.eval()
        want = set(dict(model.named_parameters()).keys())
        missing = want - set(sd.keys())
        if missing:  # reference :80-94: xavier for matrices, zeros for vectors
            print(f"        Initializing missing parameters: {missing}")
            for name, p in model.named_parameters():
                if name in missing:
                    t = torch.empty(p.shape, dtype=torch_dtype, device=device)
                    if t.dim() >= 2:
                        torch.nn.init.xavier_uniform_(t)
                    else:
                        t.zero_()
                    sd[name] = t
        model.load_state_dict(sd, assign=True)
        model = model.to(dtype=torch_dtype, device=device)
        names.append(model_name)
        models.append(model)
    return names, models


class ModelDetectorFromSingleFile:
    def __init__(self, configs):
        self.by_shape, self.by_keys = {}, {}
        for keys_hash, keys_hash_with_shape, names, classes, resource in configs:
            self.by_shape[keys_hash_with_shape] = (names, classes, resource)
            if keys_hash is not None:
                self.by_keys[keys_hash] = (names, classes, resource)

    def _lookup(self, state_dict):
        return (self.by_shape.get(hash_state_dict_keys(state_dict, with_shape=True))
                or self.by_keys.get(hash_state_dict_keys(state_dict, with_shape=False)))

    def match(self, file_path="", state_dict=None):
        if isinstance(file_path, str) and os.path.isdir(file_path):
            return False
        if not state_dict:
            state_dict = load_state_dict(file_path)
        return self._lookup(state_dict) is not None

    def load(self, file_path="", state_dict=None, device="cuda", torch_dtype=torch.float16, **kwargs):
        if not state_dict:
            state_dict = load_state_dict(file_path)
        names, classes, resource = self._lookup(state_dict)
        return load_model_from_single_file(state_dict, names, classes, resource, torch_dtype, device)


class ModelManager:
    def __init__(self, torch_dtype=torch.float16, device="cuda", model_id_list: List[str] = [],
                 downloading_priority: List[str] = ["ModelScope", "HuggingFace"], file_path_list: List[str] = [],
                 train_architecture="lora"):
        if model_id_list:
            raise RuntimeError("svi_b200: model downloading is not part of the hot path (no network); pass file paths")
        self.torch_dtype = torch_dtype
        self.device = device
        self.model, self.model_path, self.model_name = [], [], []
        self.model_detector = [ModelDetectorFromSingleFile(_loader_table())]
        self.state_dict_new = {}
        self.state_dict_new_module = {}
        self.load_models(list(file_path_list))

    # ---------------------------------------------------------------- models
    def add_model(self, model_name, model, model_path="<in-memory>"):
        """Register an already constructed model (random-init benchmarks / tests; no reference counterpart)."""
        self.model.append(model)
        self.model_path.append(model_path)
        self.model_name.append(model_name)

    def load_model(self, file_path, model_names=None, device=None, torch_dtype=None):
        print(f"Loading models from: {file_path}")
        device = self.device if device is None else device
        torch_dtype = self.torch_dtype if torch_dtype is None else torch_dtype
        if isinstance(file_path, list):      # sharded checkpoint: merge the shards (reference :660-663)
            state_dict = {}
            for path in file_path:
                state_dict.update(load_state_dict(path))
        elif os.path.isfile(file_path):
            state_dict = load_state_dict(file_path)
        else:
            state_dict = None
        for det in self.model_detector:
            if det.match(file_path, state_dict):
                names, models = det.load(file_path, state_dict, device=device, torch_dtype=torch_dtype,
                                         allowed_model_names=model_names, model_manager=self)
                for n, m in zip(names, models):
                    self.add_model(n, m, file_path)
                print(f"    The following models are loaded: {names}.")
                return
        # the reference drops into ipdb here (model_manager.py:681); raise instead
        raise RuntimeError(f"We cannot detect the model type of {file_path}. No models are loaded.")

    def load_models(self, file_path_list, model_names=None, device=None, torch_dtype=None):
        for file_path in file_path_list:
            self.load_model(file_path, model_names, device=device, torch_dtype=torch_dtype)

    def fetch_model(self, model_name, file_path=None, require_model_path=False):
        hits = [(m, p) for m, p, n in zip(self.model, self.model_path, self.model_name)
                if n == model_name and (file_path is None or file_path == p)]
        if not hits:
            print(f"No {model_name} models available.")
            return None
        if len(hits) == 1:
            print(f"Using {model_name} from {hits[0][1]}.")
        else:
            print(f"More than one {model_name} models are loaded in model manager: {[p for _, p in hits]}. "
                  f"Using {model_name} from {hits[0][1]}.")
        return hits[0] if require_model_path else hits[0][0]

    def to(self, device):
        for m in self.model:
            m.to(device)

    # ---------------------------------------------------------------- LoRA
    def _try_lora(self, state_dict, lora_alpha):
        for name, model, path in zip(self.model_name, self.model, self.model_path):
            for lora in get_lora_loaders():
                res = lora.match(model, state_dict)
                if res is not None:
                    print(f"    Adding LoRA to {name} ({path}).")
                    lora.load(model, state_dict, res[0], alpha=lora_alpha, model_resource=res[1])
                    return True
        return False

    def load_lora(self, file_path="", state_dict=None, lora_alpha=1.0):
        sd = state_dict if state_dict else load_state_dict(file_path)
        if not self._try_lora(sd, lora_alpha):
            print(f"    Cannot load LoRA: {file_path}")

    def load_lora_v2(self, file_path="", state_dict=None, lora_alpha=1.0, is_final=True):
        """reference model_manager.py:490-560: SVI LoRA files carry 'pipe.dit.'-prefixed peft keys (possibly split
        over several files); the prefix is stripped, the pieces are accumulated and merged on the final file."""
        if isinstance(file_path, list):
            if not file_path:
                raise RuntimeError(f"    ERROR: Cannot load LoRA from {file_path}.")
            for i, fp in enumerate(file_path):
                self.load_lora_v2(fp, state_dict=state_dict, lora_alpha=lora_alpha, is_final=(i == len(file_path) - 1))
            return
        print(f"Loading LoRA models from file: {file_path}")
        sd = state_dict if state_dict else load_state_dict(file_path)
        for key in sd:
            if any(t in key for t in ("dwpose_embedding", "randomref_embedding_pose", "inpaint_embedding",
                                      "learn_in_embedding", "randomref")):
                self.state_dict_new_module[key] = sd[key]
        loaded = self._try_lora(sd, lora_alpha)
        if not loaded:
            for key in sd:
                if "lora" in key and "pipe.dit." in key:
                    self.state_dict_new[key.split("pipe.dit.")[1]] = sd[key]
            if not is_final:
                return
            loaded = self._try_lora(self.state_dict_new, lora_alpha)
        if not loaded:
            msg = (f"    ERROR: Cannot load LoRA from {file_path}. No compatible LoRA weights found or failed to "
                   f"match with any model.")
            print(msg)
            raise RuntimeError(msg)
