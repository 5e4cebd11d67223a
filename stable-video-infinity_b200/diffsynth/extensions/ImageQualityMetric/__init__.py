"""Image-text quality scoring (reference ``diffsynth/extensions/ImageQualityMetric``) on the kernel library: CLIP score,
HPSv2 / v2.1, PickScore, the LAION aesthetic score, ImageReward and MPS, with the reference's names, arguments and
return values.

``load_preference_model(model_name, device, path)`` builds one by the reference's name.  ``download_preference_model``
is not provided (it needs modelscope and a network).  See INTEGRATION.md.
"""
from typing import Literal

from .config import MODEL_PATHS, get_model_path
from .reward import ImageRewardScore, MPScore
from .scorers import AestheticScore, CLIPScore, HPScore_v2, PickScore
from .tokenizer import SimpleTokenizer

preference_model_id = Literal["ImageReward", "Aesthetic", "PickScore", "CLIP", "HPSv2", "HPSv2.1", "MPS"]

model_dict = {
    "ImageReward": {"model_class": ImageRewardScore},
    "Aesthetic": {"model_class": AestheticScore},
    "PickScore": {"model_class": PickScore},
    "CLIP": {"model_class": CLIPScore},
    "HPSv2": {"model_class": HPScore_v2, "extra_kwargs": {"model_version": "v2"}},
    "HPSv2.1": {"model_class": HPScore_v2, "extra_kwargs": {"model_version": "v21"}},
    "MPS": {"model_class": MPScore},
}


def load_preference_model(model_name: preference_model_id, device="cuda", path=None):
    if model_name not in model_dict:
        raise ValueError(f"ImageQualityMetric: unknown model {model_name!r}; one of {sorted(model_dict)}")
    entry = model_dict[model_name]
    return entry["model_class"](device=device, path=MODEL_PATHS if path is None else path, **entry.get("extra_kwargs", {}))


__all__ = ["AestheticScore", "CLIPScore", "HPScore_v2", "ImageRewardScore", "MPScore", "PickScore", "SimpleTokenizer",
           "MODEL_PATHS", "get_model_path", "load_preference_model", "model_dict"]
