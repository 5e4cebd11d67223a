"""H100-native (sm_90a) drop-in for the reference's ``diffsynth`` package — hot path only.

Exports the names ``test_svi.py`` imports (reference ``test_svi.py:2``):
``ModelManager``, ``save_video``, ``SVIVideoPipeline`` (+ ``WanVideoPipeline``).
Attributes are resolved lazily so that ``diffsynth._native`` can be imported on its own.
"""
_LAZY = {
    "ModelManager": ("diffsynth.models.model_manager", "ModelManager"),
    "SVIVideoPipeline": ("diffsynth.pipelines.svi_video", "SVIVideoPipeline"),
    "WanVideoPipeline": ("diffsynth.pipelines.wan_video", "WanVideoPipeline"),
    "SVIDanceVideoPipeline": ("diffsynth.pipelines.svi_video_dance", "SVIDanceVideoPipeline"),
    "SVITalkVideoPipeline": ("diffsynth.pipelines.svi_video_talk", "SVITalkVideoPipeline"),
    "save_video": ("diffsynth.data.video", "save_video"),
    "VideoData": ("diffsynth.data.video", "VideoData"),
    "StreamingVideoWriter": ("diffsynth.data.video", "StreamingVideoWriter"),
    "FlowMatchScheduler": ("diffsynth.schedulers.flow_match", "FlowMatchScheduler"),
    "WanPrompter": ("diffsynth.prompters.wan_prompter", "WanPrompter"),
}


def __getattr__(name):
    if name in _LAZY:
        import importlib
        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(mod), attr)
    raise AttributeError(f"module 'diffsynth' has no attribute {name!r}")


__all__ = list(_LAZY)
