"""VRAM management surface (reference diffsynth/vram_management/layers.py).

The reference wraps Linear / conv / norm modules so that weights beyond a parameter budget live on the CPU and
are re-copied host->device on EVERY forward (layers.py:65-71; ~20 GB per forward for the 14B model under the
default 6e9 budget, SURVEY.md §8a16).  On an 80 GB H100 everything is resident, so the policy implemented here
is "all resident": the call is accepted, models are moved to the computation device once, and the module tree
(whose parameter names are the checkpoint / LoRA key contract) is left untouched.
"""
import torch


class AutoWrappedModule(torch.nn.Module):
    """Kept for isinstance / import compatibility; never instantiated by the all-resident policy."""

    def __init__(self, module, **kwargs):
        super().__init__()
        self.module = module


class AutoWrappedLinear(torch.nn.Linear):
    pass


def enable_vram_management(model: torch.nn.Module, module_map: dict, module_config: dict, max_num_param=None,
                           overflow_module_config: dict = None):
    dev = module_config.get("computation_device", "cuda")
    model.to(dev)
    model.vram_management_enabled = False
    return model
