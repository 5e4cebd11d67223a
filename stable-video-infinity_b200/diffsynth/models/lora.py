"""LoRA on the Wan DiT, two ways.

Merged (reference diffsynth/models/lora.py:200-267, ``ModelManager.load_lora_v2``): W += alpha * (B @ A) at load time.
Key matching is host logic; the merge runs on the native wgmma GEMM (B as the row operand, A^T as the weight operand,
alpha as the per-column gate and W as the fp32 residual).  Result: W' = round_to_param_dtype(W + alpha * B A) with fp32
accumulation — on an e4m3 model the adapter is rounded to 3 mantissa bits with the weight, and undoing it needs a reload.

Unmerged (``WanModel.add_lora_adapter`` / ``set_lora_adapters``): the weights stay as loaded and the adapter runs as a
second K segment of the same GEMM (svi_gemm_lora_bf16, include/svi_b200_lora.h), ahead of its epilogue; ``adapter_weights``
below parses such an adapter.
"""
import re

import torch


class GeneralLoRAFromPeft:
    def get_name_dict(self, lora_state_dict):
        """peft key 'x.lora_B[.default].weight' -> target parameter name 'x.weight' (reference :205-219)."""
        out = {}
        for key in lora_state_dict:
            if ".lora_B." not in key:
                continue
            parts = key.split(".")
            i = parts.index("lora_B")
            if len(parts) > i + 2:
                parts.pop(i + 1)          # adapter name, e.g. 'default'
            parts.pop(i)
            if parts[0] == "diffusion_model":
                parts.pop(0)
            out[".".join(parts)] = (key, key.replace(".lora_B.", ".lora_A."))
        return out

    def match(self, model: torch.nn.Module, state_dict_lora):
        names = self.get_name_dict(state_dict_lora)
        params = {n for n, _ in model.named_parameters()}
        if len(names) > 0 and all(n in params for n in names):
            return "", ""
        return None

    def load(self, model, state_dict_lora, lora_prefix="", alpha=1.0, model_resource=""):
        from .. import _native as nv
        if not torch.cuda.is_available():
            raise RuntimeError("svi_b200: LoRA merge runs on the native GEMM and needs a CUDA device (no CPU fallback)")
        names = self.get_name_dict(state_dict_lora)
        params = dict(model.named_parameters())
        dev = torch.device("cuda", torch.cuda.current_device())
        with torch.no_grad():
            for name, (kb, ka) in names.items():
                p = params[name]
                up = state_dict_lora[kb].to(dev, torch.float32)      # B [out, r]
                down = state_dict_lora[ka].to(dev, torch.float32)    # A [r, in]
                if up.dim() == 4:
                    up, down = up.squeeze(3).squeeze(2), down.squeeze(3).squeeze(2)
                r = up.shape[1]
                rp = (r + 7) // 8 * 8
                b = torch.zeros(up.shape[0], rp, device=dev, dtype=torch.bfloat16)
                at = torch.zeros(down.shape[1], rp, device=dev, dtype=torch.bfloat16)
                b[:, :r] = up
                at[:, :r] = down.t()
                w32 = p.detach().to(dev, torch.float32).reshape(up.shape[0], -1).contiguous()
                gate = torch.full((w32.shape[1],), float(alpha), device=dev, dtype=torch.float32)
                nv.gemm(b, at, w32, gate=gate, residual=w32)
                p.copy_(w32.reshape(p.shape).to(device=p.device, dtype=p.dtype))
        if hasattr(model, "invalidate_engine"):
            model.invalidate_engine()
        print(f"    {len(names)} tensors are updated.")


# the projections an unmerged adapter may target: q, k, v, o of both attentions and the two FFN layers of every block
# (SVI's lora_target_modules="q,k,v,o,ffn.0,ffn.2")
_ADAPTER_TARGET = re.compile(r"blocks\.(\d+)\.(self_attn\.[qkvo]|cross_attn\.[qkvo]|ffn\.[02])\.weight")


def adapter_weights(model, state_dict):
    """{(block index, module): (A bf16 [r, in], B bf16 [out, r])} of a peft LoRA state dict ('x.lora_A[.name].weight',
    'x.lora_B[.name].weight', optional 'diffusion_model.' prefix) for an unmerged adapter on `model`, on the CPU.
    Raises ValueError for a key that is not a LoRA factor, a target other than the block projections above, or a shape
    that does not fit the target weight: such files can still be merged with ModelManager.load_lora_v2."""
    hint = "merge such a LoRA with ModelManager.load_lora_v2 instead"
    for key in state_dict:
        if ".lora_A." not in key and ".lora_B." not in key:
            raise ValueError(f"LoRA adapter: key {key!r} is not a LoRA factor (lora_A / lora_B); {hint}")
    names = GeneralLoRAFromPeft().get_name_dict(state_dict)
    if not names:
        raise ValueError("LoRA adapter: the state dict has no lora_B keys")
    params = dict(model.named_parameters())
    out = {}
    for name, (kb, ka) in names.items():
        m = _ADAPTER_TARGET.fullmatch(name)
        if m is None or name not in params:
            raise ValueError(f"LoRA adapter: key {kb!r} targets {name!r}; an unmerged adapter applies to q, k, v, o and "
                             f"ffn.0 / ffn.2 of the DiT blocks only; {hint}")
        if ka not in state_dict:
            raise ValueError(f"LoRA adapter: key {kb!r} has no matching {ka!r}")
        up, down = state_dict[kb], state_dict[ka]
        if up.dim() == 4:
            up, down = up.squeeze(3).squeeze(2), down.squeeze(3).squeeze(2)
        w = params[name]
        if up.dim() != 2 or down.dim() != 2 or up.shape[1] != down.shape[0] or up.shape[0] != w.shape[0] \
                or down.shape[1] != w.shape[1]:
            raise ValueError(f"LoRA adapter: key {kb!r}: B {tuple(up.shape)} x A {tuple(down.shape)} does not fit the weight "
                             f"{name!r} {tuple(w.shape)}; {hint}")
        out[(int(m.group(1)), m.group(2))] = (down.detach().to("cpu", torch.bfloat16).contiguous(),
                                              up.detach().to("cpu", torch.bfloat16).contiguous())
    return out


def get_lora_loaders():
    return [GeneralLoRAFromPeft()]
