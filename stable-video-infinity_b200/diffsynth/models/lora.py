"""Static LoRA merge  W += alpha * (B @ A)  at load time (reference diffsynth/models/lora.py:200-267).

Key matching is host logic; the merge itself runs on the native wgmma GEMM (B as the row operand, A^T as the
weight operand, alpha as the per-column gate and W as the fp32 residual), i.e. LoRA is folded through the same
GEMM epilogue the north star names.  Result: W' = round_to_param_dtype(W + alpha * B A) with fp32 accumulation.
"""
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


def get_lora_loaders():
    return [GeneralLoRAFromPeft()]
