"""Multi-GPU check of unmerged LoRA adapters (run under torchrun, 1 process per GPU): the sequence-parallel DiT forward of a
model with two active adapters against the single-GPU forward on every rank (the q and k|v launches of the split take
their column groups of one down-projection).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29613 tools/lora_sp_check.py
"""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
from tools import synth  # noqa: E402


def main():
    from test_lora_adapters_cpu import make_lora
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from diffsynth.distributed.sequence_parallel import SequenceParallelGroup
    from diffsynth.models.wan_video_dit import WanModel
    ok = True
    for cfg, (f, h, w) in ((synth.CFG_TINY_T2V, (4, 32, 32)), (synth.CFG_TINY_I2V, (3, 20, 36))):
        m = WanModel(**cfg).eval()
        m.load_state_dict(synth.make_dit_state_dict(cfg, seed=0))
        m.to(dev)
        m.add_lora_adapter("a", make_lora(cfg, 1, rank=128))
        m.add_lora_adapter("b", make_lora(cfg, 2, rank=16, targets=("self_attn.k", "self_attn.v", "ffn.0")))
        m.set_lora_adapters({"a": 0.7, "b": -0.3})
        eng = m.engine(dev)
        inp = synth.make_dit_inputs(cfg, f, h, w, seed=0, ctx_len=40)
        x = inp["x"].to(dev)
        kw = {k: inp[k].to(dev) for k in ("clip_feature", "y") if k in inp}
        ref = eng.forward(x, 500.0, inp["context"].to(dev), **kw).clone()
        sp = SequenceParallelGroup(world, rank, cfg_parallel=False)
        out = eng.forward(x, 500.0, inp["context"].to(dev), sp=sp, **kw)
        err = (out - ref).abs().max().item()
        good = err < 2e-2
        ok &= good
        print(f"[rank {rank}] {sp.describe()} has_image={cfg['has_image_input']} max|sp - single| = {err:.3e} "
              f"{'OK' if good else 'BAD'}", flush=True)
        if sp._peer is not None:
            sp._peer.close()
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("LORA_SP_CHECK PASS" if flag.item() else "LORA_SP_CHECK FAIL", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
