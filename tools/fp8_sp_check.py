"""Multi-GPU check of e4m3 weights under the sequence-parallel plan (run under torchrun, 1 process per GPU): a tiny DiT cast
to float8_e4m3fn, whose rank-local q and k|v GEMMs read row slices (w_q, w_kv) of the fused e4m3 q|k|v matrix, against its
bf16(e4m3(p)) twin under the same plan, on every rank.  Bit-identical where the twin is reproducible from run to run.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29613 tools/fp8_sp_check.py
"""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-video-infinity_b200")):
    sys.path.insert(0, p)
from tools import synth  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from diffsynth.distributed.sequence_parallel import SequenceParallelGroup
    from diffsynth.models.wan_video_dit import WanModel
    ok = True
    for cfg, (f, h, w) in ((synth.CFG_TINY_T2V, (4, 32, 32)), (synth.CFG_TINY_I2V, (3, 20, 36))):
        sd = synth.make_dit_state_dict(cfg, seed=0)
        m8 = WanModel(**cfg).eval()
        m8.load_state_dict(sd)
        m8.to(device=dev, dtype=torch.float8_e4m3fn)
        twin = WanModel(**cfg).eval()
        twin.load_state_dict({k: v.to(torch.float8_e4m3fn).to(torch.bfloat16) for k, v in sd.items()})
        twin.to(device=dev, dtype=torch.bfloat16)
        inp = synth.make_dit_inputs(cfg, f, h, w, seed=0, ctx_len=40)
        x = inp["x"].to(dev)
        kw = {k: inp[k].to(dev) for k in ("clip_feature", "y") if k in inp}
        for cfg_parallel in (False, True):
            sp = SequenceParallelGroup(world, rank, cfg_parallel=cfg_parallel)
            if sp.sp_size == 1:
                continue
            outs = [m.engine(dev).forward(x, 500.0, inp["context"].to(dev), sp=sp, **kw).clone() for m in (m8, twin, twin)]
            spread = (outs[1] - outs[2]).abs().max().item()
            err = (outs[0] - outs[1]).abs().max().item()
            good = torch.equal(outs[0], outs[1]) if spread == 0 else err <= 2 * spread
            ok &= good
            print(f"[rank {rank}] {sp.describe()} L={f * (h // 2) * (w // 2)} has_image={cfg['has_image_input']} "
                  f"max|e4m3 - bf16 twin| = {err:.3e} (twin run-to-run {spread:.3e}) {'OK' if good else 'BAD'}", flush=True)
            if sp._peer is not None:
                sp._peer.close()
                sp._peer = None
        del m8, twin
        torch.cuda.empty_cache()
    t = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    if rank == 0:
        print("FP8_SP_CHECK", "PASS" if t.item() == 1.0 else "FAIL", flush=True)
    sys.exit(0 if t.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
