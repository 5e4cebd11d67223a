"""Native multi-GPU plan for the DiT hot loop: CFG-parallel x token-axis sequence parallelism over NCCL.

Replaces the reference's xfuser "USP" wiring (``diffsynth/distributed/xdit_context_parallel.py``:
``usp_dit_forward`` :42-105 chunks tokens on dim 1 and all-gathers the head output; ``usp_attn_forward``
:108-129 runs Ulysses/ring attention).  xfuser/yunchang are unvendored and unpinned, so their numerics are
"parity unpinned" (SURVEY.md §8c): this implementation is checked against the native single-GPU result.

Plan for N ranks (one process per GPU):
  * the two classifier-free-guidance branches are independent -> ranks [0, N/2) run the conditional forward,
    ranks [N/2, N) the unconditional one (zero communication inside a forward); one all-gather of the two
    velocity fields (8 MB) per step joins them;
  * inside a branch the token axis is split over sp_size = N/2 ranks: every row-local op (LayerNorm, GEMMs,
    RMSNorm, RoPE with a row offset, cross-attention, FFN) runs on L/sp rows; self-attention needs all K/V:
    on GPUs every rank pushes its rows of the [L, 2d] K|V buffer into its peers' buffers over NVLink peer memory
    (copy engines, side stream) and the attention kernel consumes remote rows as their arrival flags flip
    (`PeerExchange`, csrc/sp_exchange.cu, svi_attn_fwd_sp) — no collective call, transfer overlapped with the
    attention on the local rows.  SVI_SP_EXCHANGE=nccl (and the CPU/gloo tests) use one in-place all-gather
    per layer instead;
  * the head output rows are all-gathered once per forward (reference: get_sp_group().all_gather).
Requires L % sp_size == 0 like the reference (torch.chunk + equal-size gather).
"""
import torch
import torch.distributed as dist

_GROUP = None


def partition(world, rank, cfg_parallel=True):
    """Pure host logic: (cfg_groups, sp_size, cfg_idx, sp_rank) for a rank."""
    cfg_groups = 2 if (cfg_parallel and world % 2 == 0) else 1
    sp_size = world // cfg_groups
    return cfg_groups, sp_size, rank // sp_size, rank % sp_size


def all_gather_inplace(full, local, group=None):
    """full[r*n:(r+1)*n] = local of rank r; `local` may alias its own slice of `full`."""
    try:
        dist.all_gather_into_tensor(full, local, group=group)
    except (RuntimeError, NotImplementedError):   # gloo (CPU tests): list form
        n = dist.get_world_size(group)
        dist.all_gather([c.view_as(local) for c in full.chunk(n, dim=0)], local.clone(), group=group)
    return full


def push_order(sp_rank, sp_size):
    """Peers in the order a rank pushes its rows: nearest lower rank first.  Every consumer walks the chunks upwards
    from its own (c, c+1, ...), so the chunk it needs next is always at the head of its owner's queue."""
    return [(sp_rank - i) % sp_size for i in range(1, sp_size)]


def epoch_of(launch, modulus=1 << 16):
    """Flag value of the launch-th exchange (launch = 1, 2, ...): cycles through 1..modulus-1, never the 0 the flag
    words are initialised with."""
    return 1 + (launch - 1) % (modulus - 1)


class PeerExchange:
    """Symmetric K|V buffers of one sequence-parallel group, mapped into every member process (CUDA IPC).

    Two buffers alternate by launch parity.  That is enough: a rank pushes launch c+2 only after its own attention
    c+1 has run, which needed every peer's push c+1, which each peer issued after finishing its attention c — so
    nobody still reads the buffer of parity c when it is overwritten (DESIGN.md §6).  Flag words hold the launch
    number (epoch) of the rows currently in the buffer.
    """

    EPOCHS = 1 << 16

    def __init__(self, sp, L_total, width, device):
        from .. import _native as nv
        self.nv, self.sp, self.device = nv, sp, device
        self.L, self.width = L_total, width
        self.rows = L_total // sp.sp_size
        self.kv_bytes = L_total * width * 2
        flag_off = (self.kv_bytes + 255) // 256 * 256
        self.slab_bytes = self.rows * width * 2
        nbytes = flag_off + 256
        self.ptrs, self.kv, self.flags, handles = [], [], [], []
        for _ in range(2):
            ptr, handle, view = nv.sp_alloc(nbytes, device)
            self.ptrs.append(ptr)
            handles.append(handle)
            self.kv.append(view[:self.kv_bytes].view(torch.bfloat16).view(L_total, width))
            self.flags.append(view[flag_off:flag_off + 4 * sp.sp_size].view(torch.int32))
        gathered = [None] * sp.sp_size
        dist.all_gather_object(gathered, handles, group=sp.sp_group)
        self.peers = push_order(sp.sp_rank, sp.sp_size)
        self.peer_base = {r: [nv.sp_open(h) for h in gathered[r]] for r in self.peers}
        off = sp.sp_rank * self.slab_bytes
        self.peer_dst = [[self.peer_base[r][b] + off for r in self.peers] for b in range(2)]
        self.peer_flag = [[self.peer_base[r][b] + flag_off + 4 * sp.sp_rank for r in self.peers] for b in range(2)]
        self.src = [self.ptrs[b] + off for b in range(2)]
        self.epoch_table = torch.arange(self.EPOCHS, dtype=torch.int32, device=device)
        self.stream = torch.cuda.Stream(device=device)
        self.pushed = [None, None]       # event: my last push out of buffer b has left (the slab may be rewritten)
        self.launch = 0
        dist.barrier(group=sp.sp_group)  # everybody has mapped everybody before the first push

    def begin(self):
        """Next launch: returns (buffer index, local K|V slab to fill).  Waits for the previous push out of the slab."""
        self.launch += 1
        b = self.launch & 1
        if self.pushed[b] is not None:
            torch.cuda.current_stream().wait_event(self.pushed[b])
        r = self.sp.sp_rank
        return b, self.kv[b][r * self.rows:(r + 1) * self.rows]

    @property
    def epoch(self):
        return epoch_of(self.launch, self.EPOCHS)

    def push(self, b):
        """The local slab of buffer b is complete on the current stream: send it to every peer."""
        ready = torch.cuda.Event()
        ready.record()
        self.stream.wait_event(ready)
        self.nv.sp_push(self.src[b], self.peer_dst[b], self.peer_flag[b], self.slab_bytes,
                        self.epoch_table.data_ptr() + 4 * self.epoch, self.stream)
        ev = torch.cuda.Event()
        ev.record(self.stream)
        self.pushed[b] = ev

    def close(self):
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.sp.sp_group)
        for r in self.peers:
            for p in self.peer_base[r]:
                self.nv.sp_close(p)
        self.kv, self.flags = [], []
        for p in self.ptrs:
            self.nv.sp_free(p)
        self.ptrs = []


class SequenceParallelGroup:
    def __init__(self, world, rank, cfg_parallel=True):
        self.world, self.rank = world, rank
        self.cfg_groups, self.sp_size, self.cfg_idx, self.sp_rank = partition(world, rank, cfg_parallel)
        self.sp_group = None
        self.cfg_group = None
        # every rank creates every group, in the same order
        for c in range(self.cfg_groups):
            ranks = list(range(c * self.sp_size, (c + 1) * self.sp_size))
            g = dist.new_group(ranks) if self.sp_size > 1 else None
            if c == self.cfg_idx:
                self.sp_group = g
        for s in range(self.sp_size):
            ranks = [c * self.sp_size + s for c in range(self.cfg_groups)]
            g = dist.new_group(ranks) if self.cfg_groups > 1 else None
            if s == self.sp_rank:
                self.cfg_group = g
        self._rows = None
        self._bufs = {}
        self._peer = None

    def describe(self):
        return f"cfg{self.cfg_groups}xsp{self.sp_size}"

    # ---- token partition
    def local_rows(self, L):
        if L % self.sp_size != 0:
            raise RuntimeError(f"sequence parallelism needs L % sp_size == 0 (L={L}, sp_size={self.sp_size}); "
                               f"the reference has the same constraint (torch.chunk + equal all_gather)")
        return L // self.sp_size

    def set_tokens(self, L):
        self._rows = self.local_rows(L)

    @property
    def row_offset(self):
        return self.sp_rank * self._rows

    def local_slice(self, full):
        n = full.shape[0] // self.sp_size
        return full[self.sp_rank * n:(self.sp_rank + 1) * n]

    # ---- K|V exchange over peer memory (GPU only)
    def peer_exchange(self, L_total, width, device):
        """The group's PeerExchange for [L_total, width] K|V buffers, or None when the NCCL/gloo all-gather is to be used
        (CPU tensors, SVI_SP_EXCHANGE=nccl, or slabs narrower than one attention tile)."""
        import os
        if self.sp_size == 1 or device.type != "cuda" or os.environ.get("SVI_SP_EXCHANGE", "peer") == "nccl":
            return None
        if L_total // self.sp_size < 128:
            return None
        pe = self._peer
        if pe is None or pe.L != L_total or pe.width != width:
            if pe is not None:
                pe.close()
            pe = self._peer = PeerExchange(self, L_total, width, device)
        return pe

    # ---- collectives
    def all_gather_rows(self, full):
        """in-place all-gather of a row-sharded [L, *] buffer inside the sequence-parallel group"""
        if self.sp_size > 1:
            all_gather_inplace(full, self.local_slice(full), self.sp_group)
        return full

    def cfg_parallel_step(self, eng, lat, t, cp, cn, v_c, v_u, cfg_scale, sigma, nxt, y=None, tea=(None, None),
                          add_condition=(None, None)):
        """One denoise step under the plan above; lat is replicated on every rank and updated identically.
        cp / cn: the conditional / unconditional ContextState (a CFG-parallel rank needs only its own branch's; the other
        may be None); tea / add_condition: (conditional, unconditional) TeaCache objects and token-space conditions."""
        inner = self if self.sp_size > 1 else None
        if self.cfg_groups == 2:
            key = ("vpair", tuple(lat.shape))
            vp = self._bufs.get(key)
            if vp is None:
                vp = torch.empty((2,) + tuple(lat.shape), device=lat.device, dtype=torch.float32)
                self._bufs[key] = vp
            b = self.cfg_idx
            eng.forward(lat, t, cp if b == 0 else cn, y=y, sp=inner, out=vp[b], tea_cache=tea[b], add_condition=add_condition[b])
            all_gather_inplace(vp, vp[b], self.cfg_group)
            eng.k.cfg_euler_step(lat, vp[0], vp[1], cfg_scale, sigma, nxt)
        else:
            eng.forward(lat, t, cp, y=y, sp=inner, out=v_c, tea_cache=tea[0], add_condition=add_condition[0])
            eng.forward(lat, t, cn, y=y, sp=inner, out=v_u, tea_cache=tea[1], add_condition=add_condition[1])
            eng.k.cfg_euler_step(lat, v_c, v_u, cfg_scale, sigma, nxt)
        return lat

    def owns_branch(self, b):
        """True when this rank computes CFG branch b (0 = conditional, 1 = unconditional) under the plan."""
        return self.cfg_groups == 1 or self.cfg_idx == b


def init_sp_groups(world=None, rank=None, cfg_parallel=True):
    global _GROUP
    world = dist.get_world_size() if world is None else world
    rank = dist.get_rank() if rank is None else rank
    _GROUP = SequenceParallelGroup(world, rank, cfg_parallel)
    return _GROUP


def get_sp_group():
    """The process-wide plan behind `use_usp=True` (reference: xfuser's get_sp_group(), svi_video.py:266-273).  Default =
    CFG-parallel x sequence-parallel for an even world size (N=2: cfg2 x sp1, N=8: cfg2 x sp4);
    SVI_SP_PLAN=sp splits only the token axis (sp = N), like the reference."""
    if _GROUP is None:
        if not dist.is_initialized():
            raise RuntimeError("sequence parallelism requested but torch.distributed is not initialised")
        import os
        return init_sp_groups(cfg_parallel=os.environ.get("SVI_SP_PLAN", "cfg") != "sp")
    return _GROUP
