"""CPU: property tests (hypothesis) of the pure host logic that decides WHAT the kernels are asked to do."""
import torch
from hypothesis import given, settings
from hypothesis import strategies as st


@settings(max_examples=200, deadline=None)
@given(units=st.integers(1, 20000), kv_tiles=st.integers(1, 1024), sms=st.sampled_from([132, 148, 160]),
       ws_slices=st.integers(0, 4000))
def test_attention_plan_invariants(units, kv_tiles, sms, ws_slices):
    """svi_attn_plan: whole units + sliced units = all units; slices fit the workspace; slicing never costs more rounds than
    running everything whole; units that fill whole waves are never sliced."""
    from diffsynth import _native as nv
    slice_bytes = 128 * 128 * 4 + 128 * 8   # one 128-row Q tile: partial O + (row max, row sum)
    n_full, split = nv.attention_plan(units, kv_tiles, sms, ws_slices * slice_bytes)
    tail = units - n_full
    assert 0 <= n_full <= units and 1 <= split <= 8
    if split == 1:
        assert n_full == units
    else:
        assert tail > 0 and n_full % sms == 0 and tail * split <= ws_slices and kv_tiles // split >= 8
        whole = -(-units // sms)
        sliced = n_full // sms + -(-tail * split // sms) / split
        assert sliced < whole


@settings(max_examples=100, deadline=None)
@given(world=st.integers(1, 16), cfg_parallel=st.booleans())
def test_partition_covers_every_rank_once(world, cfg_parallel):
    from diffsynth.distributed.sequence_parallel import partition
    seen = set()
    for r in range(world):
        groups, sp, ci, sr = partition(world, r, cfg_parallel)
        assert groups * sp == world and 0 <= ci < groups and 0 <= sr < sp and r == ci * sp + sr
        seen.add((ci, sr))
    assert len(seen) == world


@settings(max_examples=60, deadline=None)
@given(T=st.integers(1, 9), stride=st.sampled_from([1, 2]), seed=st.integers(0, 1000))
def test_slot_table_is_conv3d_temporal_padding(T, stride, seed):
    """models.dwpose_embedding.slot_table == the frames nn.Conv3d(kernel 3, padding 1, stride) reads along time."""
    import torch.nn.functional as F
    from diffsynth.models.dwpose_embedding import slot_table
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 1, T, 1, 1, generator=g)
    w = torch.randn(1, 1, 3, 1, 1, generator=g)
    want = F.conv3d(x, w, stride=(stride, 1, 1), padding=(1, 0, 0)).flatten()
    T_out = (T + 2 - 3) // stride + 1
    table = slot_table(list(range(T)), T, T_out, stride, 3)
    frames = torch.cat([x.flatten(), torch.zeros(1)])          # slot T is the zero frame
    got = torch.stack([sum(w.flatten()[a] * frames[table[t][a]] for a in range(3)) for t in range(T_out)])
    assert want.shape == got.shape and torch.allclose(want, got, atol=1e-5)


@settings(max_examples=60, deadline=None)
@given(P=st.integers(2, 8))
def test_push_order_serves_consumers_in_chunk_order(P):
    from diffsynth.distributed.sequence_parallel import push_order
    for c in range(P):
        arrival = {}                                       # chunk -> position in its owner's push queue towards c
        for owner in range(P):
            if owner != c:
                arrival[owner] = push_order(owner, P).index(c)
        visit = [(c + k) % P for k in range(1, P)]         # order in which consumer c needs the chunks
        assert [arrival[o] for o in visit] == sorted(arrival[o] for o in visit)
