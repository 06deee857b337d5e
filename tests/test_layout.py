"""Flat arena layout invariants (``parallel/layout.py``): tile alignment, reverse (backward) order, tile table."""
import torch
from hypothesis import given, settings, strategies as st

from pytorch_ps_mpi_b200.codings import TILE, DeviceCodeSpec, KIND_DENSE, KIND_TOPK, WIRE_BF16, WIRE_F32, tile_k
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout


def _layout(shapes, groups=None):
    params = [torch.nn.Parameter(torch.zeros(s)) for s in shapes]
    groups = groups or [list(range(len(shapes)))]
    pg = [{"params": [params[i] for i in g]} for g in groups]
    return FlatLayout(pg, {id(p): f"p{i}" for i, p in enumerate(params)}), params


def test_reverse_registration_order_and_alignment():
    L, params = _layout([(3, 5), (TILE * 2 + 1,), (7,), (TILE,)], groups=[[0, 1], [2, 3]])
    assert [s.name for s in L.slots] == ["p3", "p2", "p1", "p0"]          # backward order (ps.py:121-123)
    assert [s.group for s in L.slots] == [1, 1, 0, 0]
    t = 0
    for s in L.slots:
        assert s.first_tile == t and s.offset == t * TILE and s.ntiles == max(1, -(-s.numel // TILE))
        t += s.ntiles
    assert L.ntiles == t and L.numel_padded == t * TILE and L.by_id[id(params[1])].ntiles == 3


@settings(max_examples=25, deadline=None)
@given(st.lists(st.integers(min_value=1, max_value=3 * TILE + 5), min_size=1, max_size=8))
def test_tile_table_matches_slow_construction(sizes):
    L, _ = _layout([(n,) for n in sizes])
    fast, slow = L.tile_table_fast(), L.tile_table()
    assert torch.equal(fast, slow)
    # every element of every parameter is covered exactly once by the valid ranges
    for s in L.slots:
        rows = fast[s.first_tile: s.first_tile + s.ntiles]
        assert int(rows[:, 1].sum()) == s.numel and bool((rows[:, 0] == s.index).all()) and bool((rows[:, 3] == s.first_tile).all())
        assert bool((rows[:-1, 1] == TILE).all())


def test_device_spec_wire_sizes():
    dense = DeviceCodeSpec(KIND_DENSE, -1)
    assert dense.bytes_per_tile(torch.bfloat16) == TILE * 2 and dense.bytes_per_tile(torch.float32) == TILE * 4
    tk = DeviceCodeSpec(KIND_TOPK, WIRE_BF16, 0.01)
    assert tk.tile_capacity() == tile_k(0.01, TILE) == 21 and tk.bytes_per_tile(torch.bfloat16) == 96     # 21*4 → 16-byte multiple
    tk32 = DeviceCodeSpec(KIND_TOPK, WIRE_F32, 0.5)
    assert tk32.bytes_per_tile(torch.float32) == 1024 * 8
    assert tile_k(0.1, 10) == 1 and tile_k(1.0, 7) == 7 and tile_k(0.001, 5) == 1


def test_pipeline_chunk_plan():
    """Chunks of the update pipeline: whole parameters, arena order, contiguous tile ranges, >= chunk_bytes each except the last,
    capped in number, identical for identical layouts; ``single=True`` is the unpipelined plan."""
    import torch
    from pytorch_ps_mpi_b200 import models
    from pytorch_ps_mpi_b200.codings import TILE
    from pytorch_ps_mpi_b200.parallel.layout import FlatLayout
    model = models.resnet18(num_classes=1000)
    groups = [{"params": list(model.parameters())}]
    L = FlatLayout(groups, {id(p): n for n, p in model.named_parameters()})
    chunks = L.plan_chunks(2, 4 << 20)
    assert [s.index for c in chunks for s in c] == list(range(L.nparams))           # a partition, in arena order
    for c in chunks:
        assert all(a.first_tile + a.ntiles == b.first_tile for a, b in zip(c, c[1:]))   # contiguous tiles
    sizes = [sum(s.ntiles for s in c) * TILE * 2 for c in chunks]
    assert all(sz >= (4 << 20) for sz in sizes[:-1]) and 2 <= len(chunks) <= 48
    assert chunks[0][0].name.startswith("fc")                                          # backward order: the head comes first
    assert len(L.plan_chunks(2, 4 << 20, single=True)) == 1
    assert len(L.plan_chunks(2, 1)) <= 48                                               # tiny request: capped
    again = FlatLayout(groups, {id(p): n for n, p in model.named_parameters()}).plan_chunks(2, 4 << 20)
    assert [[s.name for s in c] for c in again] == [[s.name for s in c] for c in chunks]


def test_custom_arena_placement_hint():
    """``param.ps_arena_layout = (strides, span)``: the slot takes the span, an impossible hint is rejected."""
    import pytest
    import torch
    from pytorch_ps_mpi_b200 import models
    from pytorch_ps_mpi_b200.ops.stem import STEM_K, STEM_STRIDES
    from pytorch_ps_mpi_b200.parallel.layout import FlatLayout
    model = models.resnet18(num_classes=10)
    groups = [{"params": list(model.parameters())}]
    L = FlatLayout(groups, {id(p): n for n, p in model.named_parameters()})
    slot = L.by_id[id(model.conv1.weight)]
    assert slot.numel == 64 * STEM_K and slot.strides == STEM_STRIDES and slot.ntiles == -(-64 * STEM_K // 2048)
    p = torch.nn.Parameter(torch.zeros(4, 4))
    p.ps_arena_layout = ((8, 1), 16)                      # reaches element 3*8 + 3 = 27 >= 16
    with pytest.raises(ValueError):
        FlatLayout([{"params": [p]}], {id(p): "p"})


def test_slot_view_keeps_the_physical_layout():
    """``ParamSlot.view``: a flat arena slice seen with the parameter's shape — contiguous, the parameter's own dense strides
    (channels_last), or the module's custom placement over a padded span (the stem's [64,176] GEMM matrix)."""
    from pytorch_ps_mpi_b200.ops.stem import STEM_K, STEM_STRIDES
    contiguous = torch.nn.Parameter(torch.randn(5, 7))
    cl = torch.nn.Parameter(torch.randn(8, 4, 3, 3).contiguous(memory_format=torch.channels_last))
    stem = torch.nn.Parameter(torch.randn(64, 3, 7, 7))
    stem.ps_arena_layout = (STEM_STRIDES, 64 * STEM_K)
    strided = torch.nn.Parameter(torch.randn(6, 10)[:, ::2])         # not dense: the arena holds it contiguously
    params = [contiguous, cl, stem, strided]
    L = FlatLayout([{"params": params}], {id(p): f"p{i}" for i, p in enumerate(params)})
    arena = torch.zeros(L.numel_padded)
    want = {id(contiguous): (5 * 7, (7, 1)), id(cl): (8 * 4 * 3 * 3, cl.stride()), id(stem): (64 * STEM_K, STEM_STRIDES),
            id(strided): (6 * 5, (5, 1))}
    for s in L.slots:
        flat = arena[s.offset: s.offset + s.numel]
        v = s.view(flat)
        assert s.numel == want[id(s.param)][0] and v.shape == s.param.shape and v.stride() == tuple(want[id(s.param)][1])
        assert v.data_ptr() == flat.data_ptr()
        v.copy_(s.param.detach())
        assert torch.equal(v, s.param.detach())
    s = L.by_id[id(stem)]
    stem_span = arena[s.offset: s.offset + s.numel].view(64, STEM_K)
    assert torch.equal(stem_span[:, :168].reshape(64, 7, 8, 3)[:, :, :7].permute(0, 3, 1, 2), stem.detach())   # (kh, kw, c)
    assert not stem_span[:, 168:].any() and not stem_span[:, :168].reshape(64, 7, 8, 3)[:, :, 7:].any()      # padding stays 0
    s = L.by_id[id(cl)]
    assert torch.equal(arena[s.offset: s.offset + s.numel], cl.detach().permute(0, 2, 3, 1).reshape(-1))   # NHWC in the arena
