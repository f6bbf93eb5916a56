"""CPU: the training arena that every resolution bucket's workspace is carved from.  Each shape's views are its
``workspace_plan`` (names, shapes, dtypes), aligned as separate allocations (512 bytes), disjoint and inside the arena; the arena holds the largest
plan seen so far, grows (dropping every view and the old arena, bumping the generation) only when a plan does not fit,
and is released by a re-pack."""
import math

import pytest
import torch

from _util import SMALL

# (B, S, L): latent grids of different sizes, a single-frame bucket, B = 2 and another text length
SHAPES = [(1, 4 * 6 * 8, 24), (1, 3 * 6 * 7, 24), (1, 1 * 6 * 8, 24), (2, 2 * 4 * 9, 24), (1, 4 * 6 * 8, 16)]


def _model(ckpt=None, nl=3):
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig, apply_activation_checkpointing
    m = B200LTXTransformer(LTXConfig(**dict(SMALL, num_layers=nl)), torch.bfloat16, "cpu")
    m.add_adapter(64, 64)
    if ckpt is not None:
        apply_activation_checkpointing(m, *ckpt)
    m.prepare()
    return m


def _span(t):
    """[first byte, end byte) of a contiguous view, relative to its storage."""
    b = t.storage_offset() * t.element_size()
    return b, b + t.numel() * t.element_size()


def _check_views(m, key):
    ws = m._workspace(*key)
    plan = m.workspace_plan(*key)
    assert list(ws) == list(plan)
    assert {k: (tuple(v.shape), v.dtype) for k, v in ws.items()} == plan
    arena = m._arena
    base = arena.data_ptr()
    spans = []
    for name, v in ws.items():
        assert v.is_contiguous(), name
        assert v.untyped_storage().data_ptr() == arena.untyped_storage().data_ptr(), name
        assert (v.data_ptr() - base) % m.ARENA_ALIGN == 0 and m.ARENA_ALIGN % 16 == 0, name
        lo, hi = _span(v)
        assert 0 <= lo <= hi <= arena.numel(), (name, lo, hi, arena.numel())
        spans.append((lo, hi, name))
    spans.sort()
    for (_, hi, a), (lo, _, b) in zip(spans, spans[1:]):
        assert hi <= lo, (a, b)
    return ws


@pytest.mark.parametrize("ckpt", [None, ("full",), ("block_skip", 2)], ids=["keep_all", "full", "block_skip2"])
def test_every_shape_is_its_plan_carved_from_one_arena(ckpt):
    m = _model(ckpt)
    largest = 0
    for key in SHAPES:
        _check_views(m, key)
        plan_bytes = m.workspace_bytes(*key)
        largest = max(largest, plan_bytes)
        # the arena is the largest plan so far, plus less than ARENA_ALIGN bytes of alignment padding per tensor
        assert largest <= m._arena.numel() < largest + m.ARENA_ALIGN * len(m.workspace_plan(*key))
        assert m._arena.numel() == max(m.arena_layout(m.workspace_plan(*k))[1] for k in SHAPES[:SHAPES.index(key) + 1])


@pytest.mark.parametrize("key", SHAPES)
def test_arena_of_one_shape_is_its_workspace(key):
    """A single-shape run allocates what one allocation per tensor took: each plan tensor rounded up to 512 bytes."""
    m = _model()
    m._workspace(*key)
    per_tensor = sum(-(-math.prod(s) * dt.itemsize // 512) * 512 for s, dt in m.workspace_plan(*key).values())
    assert m._arena.numel() == per_tensor
    assert m.workspace_generation == 1


def test_growth_releases_the_old_arena_and_bumps_the_generation():
    import weakref
    m = _model()
    small, large = SHAPES[2], SHAPES[0]
    assert m.workspace_bytes(*small) < m.workspace_bytes(*large)
    assert m.workspace_generation == 0 and m._arena is None
    ws_small = m._workspace(*small)
    old = weakref.ref(m._arena.untyped_storage())
    assert m.workspace_generation == 1
    del ws_small
    m._workspace(*large)
    assert m.workspace_generation == 2
    assert old() is None, "the old arena outlived the growth"
    assert list(m._ws) == [large]           # every view of the old arena was dropped
    ws_small = m._workspace(*small)         # a smaller shape after a larger one: carved from the same arena
    assert m.workspace_generation == 2 and m._arena.numel() == m.arena_layout(m.workspace_plan(*large))[1]
    assert set(m._ws) == {small, large}
    assert ws_small["h"].untyped_storage().data_ptr() == m._ws[large]["h"].untyped_storage().data_ptr()
    assert m._workspace(*small) is ws_small  # cached per shape


def test_repack_releases_the_arena():
    m = _model()
    m._workspace(*SHAPES[0])
    gen = m.workspace_generation
    m.prepare()
    assert m._arena is None and not m._ws
    m._workspace(*SHAPES[2])
    assert m.workspace_generation == gen + 1
    assert m._arena.numel() == m.arena_layout(m.workspace_plan(*SHAPES[2]))[1]
    m.to(torch.float32)                      # a dtype change re-packs: the arena goes with the views
    assert m._arena is None and not m._ws


def test_policy_guard_still_sees_the_workspace():
    m = _model()
    m._workspace(*SHAPES[1])
    with pytest.raises(ValueError, match="before the first forward"):
        m.enable_gradient_checkpointing()
