"""The ring producer's L2 prefetch cursor, replayed on the host (wm_ring_prefetch_check) at budgets other than the built
one (wm_ring_schedule_check replays the built budget over every width, grid and depth): every chunk the cursor prefetches
is copied later in the same launch, in prefetch order, or is one of the tail program's leading weight chunks (the next
launch's first copies); the bytes prefetched and not yet copied never exceed the budget; with a budget every copy was
prefetched first; and the copies themselves are still the slots the compute warps take."""
import ctypes as C

import pytest

BUDGETS = (0, 41984, 128 * 1024, 192 * 1024)


def _check(lib, d, grid, budget, block=0, K=10, n_tree=11, n_layers=2):
    bad = C.c_int32(-1)
    first = (C.c_int32 * 4)()
    assert lib.wm_ring_prefetch_check(d, n_layers, block, K, n_tree, grid, budget, C.byref(bad), first) == 0
    assert bad.value == 0, (d, grid, budget, block, n_tree, "first failing launch {kv_len, L, need_a, cta}:", list(first))


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("d,grid", [(1280, 132), (512, 37), (128, 33)])
def test_prefetch_cursor_at_every_budget(engine_lib, d, grid, budget):
    """Chains with K = 10 on the full grid and on partial grids (several self-attention items per CTA)."""
    _check(engine_lib, d, grid, budget)


@pytest.mark.parametrize("budget", (41984, 192 * 1024))
def test_prefetch_cursor_block_heads_and_trees(engine_lib, budget):
    """Medusa-Block heads: the tail program holds the block layer's self-attention, where the next launch's warm-up
    stops; and a 16-node tree with K = 3."""
    _check(engine_lib, 512, 66, budget, block=1)
    _check(engine_lib, 1280, 132, budget, block=1, K=3, n_tree=16)


def test_rejects_budgets_below_one_chunk(engine_lib):
    bad = C.c_int32(-1)
    first = (C.c_int32 * 4)()
    for budget in (-1, 1, 41983):
        assert engine_lib.wm_ring_prefetch_check(1280, 2, 0, 10, 11, 132, budget, C.byref(bad), first) != 0, budget
