"""The persistent decode kernel's weight ring, replayed on the host (wm_ring_schedule_check): for every CTA, the chunks the
producer warp copies must be the slots the compute warps take, in the same order, or one side waits on an mbarrier
forever.  The self-attention prefix chunks are sized only at launch from the loop state (sa_prefix_chunk in decode.cu),
so the replay covers every kv_len in [0, WM_MAX_POS - 16] with sweep A skipped, with sweep A over 1...16 rows, and
prefill chunks, for chains, Medusa-Block heads and 16-node trees on full and partial grids."""
import ctypes as C

import pytest

WIDTHS = (128, 384, 512, 768, 1024, 1280)
GRIDS = (132, 131, 66, 37, 33)


def _check(lib, d, grid, block=0, K=10, n_tree=11, n_layers=2):
    bad = C.c_int32(-1)
    first = (C.c_int32 * 4)()
    assert lib.wm_ring_schedule_check(d, n_layers, block, K, n_tree, grid, C.byref(bad), first) == 0
    assert bad.value == 0, (d, grid, block, n_tree, "first mismatch {kv_len, L, need_a, cta}:", list(first))


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("d", WIDTHS)
def test_chain_schedule_every_width_and_grid(engine_lib, d, grid):
    """Chain with K = 10 (11 verify rows)."""
    _check(engine_lib, d, grid)


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("d", (512, 1280))
def test_block_heads_and_16_node_trees(engine_lib, d, grid):
    """Medusa-Block heads (the block layer's self-attention runs in the tail), chains and a 16-node tree with K = 3."""
    _check(engine_lib, d, grid, block=1)
    _check(engine_lib, d, grid, block=1, K=3, n_tree=16)
    _check(engine_lib, d, grid, K=3, n_tree=16)


#: (d_model, decoder layers, Block layer): every Whisper size at its real depth, and the deepest model wm_create takes
#: (39 layers + the Block layer = all 40 decoder-layer records)
DEPTHS = ((384, 4, 0), (512, 6, 0), (768, 12, 0), (1024, 24, 0), (1280, 32, 0), (128, 39, 0), (128, 39, 1))


@pytest.mark.parametrize("d,n_layers,block", DEPTHS, ids=[f"d{d}-L{n}" + ("-block" if b else "") for d, n, b in DEPTHS])
def test_schedule_at_full_depth(engine_lib, d, n_layers, block):
    """The stage records and weight chunks of every layer, not just layers 0 and 1: a chain with K = 10 on the full grid
    and a 16-node tree with K = 3 on 37 CTAs."""
    _check(engine_lib, d, 132, block=block, n_layers=n_layers)
    _check(engine_lib, d, 37, block=block, K=3, n_tree=16, n_layers=n_layers)


def test_rejects_out_of_range_shapes(engine_lib):
    bad = C.c_int32(-1)
    first = (C.c_int32 * 4)()
    for args in [(100, 2, 0, 10, 11, 132), (512, 0, 0, 10, 11, 132), (512, 2, 0, 10, 17, 132), (512, 2, 0, 10, 11, 0),
                 (128, 40, 0, 10, 11, 132), (128, 40, 1, 10, 11, 132)]:
        assert engine_lib.wm_ring_schedule_check(*args, C.byref(bad), first) != 0, args
