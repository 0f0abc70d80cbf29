"""CPU: the tile schedules of tc_gemm_kernel restated (csrc/tc_gemm.cu: strided for the plain kernels, contiguous ranges for the
LayerNorm-prologue form; a unit = one CTA or one 2-CTA cluster of the pair form) — every output tile is computed exactly once, and with the
LayerNorm prologue every row block a unit loads was normalised by that same unit (no cross-CTA dependency), at most 2-3 blocks each."""
import pytest


def units_and_tiles(M, N, pair, sms=132):
    tiles_n = -(-N // 128)
    tiles_m = -(-M // 128)
    num = tiles_n * (-(-tiles_m // 2) if pair else tiles_m)
    units = min(num, sms // 2 if pair else sms)
    return tiles_n, num, units


@pytest.mark.parametrize("M,N", [(7936, 2048), (7936, 768), (7936, 512), (7936, 4233), (1000, 768), (129, 2048), (385, 4233), (300, 256)])
@pytest.mark.parametrize("pair", [False, True])
def test_every_tile_once_and_rows_normalised_by_their_own_unit(M, N, pair):
    tiles_n, num, units = units_and_tiles(M, N, pair)
    assert units >= 1
    # strided schedule (plain kernels)
    seen = sorted(t for u in range(units) for t in range(u, num, units))
    assert seen == list(range(num))
    # contiguous ranges (LayerNorm prologue): [num*u/units, num*(u+1)/units)
    seen, max_blocks = [], 0
    for u in range(units):
        b, e = num * u // units, num * (u + 1) // units
        assert b < e                                              # units <= num: no empty range
        tiles = list(range(b, e))
        seen += tiles
        normalised = set(range(b // tiles_n, (e - 1) // tiles_n + 1))          # the blocks the prologue walks
        assert {t // tiles_n for t in tiles} <= normalised        # every A tile this unit loads was written by this unit
        max_blocks = max(max_blocks, len(normalised))
    assert seen == list(range(num))
    per_unit = -(-num // units)
    assert max_blocks <= -(-per_unit // tiles_n) + 1
    # row coverage: a pair unit's two CTAs own rows [256 blk + 128 r, +128), a single CTA rows [128 blk, +128): all rows < M covered
    rows_per_block = 256 if pair else 128
    blocks = {t // tiles_n for t in range(num)}
    assert max(blocks) * rows_per_block < M <= (max(blocks) + 1) * rows_per_block
