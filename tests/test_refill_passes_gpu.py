"""The BULKD refill (what GSB_VARIANT_AUTO runs for VERIFY_REFILL) walks its window as a verify pass and then a write
pass inside one launch. A CTA may store a tile only once every verify tile of the launch has been consumed, and every
CTA adds its count of consumed verify tiles however it leaves the verify pass. These windows put the boundary between
the passes inside the claims the CTAs hold in flight: windows of one and two tiles, where most CTAs go straight from
the verify pass to the end of the walk, windows around grid x (S + 1) tiles, and a grid larger than one wave of
resident CTAs. Bit-exact against the numpy oracle."""
import numpy as np
import pytest

from oracle import probe_oracle as po

pytestmark = pytest.mark.gpu

from gpushare_device_plugin_b200 import _abi  # noqa: E402

TILE = 16 * 256 * 8  # bytes of one BULKD tile: 256 threads x 8 words
IN_FLIGHT = 3 + 1    # claims one CTA can hold: its S = 3 issued slots and the one in hand
BACKGROUND, OLD, NEW = 11, 0x5EED, 0x5EEE
MANY = 1 << 20       # a grid request past the most CTAs the library launches: it is capped there


def read_words(gsb, offset, nbytes):
    return np.frombuffer(gsb.arena_read(0, offset, nbytes), dtype=np.uint32).reshape(-1, 4)


def refill_once(gsb, offset, nbytes, grid):
    fw, nw = offset // 16, nbytes // 16
    end = offset + nbytes
    gsb.probe(0, _abi.GSB_OP_FILL, variant=_abi.GSB_VARIANT_DIRECT, nbytes=end + 1024, seed_write=BACKGROUND)
    gsb.probe(0, _abi.GSB_OP_FILL, variant=_abi.GSB_VARIANT_DIRECT, offset=offset, nbytes=nbytes, seed_write=OLD)
    r = gsb.probe(0, _abi.GSB_OP_VERIFY_REFILL, offset=offset, nbytes=nbytes, seed_expect=OLD, seed_write=NEW,
                  grid=grid)
    assert r.variant == _abi.GSB_VARIANT_BULKD
    assert (r.mismatch_words, r.mismatch_bits, r.first_bad_offset) == (0, 0, _abi.UINT64_MAX)
    assert (r.checksum_xor, r.checksum_sum) == po.checksums(po.pattern(fw, nw, OLD))  # of the words read
    assert (r.bytes_read, r.bytes_written) == (nbytes, nbytes)
    assert np.array_equal(read_words(gsb, offset, nbytes), po.pattern(fw, nw, NEW))
    # 64 words either side still hold the background generation
    if offset >= 1024:
        assert np.array_equal(read_words(gsb, offset - 1024, 1024), po.pattern(fw - 64, 64, BACKGROUND))
    assert np.array_equal(read_words(gsb, end, 1024), po.pattern(fw + nw, 64, BACKGROUND))
    return r


@pytest.mark.parametrize("grid", [1, 3, 133, MANY], ids=["1", "3", "133", "more_than_resident"])
def test_two_pass_refill_matches_oracle_at_the_pass_boundary(gsb, small_arena, grid):
    r = refill_once(gsb, 0, TILE, grid)
    g = r.grid_ctas
    if grid == MANY:
        sm_count = gsb.device_info(0).sm_count
        assert g > 2 * sm_count  # more CTAs than fit at once (two per SM)
    else:
        assert g == grid
    edge = g * IN_FLIGHT * TILE
    for offset, nbytes in [(TILE, 2 * TILE), (1 << 20, edge // 2), (0, edge - TILE), (0, edge + TILE),
                           (16 * 3, 16 * (edge // 16 + 2048 * 5 + 7))]:
        assert offset + nbytes + 1024 <= small_arena
        refill_once(gsb, offset, nbytes, grid)
