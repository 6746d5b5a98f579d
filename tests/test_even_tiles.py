"""No GPU needed: distributed.even_tiles, the row bands of the multi-GPU from-materials calls. Its inner boundaries must be even
rows (a band's 2x2 quads are the frame's quads), its sizes differ by at most two, and the bands cover [0, n) in order."""
import pytest

from vqengine_b200.distributed import equal_tiles, even_tiles


@pytest.mark.parametrize("world", range(1, 9))
def test_bands_cover_the_frame_with_even_inner_boundaries(world):
    for n in range(1, 4322):
        t = even_tiles(n, world)
        assert len(t) == world and t[0][0] == 0 and t[-1][1] == n, (n, t)
        assert all(t[i][1] == t[i + 1][0] for i in range(world - 1)), (n, t)
        assert all(a <= b for a, b in t), (n, t)
        assert all(b % 2 == 0 for _, b in t[:-1]), (n, t)
        sizes = [b - a for a, b in t]
        assert max(sizes) - min(sizes) <= 2, (n, t)


def test_1080_rows_over_8_ranks():
    """equal_tiles cuts 1080 rows at row 135; even_tiles does not"""
    assert 135 in [b for _, b in equal_tiles(1080, 8)]
    t = even_tiles(1080, 8)
    assert t == [(0, 136), (136, 270), (270, 406), (406, 540), (540, 676), (676, 810), (810, 946), (946, 1080)]


def test_odd_last_row_goes_to_a_small_band():
    assert even_tiles(7, 2) == [(0, 4), (4, 7)]
    assert even_tiles(4321, 8)[-1] == (3780, 4321)
