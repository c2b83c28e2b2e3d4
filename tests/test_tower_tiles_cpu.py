"""The numpy restatement of the regression tower's tile lists (tests/tower_tiles_cases.py), checked without a GPU against the definition it
serves: every pixel of S_d lies in exactly one listed tile, no listed tile misses S_d, the list fits the library's capacity, and the
capacity and the map-size bound agree with the library's host entries."""
import numpy as np
import pytest

import tower_tiles_cases as tt


@pytest.mark.parametrize("name", sorted(tt.maps()))
@pytest.mark.parametrize("d", [1, 2, 3])
def test_tiles_cover_the_dilated_set_once(name, d):
    cand = tt.maps()[name]
    B, H, W = cand.shape
    s, lst = tt.tiles(cand, d)
    # S_d by its definition: Chebyshev distance <= d from a candidate pixel of the same image
    for b in range(B):
        ys, xs = np.nonzero(cand[b])
        yy, xx = np.mgrid[0:H, 0:W]
        want = np.zeros((H, W), bool)
        for y, x in zip(ys, xs):
            want |= (np.abs(yy - y) <= d) & (np.abs(xx - x) <= d)
        assert np.array_equal(s[b], want)
    covered = np.zeros((B, H, W), np.int32)
    for b, y0, x0, z in lst:
        assert z == 0 and 0 <= y0 < H and 0 <= x0 < W and x0 % tt.TW == 0
        tile = s[b, y0:y0 + tt.TH, x0:x0 + tt.TW]
        assert tile.any(), "a listed tile holds no pixel of S_d"
        covered[b, y0:y0 + tt.TH, x0:x0 + tt.TW] += 1
    assert (covered[s] == 1).all(), "every pixel of S_d in exactly one tile"
    assert (covered <= 1).all(), "tiles of one image do not overlap"
    assert len(lst) <= tt.cap(B, H, W)
    keys = [tuple(e[:3]) for e in lst]
    assert keys == sorted(keys), "order: image, tile row, tile column"


def test_full_map_lists_every_dense_tile():
    cand = tt.maps()["full"]
    B, H, W = cand.shape
    for d in (1, 2, 3):
        _, lst = tt.tiles(cand, d)
        assert len(lst) == B * -(-H // tt.TH) * -(-W // tt.TW)


def test_library_capacity_and_fit():
    from visualdet3d_b200 import _lib
    from visualdet3d_b200 import engine as E
    lib = _lib.load()
    for B, H, W in ((8, 24, 80), (3, 13, 37), (1, 1, 1), (2, 100, 17)):
        assert lib.vd3d_reg_tower_tile_cap(B, H, W) == tt.cap(B, H, W) == E.tower_tile_cap(B, H, W)
    assert E.tower_tiles_fit(24, 80) and E.tower_tiles_fit(48, 160) and not E.tower_tiles_fit(200, 200)
    # bad arguments return an error code and a message instead of launching anything
    assert lib.vd3d_reg_tower_tiles(None, 1, 8, 8, 1, None, None, None, None) != 0
    assert b"bad args" in lib.vd3d_last_error()
