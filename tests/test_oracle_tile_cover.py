"""The oracle's tile binning (orc_get_allocate_size + orc_create_table, the fp32 restatement the GPU kernels match bit for bit)
against the fp64 coverage reference of tests/tile_cover_oracle.py: every tile holding a pixel centre where the raster blends
a splat is in that splat's list, and no listed tile lies off the splat's widened ellipse (must <= listed <= may).

Cases: random splats at all four tile shapes on ragged images with off-screen centres, and the constructed cases the GPU
module also runs -- ellipses ending or starting a fraction of a pixel past a tile boundary on either axis and in either
slicing direction, sub-pixel splats at the low-pass floor, opacity just above 1/255, needles, off-screen centres reaching
less than a pixel in, splats over hundreds of tiles.  The reference's rectangle (exact_tile_bound=False) loses tiles on
these cases; one test pins that, so the cases keep exercising the fault they were built for."""
import math

import numpy as np
import pytest

import oracle
from tests import tile_cover_oracle as tc

TILES = [(16, 16), (8, 16), (12, 16), (8, 8)]
TILE_IDS = [f"{h}x{w}" for h, w in TILES]
RANDOM = {(16, 16): (0, (128, 160)), (8, 16): (1, (96, 200)), (12, 16): (2, (100, 130)), (8, 8): (3, (77, 91))}
HW = {(16, 16): (150, 181), (8, 16): (99, 203), (12, 16): (101, 131), (8, 8): (77, 91)}


def oracle_lists(recs, hw, tile, exact=True, depth=None):
    """Bin the 2D records with the fp32 oracle -> (inputs, per-splat tile lists, allocate sizes)."""
    inp = tc.inputs_2d(recs, hw, depth)
    _, vals, _, keys = oracle.binning(inp["ndc"], inp["vz"], inp["inv"], inp["op"], None, hw, tile, fix_last=exact)
    _, _, alloc = oracle.get_allocate_size(inp["ndc"], inp["vz"], inp["inv"], inp["op"], hw[0], hw[1], *tile, exact_tile_bound=exact)
    return inp, tc.lists_by_splat(keys[0], vals[0], len(recs)), alloc[0]


def assert_cover(recs, hw, tile, exact=True, what=""):
    inp, listed, alloc = oracle_lists(recs, hw, tile, exact)
    assert np.array_equal(alloc, [len(l) for l in listed]), what
    assert all(len(l) == len(set(l)) for l in listed), what
    r = tc.check_cover(inp["rec"], listed, hw, tile)
    assert r["n_must"] > 0
    assert not r["missing"] and not r["extra"], (what, len(r["missing"]), r["missing"][:4], len(r["extra"]), r["extra"][:4])
    return inp, r


def constructed(hw, tile):
    """The constructed cases as one record array, and the grazing cases' metadata."""
    cases = tc.constructed_cases(hw, tile)
    return np.array([c["rec"] for c in cases], np.float64), [c for c in cases if c["kind"] == "grazing"]


def test_reference_helpers():
    """The coverage reference itself on cases with a known answer: a unit circle at a pixel centre, and the rectangle
    minimum against brute force."""
    r = (20.0, 20.0, 1.0, 0.0, 1.0, 0.99)
    t = tc.threshold(0.99)
    rad = math.sqrt(t)
    must = tc.must_tiles(r, (64, 64), (8, 8))
    want = {(y // 8) * 8 + x // 8 for y in range(64) for x in range(64) if (x - 20) ** 2 + (y - 20) ** 2 <= t * (1 - 1e-4) - 1e-4}
    assert set(must.tolist()) == want
    may = tc.may_tiles(r, (64, 64), (8, 8))
    assert set(must.tolist()) <= set(may.tolist())
    lo, hi = int((20 - rad) // 8), int((20 + rad) // 8)
    assert set(may.tolist()) <= {v * 8 + u for v in range(lo, hi + 1) for u in range(lo, hi + 1)}
    rng = np.random.default_rng(0)
    for _ in range(200):
        A, B, C = tc.conic(*rng.uniform(0.5, 5, 2), rng.uniform(0, np.pi))
        X0, Y0 = rng.uniform(-6, 6, 2)
        X1, Y1 = X0 + rng.uniform(0, 4), Y0 + rng.uniform(0, 4)
        xs, ys = np.meshgrid(np.linspace(X0, X1, 201), np.linspace(Y0, Y1, 201))
        brute = (A * xs * xs + 2 * B * xs * ys + C * ys * ys).min()
        got = float(tc._rect_min_q(A, B, C, np.array(X0), np.array(X1), np.array(Y0), np.array(Y1)))
        assert got <= brute + 1e-12 and brute - got < 1e-3 * max(1.0, brute)


@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_random_splats_cover_their_pixels(tile):
    """3,000 random splats per tile shape (sigma 0.3-60 px, anisotropy to 60:1, opacity 1/255-0.99, centres in ndc +-1.3) on
    images that are not a multiple of the tile."""
    seed, hw = RANDOM[tile]
    recs = tc.random_cases(seed, 3000, hw)
    inp, r = assert_cover(recs, hw, tile, what="random")
    assert (np.abs(inp["nx"]) > 1.0).sum() > 500 and (np.abs(inp["ny"]) > 1.0).sum() > 500     # off-screen centres
    print(f"tile {tile}: {r['n_must']} must tiles, {r['n_wasted']} listed pairs hold no pixel centre with Q <= t")


@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_constructed_splats_cover_their_pixels(tile):
    hw = HW[tile]
    recs, g = constructed(hw, tile)
    inp, r = assert_cover(recs, hw, tile, what="constructed")
    # each grazing case reaches its condition: bbox_max in [kT, kT + 1) or bbox_min in (kT - 1, kT] (fp64 extent of the fp32
    # record), and the pixel centre on the boundary is a must pixel
    for j, c in enumerate(g):
        px, py, A, B, C, o = inp["rec"][j]
        ex, ey = tc._extent(A, B, C, tc.threshold(o))
        ctr, e = (px, ex) if c["axis"] == 0 else (py, ey)
        edge = c["k"] * c["T"]
        if c["side"] == "max":
            assert edge + 1e-3 < ctr + e < edge + 1 - 1e-3, (j, c)
        else:
            assert edge - 1 + 1e-3 < ctr - e < edge - 1e-3, (j, c)
        must = tc.must_tiles(inp["rec"][j], hw, tile)
        gx = -(-hw[1] // tile[1])
        cols = must % gx if c["axis"] == 0 else must // gx
        assert c["k"] in cols.tolist() or c["side"] == "min", (j, c)
    assert np.all(np.abs(inp["nx"]) <= 1.3) and np.all(np.abs(inp["ny"]) <= 1.3)


@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_reference_rectangle_loses_tiles_on_these_cases(tile):
    """With the reference's rectangle floor((bbox_max + T - 1) / T) the same oracle misses must tiles on the grazing and
    random cases; the corrected rule is the only difference between this and the tests above."""
    hw = HW[tile]
    recs, _ = constructed(hw, tile)
    inp, listed, _ = oracle_lists(recs, hw, tile, exact=False)
    r = tc.check_cover(inp["rec"], listed, hw, tile)
    assert len(r["missing"]) >= 20 and not r["extra"], len(r["missing"])
    seed, rhw = RANDOM[tile]
    inp, listed, _ = oracle_lists(tc.random_cases(seed, 3000, rhw), rhw, tile, exact=False)
    assert len(tc.check_cover(inp["rec"], listed, rhw, tile)["missing"]) > 100


def test_sub_pixel_splat_below_a_tile_row():
    """sigma = 0.548 px (the low-pass floor), o = 0.99, 8x16 tiles, centre 0.83 px above a tile-row boundary: the pixel just
    below the boundary has alpha 0.314, and its tile is listed."""
    hw, tile = (64, 64), (8, 16)
    s = math.sqrt(0.3)
    rec = np.array([(20.0, 16 - 0.83, *tc.conic(s, s, 0.0), 0.99)])
    inp, listed, _ = oracle_lists(rec, hw, tile)
    px, py, A, B, C, o = inp["rec"][0]
    alpha = o * math.exp(-0.5 * (A * (px - 20) ** 2 + C * (py - 16) ** 2))
    assert abs(alpha - 0.314) < 1e-3
    assert (16 // 8) * 4 + 20 // 16 in listed[0]
    _, old, _ = oracle_lists(rec, hw, tile, exact=False)
    assert (16 // 8) * 4 + 20 // 16 not in old[0]


def test_count_and_emit_use_one_rule():
    """create_table writes exactly the pairs the counts promised, with either rule, so no run overlaps the next one."""
    hw, tile = HW[(8, 16)], (8, 16)
    recs, _ = constructed(hw, tile)
    for exact in (True, False):
        inp, listed, alloc = oracle_lists(recs, hw, tile, exact)
        assert sum(len(l) for l in listed) == int(alloc.sum())
        assert np.array_equal(alloc, [len(l) for l in listed])
