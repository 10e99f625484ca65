"""Tile binning on the GPU against the fp64 coverage reference (tests/tile_cover_oracle.py): for every splat, the tiles holding
a pixel centre where the raster blends it are listed, and every listed tile meets its widened ellipse (must <= listed <= may).

Paths:
  * Level A: lgs_get_allocate_size + lgs_create_table + lgs_tile_range on constructed and random 2D records, which must also
    equal the oracle's tables;
  * fused path: 3D Gaussians placed, by a few corrective passes through the projection, so that their records land on the
    constructed conditions -- an ellipse ending or starting a fraction of a pixel past a tile boundary on either axis, in both
    slicing directions and with both signs of B; sub-pixel splats at the low-pass floor; opacity just above 1/255; needles
    to 100:1; off-screen centres reaching less than a pixel in; near-camera splats with more than one 512-pair emit window, in
    one warp; and a 2048x2048 grid of 65,536 8x8 tiles (32-bit tile keys).  must / may are evaluated from the records the
    kernel wrote, so the projection's rounding is not under test.  render_view_forward and ViewWorkspace must give the same
    lists; tile_count must be each splat's number of pairs, the pair total their sum; each tile's list is free of duplicates,
    in ascending depth, ties in record order;
  * end to end: the fused raster from its own lists against the fp64 oracle raster over brute-force lists (every splat in every
    tile, in depth order), to 1e-4 on every pixel outside the Q14 band (some splat's alpha within [1/256, 1/255], widened)
    and the oracle's fragile pixels.

Listed pairs that hold no pixel centre with Q <= t are wasted raster work; their number is printed, not gated."""
import math

import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import fused, pipeline
from tests import tile_cover_oracle as tc
from tests.util import axis_camera, oracle_render_lists, screen_affine, tile_segments

pytestmark = pytest.mark.gpu
TILES = [(8, 16), (12, 16), (16, 16), (8, 8)]
TILE_IDS = [f"{h}x{w}" for h, w in TILES]
HW2D = {(16, 16): (150, 181), (8, 16): (99, 203), (12, 16): (101, 131), (8, 8): (77, 91)}
HW3D = (376, 504)                  # ragged at every tile shape but 8x8; > 512 tiles at each


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def assert_cover(recs, listed, hw, tile, what):
    r = tc.check_cover(recs, listed, hw, tile)
    assert r["n_must"] > 0, what
    assert not r["missing"] and not r["extra"], (what, len(r["missing"]), r["missing"][:4], len(r["extra"]), r["extra"][:4])
    print(f"{what}: {sum(len(l) for l in listed)} pairs, {r['n_wasted']} hold no pixel centre with Q <= t")
    return r


def check_tile_lists(ranges, pid, n_pairs, depth, what):
    """Each tile's run: no duplicates, ascending depth, ties in record order.  -> per splat the tiles it is listed in."""
    start, end = tile_segments(ranges, n_pairs)
    listed = {}
    for t in np.nonzero(start >= 0)[0]:
        ids = pid[start[t]:end[t]]
        assert np.unique(ids).size == ids.size, (what, "duplicate", t)
        d = depth[ids]
        ok = (d[1:] > d[:-1]) | ((d[1:] == d[:-1]) & (ids[1:] > ids[:-1]))
        assert ok.all(), (what, "order", t)
        for i in ids.tolist():
            listed.setdefault(i, []).append(int(t))
    assert sum(len(v) for v in listed.values()) == n_pairs, what
    return listed


# ---------------------------------------------------------------------------------------------------
# Level A
# ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_level_a_tables_cover_their_pixels(cuda, tile):
    hw = HW2D[tile]
    H, W = hw
    th, tw = tile
    gx, gy = -(-W // tw), -(-H // th)
    recs = np.concatenate([np.array([c["rec"] for c in tc.constructed_cases(hw, tile)]), tc.random_cases(7, 3000, hw)])
    N = recs.shape[0]
    inp = tc.inputs_2d(recs, hw, depth=1.0 + ((np.arange(N) * 7919) % 1000) * 1e-3)     # ties and shuffled depths
    dev = lambda a: _t(a, cuda)
    assert fused.CONFIG["fix_last_tile"]
    _, _, al = fused.get_allocate_size(dev(inp["ndc"]), dev(inp["vz"]), dev(inp["inv"]), dev(inp["op"]), H, W, th, tw, None)
    order = np.argsort(inp["vz"], axis=-1, kind="stable").astype(np.int64)
    alloc = al.cpu().numpy()
    prefix = np.cumsum(np.take_along_axis(alloc, order, axis=-1), axis=-1).astype(np.int32)
    keys, vals = fused.create_table(dev(inp["ndc"]), dev(inp["inv"]), dev(inp["op"]), dev(prefix), dev(order), None, None, H, W, th, tw)
    ranges = fused.tileRange(keys, gx * gy).cpu().numpy()
    keys, vals = keys.cpu().numpy(), vals.cpu().numpy()
    okeys, ovals = oracle.create_table(inp["ndc"], inp["inv"], inp["op"], prefix, order, int(prefix[0, -1]), H, W, th, tw)
    _, _, oalloc = oracle.get_allocate_size(inp["ndc"], inp["vz"], inp["inv"], inp["op"], H, W, th, tw)
    assert np.array_equal(alloc, oalloc) and np.array_equal(keys, okeys) and np.array_equal(vals, ovals)
    listed = check_tile_lists(ranges, vals[0], keys.shape[1], inp["vz"][0].astype(np.float64), "level A")
    per = [listed.get(i, []) for i in range(N)]
    assert np.array_equal(alloc[0], [len(l) for l in per])
    assert_cover(inp["rec"], per, hw, tile, f"level A {tile}")
    # CONFIG["fix_last_tile"] = False: the reference's rectangle, which loses must tiles here, equal to the oracle's
    old = dict(fused.CONFIG)
    fused.CONFIG["fix_last_tile"] = False
    try:
        _, _, al = fused.get_allocate_size(dev(inp["ndc"]), dev(inp["vz"]), dev(inp["inv"]), dev(inp["op"]), H, W, th, tw, None)
        alloc = al.cpu().numpy()
        prefix = np.cumsum(np.take_along_axis(alloc, order, axis=-1), axis=-1).astype(np.int32)
        keys, vals = fused.create_table(dev(inp["ndc"]), dev(inp["inv"]), dev(inp["op"]), dev(prefix), dev(order), None, None, H, W, th, tw)
    finally:
        fused.CONFIG.update(old)
    _, _, oalloc = oracle.get_allocate_size(inp["ndc"], inp["vz"], inp["inv"], inp["op"], H, W, th, tw, exact_tile_bound=False)
    okeys, ovals = oracle.create_table(inp["ndc"], inp["inv"], inp["op"], prefix, order, int(prefix[0, -1]), H, W, th, tw,
                                       exact_tile_bound=False)
    assert np.array_equal(alloc, oalloc) and np.array_equal(keys.cpu().numpy(), okeys) and np.array_equal(vals.cpu().numpy(), ovals)
    lost = tc.check_cover(inp["rec"], tc.lists_by_splat(okeys[0], ovals[0], N), hw, tile)["missing"]
    assert len(lost) > 100, len(lost)


# ---------------------------------------------------------------------------------------------------
# fused path: 3D Gaussians whose records land on the constructed conditions
# ---------------------------------------------------------------------------------------------------

def gaussians_for(cases, cam, hw, S):
    """One chunk of S Gaussians (the cases first, then invisible padding) at depths increasing with the index, shaped so that
    their projected conic is the case's: scales from the eigenvalues of the 2D covariance less the 0.3 px^2 low-pass,
    rotated about the view axis."""
    n = len(cases)
    Z = 3.0 + 0.002 * np.arange(S)
    ax, bx, ay, by = screen_affine(cam, hw, Z)
    xyz = np.zeros((3, 1, S)); xyz[2, 0] = Z
    scale = np.full((3, 1, S), math.log(1e-4)); rot = np.zeros((4, 1, S)); rot[0] = 1.0
    opac = np.full((1, 1, S), -30.0)
    for i, c in enumerate(cases):
        px, py, A, B, C, o = c["rec"]
        cov = np.linalg.inv(np.array([[A, B], [B, C]]))
        lam, vec = np.linalg.eigh(cov)
        phi = math.atan2(vec[1, 1] * ay[i] / abs(ay[i]), vec[0, 1] * ax[i] / abs(ax[i]))
        sig = np.sqrt(np.maximum(lam - 0.3, 1e-6))
        xyz[0, 0, i], xyz[1, 0, i] = (px - bx[i]) / ax[i], (py - by[i]) / ay[i]
        scale[0, 0, i], scale[1, 0, i] = math.log(sig[1] / abs(ax[i])), math.log(sig[0] / abs(ax[i]))
        rot[0, 0, i], rot[3, 0, i] = math.cos(phi / 2), math.sin(phi / 2)
        opac[0, 0, i] = math.log(o / (1 - o))
    rng = np.random.default_rng(n)
    P = dict(xyz=xyz, scale=scale, rot=rot, sh_0=rng.uniform(-1.2, 1.2, (1, 3, 1, S)), sh_rest=np.zeros((0, 3, 1, S)), opacity=opac)
    return {k: v.astype(np.float32) for k, v in P.items()}, (ax, ay)


def land(cuda, cases, hw, tile, passes=4):
    """Gaussians for `cases`, moved on screen until each grazing / off-screen case's record reaches its target extent and the
    others their target centre.  -> (params, aabb, cam, n) with the Gaussians' final positions."""
    cam = axis_camera(hw)
    n = len(cases)
    S = 32 * (-(-n // 32))
    P, (ax, ay) = gaussians_for(cases, cam, hw, S)
    for _ in range(passes):
        aabb = aabb_of(P)
        _, st, _ = forward(cuda, P, aabb, cam, hw, tile)
        rec = st.packed[0, :n, :6].double().cpu().numpy()
        for i, c in enumerate(cases):
            px, py, A, B, C, o = rec[i]
            ex, ey = tc._extent(A, B, C, tc.threshold(o)) if o > 0 else (0.0, 0.0)
            cur = [px, py]
            want = [c["rec"][0], c["rec"][1]]
            if "side" in c:
                a = c["axis"]
                cur[a] += (ex, ey)[a] if c["side"] == "max" else -(ex, ey)[a]
                want[a] = c["value"]
            P["xyz"][0, 0, i] += np.float32((want[0] - cur[0]) / ax[i])
            P["xyz"][1, 0, i] += np.float32((want[1] - cur[1]) / ay[i])
    return P, aabb_of(P), cam, n


def aabb_of(P):
    x = P["xyz"][:, 0].astype(np.float64)
    lo, hi = x.min(1), x.max(1)
    return ((0.5 * (lo + hi))[:, None].astype(np.float32), (0.5 * (hi - lo) + 1.0)[:, None].astype(np.float32))


def forward(cuda, P, aabb, cam, hw, tile):
    Pt = {k: _t(v, cuda) for k, v in P.items()}
    A = [_t(a, cuda) for a in aabb]
    C = {k: _t(v, cuda) for k, v in cam.items()}
    img, st, _ = pipeline.render_view_forward(Pt, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 0, hw, tile)
    return img, st, (Pt, A, C)


def live_mask(rec, ndc, depth):
    """Records the projection keeps (fused.cu: lgs_splat_setup's visibility test)."""
    A, B, C, o = rec[:, 2], rec[:, 3], rec[:, 4], rec[:, 5]
    return (np.abs(ndc[:, 0]) <= 1.3) & (np.abs(ndc[:, 1]) <= 1.3) & (depth > 0.2) & (o >= np.float32(1.0) / np.float32(255.0)) & \
        (A > 0) & (C > 0) & (B * B - A * C < 0)


def fused_checks(cuda, P, aabb, cam, n, hw, tile, what):
    """Forward through render_view_forward and ViewWorkspace; every list check.  -> (img, state, recs f64[n, 6], listed)."""
    H, W = hw
    img, st, (Pt, A, C) = forward(cuda, P, aabb, cam, hw, tile)
    assert st.n_chunks_visible == 1
    packed = st.packed[0].cpu().numpy()
    rec = packed[:, :6].astype(np.float64)
    depth = packed[:, 9].astype(np.float64)
    D = st.n_pairs
    pid = st.sorted_pid[0].cpu().numpy()
    listed = check_tile_lists(st.ranges.cpu().numpy(), pid, D, depth, what)
    tcount = st.tile_count.cpu().numpy()
    per = [listed.get(i, []) for i in range(packed.shape[0])]
    assert np.array_equal(tcount, [len(l) for l in per]), what
    assert int(st.counters[1]) == D == int(tcount.sum())
    live = live_mask(rec, packed[:, 10:12], depth)
    assert live[:n].all() and not live[n:].any(), what
    assert_cover(rec[:n], per[:n], hw, tile, what)
    # the GPU-driven workspace builds the same lists
    ws = pipeline.ViewWorkspace(Pt, hw, tile, pair_capacity=D + 4096, use_graphs=False)
    ws.forward(Pt, A[0], A[1], C, 0, clamp_zero=False)
    torch.cuda.synchronize()
    assert int(ws.vparams[1]) == D and int(ws.vparams[4]) == 0
    assert np.array_equal(ws.tcount.cpu().numpy(), tcount)
    wl = check_tile_lists(ws.ranges.cpu().numpy(), ws.sorted_pid[0, :D].cpu().numpy(), D, depth, what + " (workspace)")
    assert wl == listed, what
    return img, st, rec, per


def landed_cases(cuda, hw, tile):
    cases = tc.constructed_cases(hw, tile)
    P, aabb, cam, n = land(cuda, cases, hw, tile)
    return cases, P, aabb, cam, n


def assert_conditions(cases, rec, hw, tile, per):
    """The records reached the conditions the cases were built for."""
    n_edge = 0
    for i, c in enumerate(cases):
        px, py, A, B, C, o = rec[i]
        ex, ey = tc._extent(A, B, C, tc.threshold(o))
        if c["kind"] == "grazing":
            a = c["axis"]
            end = (px, py)[a] + ((ex, ey)[a] if c["side"] == "max" else -(ex, ey)[a])
            edge = c["k"] * c["T"]
            if c["side"] == "max":
                assert edge + 1e-3 < end < edge + 1 - 1e-3, (i, c, end)
            else:
                assert edge - 1 + 1e-3 < end < edge - 1e-3, (i, c, end)
            gx = -(-hw[1] // tile[1])
            must = tc.must_tiles(rec[i], hw, tile)
            n_edge += c["side"] == "max" and c["k"] in (must % gx if a == 0 else must // gx).tolist()
        elif c["kind"] == "offscreen":
            a = c["axis"]
            end = (px, py)[a] + ((ex, ey)[a] if c["side"] == "max" else -(ex, ey)[a])
            assert abs(end - c["value"]) < 2e-3, (i, c, end)
            ctr = (px, py)[a]
            assert ctr < -0.5 or ctr > hw[1 - a] - 0.5, (i, c)
    n_grazing_max = sum(c["kind"] == "grazing" and c["side"] == "max" for c in cases)
    assert n_edge >= 0.5 * n_grazing_max, (n_edge, n_grazing_max)       # the boundary pixel line holds a must pixel
    big = [len(per[i]) for i, c in enumerate(cases) if c["kind"] == "big"]
    assert sum(b > 512 for b in big) >= 3, big                           # runs over several emit windows, in one warp


@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_fused_lists_cover_their_pixels(cuda, tile):
    hw = HW3D
    cases, P, aabb, cam, n = landed_cases(cuda, hw, tile)
    img, st, rec, per = fused_checks(cuda, P, aabb, cam, n, hw, tile, f"fused {tile}")
    assert_conditions(cases, rec, hw, tile, per)
    end_to_end(img, st, rec, n, hw, tile)


def test_fused_lists_cover_their_pixels_32bit_keys(cuda):
    """A 2048x2048 image at 8x8 tiles: 65,536 tiles, so the fused path takes 32-bit tile keys."""
    hw, tile = (2048, 2048), (8, 8)
    assert (256 * 256 + 1) >= 65536
    cases, P, aabb, cam, n = landed_cases(cuda, hw, tile)
    _, st, rec, per = fused_checks(cuda, P, aabb, cam, n, hw, tile, "fused 2048x2048 8x8")
    assert_conditions(cases, rec, hw, tile, per)


# ---------------------------------------------------------------------------------------------------
# end to end: the fused raster against the fp64 oracle over brute-force lists
# ---------------------------------------------------------------------------------------------------

def q14_mask(rec, n, hw, delta=tc.DELTA):
    """Pixels where some splat's fp64 alpha lies in [1/256, 1/255] widened by delta: there the raster blends a splat only when
    its tile is listed for a reason other than the pixel itself (SURVEY Q14)."""
    H, W = hw
    m = np.zeros(hw, bool)
    for i in range(n):
        px, py, A, B, C, o = rec[i]
        tq = 2 * math.log(256 * o * (1 + delta))
        e = tc._extent(A, B, C, tq)
        if e is None:
            continue
        x0, x1 = max(0, math.ceil(px - e[0])), min(W - 1, math.floor(px + e[0]))
        y0, y1 = max(0, math.ceil(py - e[1])), min(H - 1, math.floor(py + e[1]))
        if x0 > x1 or y0 > y1:
            continue
        dx = px - np.arange(x0, x1 + 1)[None, :]
        dy = py - np.arange(y0, y1 + 1)[:, None]
        a = o * np.exp(-0.5 * (A * dx * dx + 2 * B * dx * dy + C * dy * dy))
        m[y0:y1 + 1, x0:x1 + 1] |= (a >= (1 - delta) / 256) & (a <= (1 + delta) / 255)
    return m


def end_to_end(img, st, rec, n, hw, tile):
    H, W = hw
    th, tw = tile
    gx, gy = -(-W // tw), -(-H // th)
    ntile = gx * gy
    packed = st.packed[0].cpu().numpy()
    order = np.lexsort((np.arange(n), packed[:n, 9]))           # depth, ties in record order
    pid = np.tile(order.astype(np.int32), ntile)[None]
    ranges = np.full((1, ntile + 2), -1, np.int32)
    ranges[0, 1:] = np.arange(ntile + 1) * n
    oimg, oT, frag = oracle_render_lists(packed, pid, ranges, hw, tile)
    mask = q14_mask(rec, n, hw) | frag[:H, :W]
    assert mask.mean() < 0.03, mask.mean()
    got = img[0, :, :H, :W].cpu().numpy().astype(np.float64)
    err = np.abs(got - oimg[:, :H, :W])[:, ~mask]
    terr = np.abs(st.T[0, 0, :H, :W].cpu().numpy() - oT[:H, :W])[~mask]
    print(f"end to end {tile}: max |img - oracle| {err.max():.2e}, |T - oracle| {terr.max():.2e}, masked {mask.mean():.4f}")
    assert err.max() < 1e-4 and terr.max() < 1e-4, (err.max(), terr.max(), np.argwhere(np.abs(got - oimg[:, :H, :W]).max(0) * ~mask > 1e-4)[:5])
