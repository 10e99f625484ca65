"""The raster forward and backward kernels against the fp64 oracle on constructed edge cases, at every compiled variant.

The inputs of rasterize_forward / rasterize_backward are built directly -- records, hand-made tile lists and ranges, no
projection or binning -- so that each case sits where the kernels' structure could go wrong:
  * chunks:     list lengths on either side of the 32-record staging chunks, 0 to ~1000, empty tiles in between;
  * saturation: every pixel of a tile saturating at list position k, and a tile where only half the warp saturates;
  * clamp:      splats whose alpha is clamped to 255/256 at their centre, and pixels a safe margin either side of 1/256;
  * views:      three views in one launch, with different records and lists per view;
  * padded:     a 37x53 image, padded to whole tiles, compared on the full padded planes;
  * needles:    isolated splats up to 100:1 at several angles, whose position gradient is checked per splat;
and a screen-sized splat at 512x512 and 3840x2160 checks the range of the deterministic backward's fixed-point accumulator.

Splat centres lie on a grid where pack_kernel's fp32 screen mapping is exact, so the fp64 oracle sees the kernel's centres.
Forward variants: default, bulk staging, pixel pairs, with and without statistics; backward variants: pixel-pair (v2), v2
deterministic, scalar (v1) with the deferred and the butterfly reduce, v1 with bulk staging; each at 1, 2 and 4 warps per
block and the four tile shapes."""
import functools
import math

import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, fused
from tests.util import rel_err, scaled_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
FRAGILE_EPS = 2e-6
TILES = [(8, 16), (12, 16), (16, 16), (8, 8)]
TILE_IDS = [f"{h}x{w}" for h, w in TILES]
WPB = [1, 2, 4]

DEFAULTS = dict(staging=0, forward_pairs=0, backward_kernel=2, backward_reduce=1, deterministic=0, warps_per_block=4)
# forward variant -> (switches, enable_statistic).  The pixel-pair forward has no statistics form.
FWD = {"default": ({}, False), "default_stat": ({}, True), "bulk": (dict(staging=1), False), "bulk_stat": (dict(staging=1), True),
       "pairs": (dict(forward_pairs=1), False)}
BWD = {"v2": {}, "v2_det": dict(deterministic=1), "v1_deferred": dict(backward_kernel=1),
       "v1_butterfly": dict(backward_kernel=1, backward_reduce=0), "v1_bulk": dict(backward_kernel=1, staging=1)}
GRAD_NAMES = ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")


def _set(sw):
    for k, v in sw.items():
        _lib.call("lgs_set_" + k, v)


@pytest.fixture
def switch():
    """switch(**sw) selects a raster variant (DEFAULTS for every switch not named); the defaults are restored when the test
    ends, whatever happens."""
    try:
        yield lambda **sw: _set({**DEFAULTS, **sw})
    finally:
        _set(DEFAULTS)


# ---------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------

def ndc_for(p, size):
    """fp32 ndc of the screen coordinate p (px), snapped to the grid p = j size/4096 - 0.5 on which pack_kernel's fp32 mapping
    ((ndc + 1) 0.5 size - 0.5, each op rounded) is exact -> (ndc, snapped p in fp64).  The oracle maps in fp64, so it then sees
    the kernel's centre bit for bit."""
    j = np.rint((np.asarray(p, np.float64) + 0.5) * 4096.0 / size)
    n = (2.0 * j / 4096.0 - 1.0).astype(np.float32)
    q = j * size / 4096.0 - 0.5
    f32 = (n + np.float32(1)) * np.float32(0.5) * np.float32(size) - np.float32(0.5)
    assert np.array_equal(f32.astype(np.float64), q)
    return n, q


def conic(s1, s2, theta):
    """Inverse covariance (A, B, C) of a Gaussian with standard deviations s1 along angle theta and s2 across it."""
    c, s = np.cos(theta), np.sin(theta)
    a1, a2 = 1.0 / np.square(s1), 1.0 / np.square(s2)
    return c * c * a1 + s * s * a2, c * s * (a1 - a2), s * s * a1 + c * c * a2


def tile_lists(per_view, ntile):
    """Per-view {tile id (1-based): [splat ids]} -> (sorted_pid i32[V, cap], ranges i32[V, ntile + 2]).  ranges[t] is the start
    of tile t's run and ranges[t + 1] its end, as the kernels read them; a tile absent from the dict keeps -1, or reads as
    empty (start = end) when it follows a listed tile."""
    ids, rgs = [], []
    for lists in per_view:
        r = np.full(ntile + 2, -1, np.int32)
        flat = []
        for t in range(1, ntile + 1):
            if t in lists:
                r[t] = len(flat)
                flat += [int(i) for i in lists[t]]
                r[t + 1] = len(flat)
        ids.append(flat)
        rgs.append(r)
    pid = np.zeros((len(ids), max(1, max(len(f) for f in ids))), np.int32)
    for b, f in enumerate(ids):
        pid[b, :len(f)] = f
    return pid, np.stack(rgs)


def box_lists(px, py, rad, order, H, W, th, tw):
    """{tile id: splat ids in `order`} of the splats whose box of half-size rad reaches the tile (padded grid)."""
    gx, gy = -(-W // tw), -(-H // th)
    lists = {}
    for i in order:
        x0, x1 = math.floor((px[i] - rad[i]) / tw), math.floor((px[i] + rad[i]) / tw)
        y0, y1 = math.floor((py[i] - rad[i]) / th), math.floor((py[i] + rad[i]) / th)
        for ty in range(max(y0, 0), min(y1, gy - 1) + 1):
            for tx in range(max(x0, 0), min(x1, gx - 1) + 1):
                lists.setdefault(ty * gx + tx + 1, []).append(int(i))
    return lists


def assemble(H, W, tile, px, py, s1, s2, theta, op, col, lists):
    """[V, N] centres and shapes, op [N], col [V, 3, N], per-view tile lists -> the raster inputs (fp32) and, in fp64, the
    centres and conics the kernel sees."""
    th, tw = tile
    gx, gy = -(-W // tw), -(-H // th)
    V, N = np.shape(px)
    nx, qx = ndc_for(px, W)
    ny, qy = ndc_for(py, H)
    ndc = np.zeros((V, 4, N), np.float32)
    ndc[:, 0], ndc[:, 1], ndc[:, 2], ndc[:, 3] = nx, ny, 1.0, 1.0
    A, B, C = (np.asarray(a, np.float32) for a in conic(np.asarray(s1, np.float64), np.asarray(s2, np.float64), np.asarray(theta, np.float64)))
    inv = np.ascontiguousarray(np.stack([np.stack([A, B], 1), np.stack([B, C], 1)], 1))       # [V, 2, 2, N]
    pid, ranges = tile_lists(lists, gx * gy)
    return dict(H=H, W=W, Hp=gy * th, Wp=gx * tw, ndc=ndc, inv=inv, col=np.asarray(col, np.float32),
                op=np.asarray(op, np.float32).reshape(1, N), pid=pid, ranges=ranges, px=qx, py=qy,
                A=A.astype(np.float64), B=B.astype(np.float64), C=C.astype(np.float64))


LENGTHS = [1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 96, 97, 1000]


def case_chunks(tile):
    """One tile per list length in LENGTHS, each followed by an empty tile (start = end) and a tile with range -1 (tile 1 is
    -1 too).  Faint splats: every pixel stays active through its whole list."""
    th, tw = tile
    gx, gy = 7, 7
    H, W = gy * th, gx * tw
    rng = np.random.default_rng(11)
    cols = [[], [], [], [], [], [], []]               # px py s1 s2 theta op col
    lists, n = {}, 0
    for j, L in enumerate(LENGTHS):
        t = 2 + 3 * j                                  # tiles 2, 5, 8, ...; the two after each stay empty
        tx, ty = (t - 1) % gx, (t - 1) // gx
        lo, hi = ((4.0, 8.0), (0.003, 0.008)) if L > 100 else ((2.0, 5.0), (0.01, 0.1))
        cols[0] += list(rng.uniform(tx * tw, tx * tw + tw - 1, L)); cols[1] += list(rng.uniform(ty * th, ty * th + th - 1, L))
        cols[2] += list(rng.uniform(*lo, L)); cols[3] += list(rng.uniform(*lo, L)); cols[4] += list(rng.uniform(0, np.pi, L))
        cols[5] += list(rng.uniform(*hi, L)); cols[6] += list(rng.uniform(0.1, 0.9, (L, 3)))
        lists[t] = list(range(n, n + L))
        n += L
    px, py, s1, s2, ang, op, col = (np.asarray(c) for c in cols)
    return assemble(H, W, tile, px[None], py[None], s1[None], s2[None], ang[None], op, col.T[None], [lists])


SAT_K = [2, 3, 4, 5, 6, 7, 8, 31, 32, 33, 64]
HALF_K = [3, 33]


def _stack_alpha(k):
    """Opacities of a k-splat stack that takes T across 1/8192 = 2^-13 at its k-th splat and not before, with a wide margin:
    the first k - 1 bring T to 2^-11 (k = 2: one clamped splat, T = 2^-8), the k-th multiplies it by 0.02."""
    a = min(1.0 - 2.0 ** (-11.0 / (k - 1)), 0.999)
    return [a] * (k - 1) + [0.98]


def case_saturation(tile):
    """Tiles whose pixels all saturate at list position k for k in SAT_K (k = 1 cannot be reached: alpha <= 255/256 leaves
    T >= 1/256 after one splat), each list running 40 opaque splats past k; and, for k in HALF_K, tiles where each row of the
    top half (lanes 0-15) saturates at its own position past k and the bottom half (lanes 16-31) never does."""
    th, tw = tile
    gx, gy = 4, 4
    H, W = gy * th, gx * tw
    rng = np.random.default_rng(12)
    rows, lists = [], {}

    def add(x, y, s1, s2, o):
        rows.append((x, y, s1, s2, 0.0, o, *rng.uniform(0.1, 0.9, 3)))
        return len(rows) - 1

    def tail(tx, ty, n, o_range):
        return [add(rng.uniform(tx * tw, tx * tw + tw - 1), rng.uniform(ty * th, ty * th + th - 1), rng.uniform(2, 6), rng.uniform(2, 6),
                    rng.uniform(*o_range)) for _ in range(n)]

    t = 1
    for k in SAT_K:
        tx, ty = (t - 1) % gx, (t - 1) // gx
        cx, cy = tx * tw + (tw - 1) / 2, ty * th + (th - 1) / 2
        lists[t] = [add(cx, cy, 1000.0, 1000.0, o) for o in _stack_alpha(k)] + tail(tx, ty, 40, (0.5, 0.9))
        t += 1
    for k in HALF_K:
        tx, ty = (t - 1) % gx, (t - 1) // gx
        cx = tx * tw + (tw - 1) / 2
        R = th // 2                                    # rows of the top half: one stack per row, narrow in y
        ids = [[add(cx, ty * th + r, 1000.0, 0.25, o) for r in range(R)] for o in _stack_alpha(k)]
        lists[t] = [i for row in ids for i in row] + tail(tx, ty, 40, (0.02, 0.1))
        t += 1
    r = np.asarray(rows)
    return assemble(H, W, tile, r[None, :, 0], r[None, :, 1], r[None, :, 2], r[None, :, 3], r[None, :, 4], r[:, 5], r[:, 6:9].T[None],
                    [lists])


def case_clamp(tile):
    """In every tile: three faint splats, then splats with o G >= 255/256 at their centre (clamped alpha) whose x neighbours
    get alpha ~1.3/256 and y neighbours ~0.7/256 (blended / skipped with a wide margin), then three faint splats behind."""
    th, tw = tile
    W, H = 128, 4 * th
    gx, gy = W // tw, 4
    rng = np.random.default_rng(13)
    rows, lists = [], {}
    opq = [0.999, 1.0, 0.9985]
    for t in range(1, gx * gy + 1):
        tx, ty = (t - 1) % gx, (t - 1) // gx
        ids = []
        for _ in range(3):
            rows.append((rng.uniform(tx * tw, tx * tw + tw), rng.uniform(ty * th, ty * th + th), rng.uniform(4, 8), rng.uniform(4, 8),
                         rng.uniform(0, np.pi), rng.uniform(0.05, 0.2), *rng.uniform(0.1, 0.9, 3)))
            ids.append(len(rows) - 1)
        for y in range(ty * th + 2, ty * th + th - 1, 4):
            for x in range(tx * tw + 2, tx * tw + tw - 1, 4):
                o = opq[len(rows) % 3]
                sx = 1.0 / math.sqrt(-2.0 * math.log(1.3 / (256.0 * o)))
                sy = 1.0 / math.sqrt(-2.0 * math.log(0.7 / (256.0 * o)))
                rows.append((x, y, sx, sy, 0.0, o, *rng.uniform(0.1, 0.9, 3)))
                ids.append(len(rows) - 1)
        for _ in range(3):
            rows.append((rng.uniform(tx * tw, tx * tw + tw), rng.uniform(ty * th, ty * th + th), rng.uniform(4, 8), rng.uniform(4, 8),
                         rng.uniform(0, np.pi), rng.uniform(0.05, 0.2), *rng.uniform(0.1, 0.9, 3)))
            ids.append(len(rows) - 1)
        lists[t] = ids
    r = np.asarray(rows)
    return assemble(H, W, tile, r[None, :, 0], r[None, :, 1], r[None, :, 2], r[None, :, 3], r[None, :, 4], r[:, 5], r[:, 6:9].T[None],
                    [lists])


def _random_views(tile, H, W, V, N, seed):
    th, tw = tile
    rng = np.random.default_rng(seed)
    px = rng.uniform(-3, W + 3, (V, N)); py = rng.uniform(-3, H + 3, (V, N))
    s1 = rng.uniform(1, 6, (V, N)); s2 = rng.uniform(1, 6, (V, N)); ang = rng.uniform(0, np.pi, (V, N))
    op = rng.uniform(0.05, 0.6, N)
    col = rng.uniform(0.05, 0.95, (V, 3, N))
    rad = 3.5 * np.maximum(s1, s2)
    lists = [box_lists(px[b], py[b], rad[b], rng.permutation(N), H, W, th, tw) for b in range(V)]
    return assemble(H, W, tile, px, py, s1, s2, ang, op, col, lists)


def case_views(tile):
    """Three views in one launch: different records, depth orders and lists per view (the opacity is shared, as in the ABI)."""
    return _random_views(tile, 80, 96, 3, 300, 14)


def case_padded(tile):
    """A 37x53 image: every tile shape pads it, and the padded pixels are rendered and differentiated like the others."""
    return _random_views(tile, 37, 53, 1, 120, 15)


NEEDLES = [(1, 0, 3.0), (5, 15, 1.0), (20, 30, 0.8), (20, 45, 1.0), (50, 45, 0.6), (100, 45, 0.5), (100, 0, 0.5), (100, 90, 0.5),
           (100, 135, 0.5)]                      # (aspect ratio, angle in degrees, minor standard deviation in px)


def case_needles(tile):
    """Nine isolated splats in a 1024x1024 image, one per 3x3 cell, up to 100:1 at several angles: no pixel is reached by
    two of them (checked), so each lies alone on black."""
    th, tw = tile
    H = W = 1024
    rng = np.random.default_rng(16)
    cell = W / 3
    px = np.array([(i % 3 + 0.5) * cell for i in range(9)]) + rng.uniform(-4, 4, 9)
    py = np.array([(i // 3 + 0.5) * cell for i in range(9)]) + rng.uniform(-4, 4, 9)
    s2 = np.array([m for _, _, m in NEEDLES]); s1 = s2 * np.array([r for r, _, _ in NEEDLES])
    ang = np.radians([a for _, a, _ in NEEDLES])
    op = rng.uniform(0.5, 0.9, 9)
    col = rng.uniform(0.2, 0.9, (1, 3, 9))
    lists = box_lists(px, py, 3.5 * s1, range(9), H, W, th, tw)
    sc = assemble(H, W, tile, px[None], py[None], s1[None], s2[None], ang[None], op, col, [lists])
    alpha = _splat_alpha(sc, range(9))
    assert ((alpha >= 0.5 / 256).sum(0) <= 1).all()
    return sc


def _splat_alpha(sc, ids, b=0):
    """o G of the given splats over the padded plane, fp64 [len(ids), Hp, Wp] (with the pixel offsets dx, dy if one id)."""
    y, x = np.mgrid[0:sc["Hp"], 0:sc["Wp"]].astype(np.float64)
    out = []
    for i in ids:
        dx, dy = sc["px"][b, i] - x, sc["py"][b, i] - y
        pw = -0.5 * (sc["A"][b, i] * dx * dx + 2 * sc["B"][b, i] * dx * dy + sc["C"][b, i] * dy * dy)
        out.append(float(sc["op"][0, i]) * np.exp(pw))
    return np.stack(out)


CASES = {"chunks": case_chunks, "saturation": case_saturation, "clamp": case_clamp, "views": case_views, "padded": case_padded,
         "needles": case_needles}


@functools.lru_cache(maxsize=None)
def scene(case, tile):
    return CASES[case](tile)


def f64(a):
    return np.asarray(a, np.float64)


@functools.lru_cache(maxsize=None)
def oracle_forward(case, tile):
    """-> (img, T, last, fragment_count, fragment_weight, fragile) of the fp64 oracle."""
    sc = scene(case, tile)
    return oracle.rasterize_forward(sc["pid"], sc["ranges"], f64(sc["ndc"]), f64(sc["inv"]), f64(sc["col"]), f64(sc["op"]), None,
                                    sc["H"], sc["W"], tile[0], tile[1], enable_statistic=True, fragile_eps=FRAGILE_EPS)


def dev(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def run_forward(cuda, sc, tile, stat):
    """-> (img, T, last, packed, fragment_count, fragment_weight) of the kernel under the current switches."""
    img, T, _, last, packed, fc, fw = fused.rasterize_forward(dev(sc["pid"], cuda), dev(sc["ranges"], cuda), dev(sc["ndc"], cuda),
                                                              dev(sc["inv"], cuda), dev(sc["col"], cuda), dev(sc["op"], cuda), None,
                                                              sc["H"], sc["W"], tile[0], tile[1], stat, False, False)
    return img, T, last, packed, fc, fw


def run_backward(cuda, sc, tile, packed, T, last, g):
    return fused.rasterize_backward(dev(sc["pid"], cuda), dev(sc["ranges"], cuda), packed, None, dev(T, cuda), dev(last, cuda), dev(g, cuda),
                                    None, None, torch.tensor([1.0], device=cuda), sc["H"], sc["W"], tile[0], tile[1], False)[:4]


@functools.lru_cache(maxsize=None)
def backward_inputs(cuda, case, tile, state):
    """(T, last, d_img, oracle gradients) for the backward.  state "oracle": the oracle's forward state; "kernel": the default
    forward kernel's own T and last, which the oracle's backward is then run on as well.  d_img is random and zero on the
    oracle's fragile pixels."""
    sc = scene(case, tile)
    _, oT, olast, _, _, frag = oracle_forward(case, tile)
    if state == "oracle":
        T, last = oT.astype(np.float32), olast
    else:
        _set(DEFAULTS)
        out = run_forward(cuda, sc, tile, False)
        T, last = out[1].cpu().numpy(), out[2].cpu().numpy()
    g = np.random.default_rng(7).normal(size=(sc["ndc"].shape[0], 3, sc["Hp"], sc["Wp"])).astype(np.float32)
    g[np.broadcast_to(frag[:, None], g.shape)] = 0.0
    ref = oracle.rasterize_backward(sc["pid"], sc["ranges"], f64(sc["ndc"]), f64(sc["inv"]), f64(sc["col"]), f64(sc["op"]), None,
                                    f64(T), last, f64(g), None, 1.0, sc["H"], sc["W"], tile[0], tile[1])
    return T, last, g, ref[:4]


# Far along a needle the power -(A dx^2 + 2 B dx dy + C dy^2)/2 is a small difference of large terms, and the kernels (like the
# reference's) evaluate it in fp32: G then carries a relative error of a few ulp of Q = (|A| dx^2 + 2 |B dx dy| + |C| dy^2)/2,
# which reaches ~1e-3 at 100:1 (an fp32 restatement of the kernels' power reproduces their image error there to the bit).  The
# needles' image, transmittance and conic, colour and opacity gradients are held to that conditioning, 2^-20 Q per pixel on
# top of 1e-4; the position gradient to the bar that does not depend on it.
COND = 2.0 ** -20


def _needle_fields(sc, i):
    """alpha, dx, dy and Q of needle i over the padded plane (fp64)."""
    y, x = np.mgrid[0:sc["Hp"], 0:sc["Wp"]].astype(np.float64)
    dx, dy = sc["px"][0, i] - x, sc["py"][0, i] - y
    A, B, C = sc["A"][0, i], sc["B"][0, i], sc["C"][0, i]
    Q = 0.5 * (abs(A) * dx * dx + 2 * np.abs(B * dx * dy) + abs(C) * dy * dy)
    return _splat_alpha(sc, [i])[0], dx, dy, Q


def needle_image_bound(sc):
    """Per-pixel bound [Hp, Wp] on the fp32 power's effect on the image and on T."""
    out = np.zeros((sc["Hp"], sc["Wp"]))
    for i in range(sc["ndc"].shape[2]):
        a, _, _, Q = _needle_fields(sc, i)
        out += COND * Q * np.where(a >= 0.5 / 256, a, 0.0)
    return out


def needle_gradient_bounds(sc, g):
    """Per-splat bounds, shaped as the four record gradients, for isolated splats alone on black (dL/dpower = alpha (c . g)):
    d_ndc: 1e-5 S with S the sum over the splat's pixels of the absolute per-pixel terms; the others: 2^-20 sum |term| Q."""
    N = sc["ndc"].shape[2]
    b_ndc, b_cov, b_col, b_op = np.zeros((1, 4, N)), np.zeros((1, 2, 2, N)), np.zeros((1, 3, N)), np.zeros((1, N))
    for i in range(N):
        a, dx, dy, Q = _needle_fields(sc, i)
        on = a >= 1.0 / 256
        cg = sum(float(sc["col"][0, c, i]) * g[0, c].astype(np.float64) for c in range(3))
        dpw = np.where(on, a * cg, 0.0)
        b_ndc[0, 0, i] = 1e-5 * 0.5 * sc["W"] * np.abs(dpw * (sc["A"][0, i] * dx + sc["B"][0, i] * dy)).sum()
        b_ndc[0, 1, i] = 1e-5 * 0.5 * sc["H"] * np.abs(dpw * (sc["B"][0, i] * dx + sc["C"][0, i] * dy)).sum()
        b_cov[0, 0, 0, i] = COND * (np.abs(0.5 * dx * dx * dpw) * Q).sum()
        b_cov[0, 0, 1, i] = b_cov[0, 1, 0, i] = COND * (np.abs(0.5 * dx * dy * dpw) * Q).sum()
        b_cov[0, 1, 1, i] = COND * (np.abs(0.5 * dy * dy * dpw) * Q).sum()
        for c in range(3):
            b_col[0, c, i] = COND * (np.abs(np.where(on, a, 0.0) * g[0, c]) * Q).sum()
        b_op[0, i] = COND * (np.abs(dpw / float(sc["op"][0, i])) * Q).sum()
    return b_ndc, b_cov, b_col, b_op


# ---------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wpb", WPB)
@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("fwd", list(FWD))
@pytest.mark.parametrize("case", list(CASES))
def test_forward_matches_fp64_oracle(cuda, switch, case, fwd, tile, wpb):
    """img, T and last against the fp64 oracle on the non-fragile pixels of the full padded planes (last exactly); every
    variant bit-identical to the default kernel at 4 warps per block, as staging form, warps per block, statistics and the
    pixel-pair body change no arithmetic; with statistics, the fragment counts and weights."""
    sc = scene(case, tile)
    oimg, oT, olast, ofc, ofw, frag = oracle_forward(case, tile)
    switch()
    ref = run_forward(cuda, sc, tile, False)
    sw, stat = FWD[fwd]
    switch(warps_per_block=wpb, **sw)
    img, T, last, _, fc, fw = run_forward(cuda, sc, tile, stat)
    for a, b, name in ((img, ref[0], "img"), (T, ref[1], "T"), (last, ref[2], "last")):
        assert torch.equal(a, b), name
    ok = ~frag
    assert frag.mean() < 0.02, frag.mean()
    last = last.cpu().numpy().astype(np.uint16)[:, 0]
    assert np.array_equal(last[ok], olast.astype(np.uint16)[:, 0][ok])
    m3 = np.broadcast_to(ok[:, None], oimg.shape)
    if case == "needles":
        bound = TOL + needle_image_bound(sc)
        assert (np.abs(img.cpu().numpy()[0] - oimg[0]) <= bound).all()
        assert (np.abs(T.cpu().numpy()[0, 0] - oT[0, 0]) <= bound).all()
    else:
        assert rel_err(img.cpu().numpy()[m3], oimg[m3]) < TOL
        assert rel_err(T.cpu().numpy()[:, 0][ok], oT[:, 0][ok]) < TOL
    if stat:
        fc, fw = fc.cpu().numpy(), fw.cpu().numpy()
        diff = np.abs(fc.astype(np.int64) - ofc)
        assert ofc.sum() > 0 and diff.sum() <= 2 * int(frag.sum()), (diff.sum(), frag.sum())
        same = diff == 0
        assert scaled_err(fw[same], ofw[same]) < 2e-4


def test_saturation_positions_are_as_built():
    """The saturation case does what it claims: on the oracle, every pixel of the k-th tile stops at list position k, and in
    the half-warp tiles the top half stops inside the stacks while the bottom half runs the whole list."""
    for tile in TILES:
        th, tw = tile
        sc = scene("saturation", tile)
        _, _, olast, _, _, _ = oracle_forward("saturation", tile)
        last = olast.astype(np.int64)[0, 0]
        gx = sc["Wp"] // tw
        for t, k in enumerate(SAT_K + HALF_K, start=1):
            ty, tx = divmod(t - 1, gx)
            blk = last[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw]
            if t <= len(SAT_K):
                assert (blk == k).all(), (tile, k)
            else:
                R = th // 2
                n = int(sc["ranges"][0, t + 1] - sc["ranges"][0, t])
                assert (blk[R:] == n).all(), (tile, k)
                assert (blk[:R] == (k - 1) * R + np.arange(R)[:, None] + 1).all(), (tile, k)


# ---------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("state", ["oracle", "kernel"])
@pytest.mark.parametrize("wpb", WPB)
@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("bwd", list(BWD))
@pytest.mark.parametrize("case", list(CASES))
def test_backward_matches_fp64_oracle(cuda, switch, case, bwd, tile, wpb, state):
    """The four record gradients against the fp64 oracle run on the same forward state (the oracle's, or the kernel's own):
    max-normalised error 1e-4, except the needles, held per splat: d_ndc to |err| <= 1e-5 S + 1e-4 |ref| with S the sum of the
    absolute per-pixel terms, the others to 1e-4 |ref| plus the fp32 power's conditioning (COND).  The deterministic backward
    twice, bit for bit."""
    sc = scene(case, tile)
    T, last, g, ref = backward_inputs(cuda, case, tile, state)
    switch()
    packed = run_forward(cuda, sc, tile, False)[3]
    switch(warps_per_block=wpb, **BWD[bwd])
    got = run_backward(cuda, sc, tile, packed, T, last, g)
    if bwd == "v2_det":
        again = run_backward(cuda, sc, tile, packed, T, last, g)
        for a, b, name in zip(got, again, GRAD_NAMES):
            assert torch.equal(a, b), name
    got = [a.cpu().numpy() for a in got]
    if case == "needles":
        for a, b, extra, name in zip(got, ref, needle_gradient_bounds(sc, g), GRAD_NAMES):
            err = np.abs(a.astype(np.float64) - b)
            assert (err <= TOL * np.abs(b) + extra).all(), (name, (err / np.maximum(TOL * np.abs(b) + extra, 1e-30)).max())
    else:
        for a, b, name in zip(got, ref, GRAD_NAMES):
            assert scaled_err(a, b) < TOL, (name, scaled_err(a, b))


@pytest.mark.parametrize("wpb", WPB)
@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
@pytest.mark.parametrize("bwd", list(BWD))
def test_views_in_one_launch_equal_single_view_launches(cuda, switch, bwd, tile, wpb):
    """V = 3 in one launch (grid.y = V, per-view cap and ntile + 2 strides) against three V = 1 launches: forward bit for bit,
    record gradients to fp32 atomic order (bit for bit in the deterministic mode); d_opacity is view 0's."""
    sc = scene("views", tile)
    T, last, g, _ = backward_inputs(cuda, "views", tile, "oracle")
    switch(warps_per_block=wpb, **BWD[bwd])
    img, Tk, lastk, packed, _, _ = run_forward(cuda, sc, tile, False)
    got = run_backward(cuda, sc, tile, packed, T, last, g)
    for b in range(3):
        one = dict(sc, ndc=sc["ndc"][b:b + 1], inv=sc["inv"][b:b + 1], col=sc["col"][b:b + 1], pid=sc["pid"][b:b + 1],
                   ranges=sc["ranges"][b:b + 1])
        i1, T1, l1, p1, _, _ = run_forward(cuda, one, tile, False)
        for a, c, name in ((img[b:b + 1], i1, "img"), (Tk[b:b + 1], T1, "T"), (lastk[b:b + 1], l1, "last"), (packed[b:b + 1], p1, "packed")):
            assert torch.equal(a, c), (b, name)
        g1 = run_backward(cuda, one, tile, p1, T[b:b + 1], last[b:b + 1], g[b:b + 1])
        pairs = [(got[k][b:b + 1], g1[k], GRAD_NAMES[k]) for k in range(3)] + ([(got[3], g1[3], "d_opacity")] if b == 0 else [])
        for a, c, name in pairs:
            if bwd == "v2_det":
                assert torch.equal(a, c), (b, name)
            else:
                assert scaled_err(a.cpu().numpy(), c.cpu().numpy()) < 1e-5, (b, name)


# ---------------------------------------------------------------------------------------------------
# range of the accumulators: one screen-sized splat
# ---------------------------------------------------------------------------------------------------

BIG = {"512x512": dict(hw=(512, 512), tile=(8, 16), centre=(420.3, 400.7), sd=(130.0, 110.0), o=0.5, c=0.5),
       "3840x2160": dict(hw=(2160, 3840), tile=(16, 16), centre=(3600.3, 1900.7), sd=(1100.0, 900.0), o=0.9, c=0.9)}


@functools.lru_cache(maxsize=None)
def big_case(size):
    """One anisotropic splat, rotated 45 degrees and placed towards a corner so that no record gradient cancels (at least 40 % of
    the sum of its terms' magnitudes survives), with d_img = 1 -> (scene, T, last, d_img, oracle gradients, raw moments)."""
    p = BIG[size]
    H, W = p["hw"]
    th, tw = p["tile"]
    gx, gy = -(-W // tw), -(-H // th)
    sc = assemble(H, W, p["tile"], np.array([[p["centre"][0]]]), np.array([[p["centre"][1]]]), np.array([[p["sd"][0]]]),
                  np.array([[p["sd"][1]]]), np.array([[math.radians(45.0)]]), np.array([p["o"]]), np.full((1, 3, 1), p["c"]),
                  [{t: [0] for t in range(1, gx * gy + 1)}])
    _, oT, olast, _, _, frag = oracle.rasterize_forward(sc["pid"], sc["ranges"], f64(sc["ndc"]), f64(sc["inv"]), f64(sc["col"]),
                                                        f64(sc["op"]), None, H, W, th, tw, fragile_eps=FRAGILE_EPS)
    g = np.ones((1, 3, sc["Hp"], sc["Wp"]), np.float32)
    g[np.broadcast_to(frag[:, None], g.shape)] = 0.0
    ref = oracle.rasterize_backward(sc["pid"], sc["ranges"], f64(sc["ndc"]), f64(sc["inv"]), f64(sc["col"]), f64(sc["op"]), None, oT,
                                    olast, f64(g), None, 1.0, H, W, th, tw)
    # raw moment of slot 2 (sum dx^2 dL/dpower), whole splat and per tile: alone on black, dL/dpower = alpha (c . g)
    a = _splat_alpha(sc, [0])[0]
    dx = sc["px"][0, 0] - np.arange(sc["Wp"], dtype=np.float64)[None, :]
    m2 = np.where(a >= 1.0 / 256, a * p["c"] * g[0].sum(0), 0.0) * dx * dx
    per_tile = m2.reshape(gy, th, gx, tw).sum((1, 3))
    return sc, oT.astype(np.float32), olast, g, ref[:4], (float(m2.sum()), float(per_tile.max()))


@pytest.mark.parametrize("bwd", list(BWD))
@pytest.mark.parametrize("size", list(BIG))
def test_screen_sized_splat_gradients(cuda, switch, size, bwd):
    """A splat covering the screen: its raw moments far exceed 2^27 (the whole splat at 512x512, a single tile's contribution
    at 3840x2160), past the range of a 64-bit accumulator at a 2^36 scale.  Every record gradient within 1e-4 relative of the
    fp64 oracle, per splat, in every backward variant; the deterministic one twice, bit for bit."""
    sc, T, last, g, ref, (m2, m2_tile) = big_case(size)
    tile = BIG[size]["tile"]
    if size == "512x512":
        assert m2 > 2.0 ** 28, m2
    else:
        assert m2_tile > 2.0 ** 27, m2_tile
    switch()
    packed = run_forward(cuda, sc, tile, False)[3]
    switch(**BWD[bwd])
    got = run_backward(cuda, sc, tile, packed, T, last, g)
    if bwd == "v2_det":
        again = run_backward(cuda, sc, tile, packed, T, last, g)
        for a, b, name in zip(got, again, GRAD_NAMES):
            assert torch.equal(a, b), name
    for a, b, name in zip(got, ref, GRAD_NAMES):
        a, b = a.cpu().numpy().astype(np.float64).reshape(-1), b.reshape(-1)
        live = np.abs(b) > 0                       # d_ndc's z and w rows are zero in both
        assert np.array_equal(np.abs(a) > 0, live), name
        err = np.abs(a[live] - b[live]) / np.abs(b[live])
        assert err.max() < TOL, (name, err.max(), a[live], b[live])
