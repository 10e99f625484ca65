"""fp64 statement of what tile binning promises, independent of how the kernels and the oracle walk the ellipse.

For one splat given as its raster record (px, py, A, B, C, o) -- Q(x, y) = A dx^2 + 2 B dx dy + C dy^2 with dx = px - x,
dy = py - y, exactly as the raster evaluates it, and alpha = o exp(-Q/2) >= 1/255 where Q <= t = 2 ln(255 o) -- on an H x W
image cut into th x tw tiles (tile id ty * gx + tx, 0-based):

  must  the tiles holding a pixel centre (x, y), x < W and y < H, with Q <= t (1 - delta) - delta: every pixel where the
        raster blends the splat, by a margin delta;
  may   the tiles whose rectangle [tx tw, (tx + 1) tw) x [ty th, (ty + 1) th) meets the widened ellipse
        Q <= t (1 + delta) + delta: the continuous footprint the ellipse/tile walk works with, which is more than the pixel
        centres.

Binning is right when must <= listed <= may for every splat.  delta absorbs the fp32 arithmetic of the walk (t rounded once to
fp32, the bounding box and the line intersections each a few single-rounded ops): relative errors of a few 1e-7 in Q, far
inside delta = 1e-4 at the image sizes of the tests.  It does not have to absorb a difference of centres: the walk forms
px = (ndc 0.5 + 0.5) W - 0.5 and the record px = ((ndc + 1) 0.5) W - 0.5, and since halving is exact in binary floating
point, fl(0.5 ndc + 0.5) = 0.5 fl(ndc + 1) and the two centres are the same fp32 number.

Work per splat is vectorised over its own pixel / tile bounding box, not the whole image."""
import math

import numpy as np

DELTA = 1e-4


def threshold(o):
    """t = 2 ln(255 o) in fp64 (the iso-ellipse of alpha = 1/255)."""
    return 2.0 * math.log(255.0 * float(o))


def _extent(A, B, C, t):
    """Half-widths (ex, ey) of the ellipse Q <= t, or None when it is empty or the conic is not positive definite."""
    det = A * C - B * B
    if not (A > 0 and C > 0 and det > 0 and t > 0):
        return None
    return math.sqrt(t * C / det), math.sqrt(t * A / det)


def must_tiles(rec, hw, tile, delta=DELTA, t_scale=None):
    """Tile ids (sorted int64) holding a pixel centre with Q <= t (1 - delta) - delta.  t_scale: use t_scale instead of
    t (1 - delta) - delta (e.g. t itself for the wasted-pair count)."""
    px, py, A, B, C, o = (float(v) for v in rec[:6])
    H, W = hw
    th, tw = tile
    if o <= 0:
        return np.zeros(0, np.int64)
    t = threshold(o)
    tm = t * (1 - delta) - delta if t_scale is None else t_scale
    e = _extent(A, B, C, tm)
    if e is None:
        return np.zeros(0, np.int64)
    ex, ey = e
    x0, x1 = max(0, math.ceil(px - ex)), min(W - 1, math.floor(px + ex))
    y0, y1 = max(0, math.ceil(py - ey)), min(H - 1, math.floor(py + ey))
    if x0 > x1 or y0 > y1:
        return np.zeros(0, np.int64)
    xs = np.arange(x0, x1 + 1, dtype=np.float64)
    ys = np.arange(y0, y1 + 1, dtype=np.float64)
    dx = px - xs[None, :]
    dy = py - ys[:, None]
    inside = A * dx * dx + 2 * B * dx * dy + C * dy * dy <= tm
    if not inside.any():
        return np.zeros(0, np.int64)
    gx = -(-W // tw)
    yy, xx = np.nonzero(inside)
    ids = (ys[yy].astype(np.int64) // th) * gx + xs[xx].astype(np.int64) // tw
    return np.unique(ids)


def _rect_min_q(A, B, C, X0, X1, Y0, Y1):
    """min of Q(X, Y) = A X^2 + 2 B X Y + C Y^2 over the rectangles [X0, X1] x [Y0, Y1] (arrays, X/Y relative to the
    centre).  Q is convex: the minimum is 0 when the centre is inside, else on an edge at the clamped 1D minimiser."""
    q = lambda X, Y: A * X * X + 2 * B * X * Y + C * Y * Y
    best = np.full(np.broadcast(X0, Y0).shape, np.inf)
    for X in (X0, X1):
        best = np.minimum(best, q(X, np.clip(-B * X / C, Y0, Y1)))
    for Y in (Y0, Y1):
        best = np.minimum(best, q(np.clip(-B * Y / A, X0, X1), Y))
    inside = (X0 <= 0) & (0 <= X1) & (Y0 <= 0) & (0 <= Y1)
    return np.where(inside, 0.0, best)


def may_tiles(rec, hw, tile, delta=DELTA):
    """Tile ids (sorted int64) whose rectangle meets the ellipse Q <= t (1 + delta) + delta.  The rectangle's far edges
    belong to the next tile; the infimum of Q over the half-open rectangle is its minimum over the closed one, which is what
    is tested."""
    px, py, A, B, C, o = (float(v) for v in rec[:6])
    H, W = hw
    th, tw = tile
    gx, gy = -(-W // tw), -(-H // th)
    if o <= 0:
        return np.zeros(0, np.int64)
    tw_ = threshold(o) * (1 + delta) + delta
    e = _extent(A, B, C, tw_)
    if e is None:
        return np.zeros(0, np.int64)
    ex, ey = e
    u0, u1 = max(0, math.floor((px - ex) / tw)), min(gx - 1, math.floor((px + ex) / tw))
    v0, v1 = max(0, math.floor((py - ey) / th)), min(gy - 1, math.floor((py + ey) / th))
    if u0 > u1 or v0 > v1:
        return np.zeros(0, np.int64)
    us = np.arange(u0, u1 + 1, dtype=np.int64)[None, :]
    vs = np.arange(v0, v1 + 1, dtype=np.int64)[:, None]
    m = _rect_min_q(A, B, C, us * tw - px, (us + 1) * tw - px, vs * th - py, (vs + 1) * th - py)
    vv, uu = np.nonzero(m <= tw_)
    return np.unique(vs[vv, 0] * gx + us[0, uu])


def check_cover(recs, listed, hw, tile, delta=DELTA):
    """recs f64[N, >=6] (px, py, A, B, C, o), listed: per splat the tile ids it was given (any int sequence).
    -> dict(missing=[(i, tiles)], extra=[(i, tiles)], n_must, n_wasted): splats whose list lacks a must tile or holds a tile
    outside may, the number of must tiles, and the number of listed pairs with no pixel centre at Q <= t (wasted work; reported,
    not a failure)."""
    missing, extra, n_must, n_wasted = [], [], 0, 0
    for i in range(len(recs)):
        got = np.unique(np.asarray(listed[i], np.int64))
        must = must_tiles(recs[i], hw, tile, delta)
        n_must += must.size
        lost = np.setdiff1d(must, got)
        if lost.size:
            missing.append((i, lost.tolist()))
        if got.size:
            over = np.setdiff1d(got, may_tiles(recs[i], hw, tile, delta))
            if over.size:
                extra.append((i, over.tolist()))
            o = float(recs[i][5])
            hit = must_tiles(recs[i], hw, tile, t_scale=threshold(o)) if o > 0 else np.zeros(0, np.int64)
            n_wasted += np.setdiff1d(got, hit).size
    return dict(missing=missing, extra=extra, n_must=n_must, n_wasted=n_wasted)


def lists_by_splat(keys, vals, n):
    """Tile-sorted pair table (keys = tile id + 1, 0 = unused slot; vals = splat) -> per splat the list of 0-based tile ids,
    duplicates kept."""
    out = [[] for _ in range(n)]
    for k, i in zip(np.asarray(keys).tolist(), np.asarray(vals).tolist()):
        if k > 0:
            out[i].append(k - 1)
    return out


# ---------------------------------------------------------------------------------------------------
# constructed 2D cases: records placed on the conditions where a tile rectangle can lose a tile
# ---------------------------------------------------------------------------------------------------

OFFSETS = (0.03, 0.1, 0.25, 0.5, 0.75, 0.9, 0.97)      # how far (px) the ellipse reaches past the tile boundary


def conic(s1, s2, theta):
    """(A, B, C) of a Gaussian with standard deviations s1 along angle theta and s2 across it."""
    c, s = math.cos(theta), math.sin(theta)
    a1, a2 = 1.0 / (s1 * s1), 1.0 / (s2 * s2)
    return c * c * a1 + s * s * a2, c * s * (a1 - a2), s * s * a1 + c * c * a2


def grazing_cases(hw, tile):
    """Splats whose ellipse ends a fraction f in OFFSETS past a tile boundary kT (bbox_max in [kT, kT + 1)) or starts that
    far before one (bbox_min in (kT - 1, kT]), on both axes, for ellipses wider than tall and taller than wide (the walk slices
    by rows in one case and by columns in the other), both signs of B and three sizes down to the low-pass floor.  The chord
    of the ellipse on the boundary's pixel column (row) is centred on a pixel row (column), so the pixel centre on the boundary
    lies inside the ellipse.  -> list of dict(rec=(px, py, A, B, C, o), axis, side, k, T, f) in fp64."""
    H, W = hw
    th, tw = tile
    out = []
    o = 0.99
    t = threshold(o)
    for axis in (0, 1):
        T, size, osize = (tw, W, H) if axis == 0 else (th, H, W)
        nk = -(-size // T)
        for side in ("max", "min"):
            for shape in ((4.0, 1.5), (1.5, 4.0), (0.6, 0.6), (12.0, 3.0), (3.0, 12.0)):
                for sgn in (1.0, -1.0):
                    for j, f in enumerate(OFFSETS):
                        theta = sgn * (0.35 + 0.1 * j)
                        A, B, C = conic(shape[0], shape[1], theta) if axis == 0 else conic(shape[1], shape[0], theta)
                        ex, ey = _extent(A, B, C, t)
                        e, across = (ex, B / C) if axis == 0 else (ey, B / A)
                        # boundaries kT (k >= 1) that keep the centre on the image
                        ks = [k for k in range(1, nk) if 0 <= (k * T + f - e if side == "max" else k * T - f + e) < size]
                        if not ks:
                            continue
                        k = ks[len(out) % len(ks)]
                        edge = k * T
                        if side == "max":
                            c_u = edge + f - e                # bbox_max = edge + f
                        else:
                            c_u = edge - f + e                # bbox_min = edge - f
                        d_u = edge - c_u                      # boundary pixel line relative to the centre, |d_u| < e
                        # the chord on the boundary pixel line is centred on pixel `row`, chosen so the centre is on the image
                        row = int(np.clip(round(osize * (0.2 + 0.6 * ((len(out) * 0.618) % 1.0)) - across * d_u), 0, osize - 1))
                        c_v = row + across * d_u
                        px, py = (c_u, c_v) if axis == 0 else (c_v, c_u)
                        out.append(dict(rec=(px, py, A, B, C, o), axis=axis, side=side, k=k, T=T, f=f,
                                        value=edge + f if side == "max" else edge - f))
    return out


def floor_cases(hw, tile):
    """Sub-pixel splats at the 0.3 px^2 low-pass floor (sigma = 0.548 px) with o = 0.99 and 0.999, centred a sweep of
    sub-pixel distances either side of tile rows and columns; and splats with opacity just above 1/255, where t is tiny,
    centred within a hundredth of a pixel of a pixel centre next to a tile boundary."""
    H, W = hw
    th, tw = tile
    out = []
    s = math.sqrt(0.3)
    for o in (0.99, 0.999):
        for d in (-1.6, -1.2, -0.83, -0.5, -0.17, 0.17, 0.5, 0.83, 1.2, 1.6):
            kx, ky = 1 + len(out) % max(1, W // tw - 1), 1 + len(out) % max(1, H // th - 1)
            out.append((kx * tw + d, ky * th + 0.5 + 0.13 * d, *conic(s, s, 0.0), o))
            out.append((kx * tw + 0.5 + 0.11 * d, ky * th + d, *conic(s, s, 0.0), o))
            out.append((kx * tw + d, ky * th + d, *conic(s * 1.4, s, 0.6), o))
    for o in (1.0 / 255 * 1.0005, 1.0 / 255 * 1.01, 1.0 / 255 * 1.2):
        for s1, s2, th_ in ((s, s, 0.0), (5.0, 1.0, 0.7), (20.0, 0.7, -0.3)):
            for dx, dy in ((0.0, 0.0), (-0.004, 0.006), (0.008, -0.002)):
                kx, ky = 1 + len(out) % max(1, W // tw - 1), 1 + len(out) % max(1, H // th - 1)
                for bx, by in ((kx * tw, ky * th), (kx * tw - 1, ky * th - 1)):
                    out.append((bx + dx, by + dy, *conic(s1, s2, th_), o))
    return out


def needle_cases(hw, tile, n_angles=12):
    """Needles up to 100:1 (sigma 40 px by 0.4 px, 20 by 0.5, 9 by 0.3) at several angles, 0 and 90 degrees among them,
    centred anywhere, crossing many tiles."""
    H, W = hw
    out = []
    for j in range(n_angles):
        ang = math.pi * j / n_angles + (0.0 if j % 3 == 0 else 0.013 * j)
        for k, (s1, s2) in enumerate(((40.0, 0.4), (20.0, 0.5), (9.0, 0.3))):
            px = (0.17 + 0.61 * ((j * 3 + k) * 0.618 % 1.0)) * W + 0.37 * k
            py = (0.15 + 0.67 * ((j * 5 + k) * 0.382 % 1.0)) * H - 0.29 * k
            out.append((px, py, *conic(s1, s2, ang), 0.95 - 0.3 * k))
    return out


def offscreen_cases(hw, tile):
    """Centres outside the image (within ndc +-1.3) whose ellipse reaches less than a pixel into it, past each of the four
    edges, at a sweep of reaches; the chord on the first (last) pixel line is centred on a pixel.  -> list of
    dict(rec, axis, side, value): the ellipse's extent on `axis` ends (side "max") or starts ("min") at `value`."""
    H, W = hw
    out = []
    o = 0.9
    t = threshold(o)
    for edge in ("left", "right", "top", "bottom"):
        for j, f in enumerate(OFFSETS):
            theta = 0.3 * (j - 3)
            axis = 0 if edge in ("left", "right") else 1
            size = W if axis == 0 else H
            sig = 0.1 * size / math.sqrt(t) + 0.5        # reaches in from beyond the edge, centre within ndc +-1.3
            A, B, C = conic(sig, 0.5 * sig, theta) if axis == 0 else conic(0.5 * sig, sig, theta)
            ex, ey = _extent(A, B, C, t)
            e, across = (ex, B / C) if axis == 0 else (ey, B / A)
            if edge in ("left", "top"):
                c_u = f - e                  # bbox_max = f: pixel line 0 is reached by f
            else:
                c_u = size - 1 - f + e       # bbox_min = size - 1 - f
            d_u = (0 if edge in ("left", "top") else size - 1) - c_u
            other = (H if axis == 0 else W)
            row = 3 + (j * 5) % max(1, other - 6)
            c_v = row + across * d_u
            px, py = (c_u, c_v) if axis == 0 else (c_v, c_u)
            side = "max" if edge in ("left", "top") else "min"
            out.append(dict(rec=(px, py, A, B, C, o), axis=axis, side=side, value=f if side == "max" else size - 1 - f))
    return out


def big_cases(hw, tile, n=6):
    """Splats covering hundreds to thousands of tiles (more than one 512-pair emit window each)."""
    H, W = hw
    out = []
    for j in range(n):
        s1 = 0.35 * max(H, W) * (0.5 + 0.1 * j)
        out.append((W * (0.3 + 0.08 * j), H * (0.6 - 0.05 * j), *conic(s1, 0.4 * s1, 0.4 * j), 0.6))
    return out


def random_cases(seed, n=3000, hw=(128, 160)):
    """n random splats: sigma 0.3 to 60 px, anisotropy up to 60:1, any angle, opacity from just above 1/255 to 0.99 (a third of
    them below 0.05), centres anywhere in ndc +-1.3."""
    H, W = hw
    rng = np.random.default_rng(seed)
    s1 = np.exp(rng.uniform(np.log(0.3), np.log(60.0), n))
    s2 = s1 / np.exp(rng.uniform(0, np.log(60.0), n))
    th = rng.uniform(0, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    S00 = c * c * s1 ** 2 + s * s * s2 ** 2 + 0.3
    S11 = s * s * s1 ** 2 + c * c * s2 ** 2 + 0.3
    S01 = c * s * (s1 ** 2 - s2 ** 2)
    det = S00 * S11 - S01 ** 2
    o = rng.uniform(1 / 255 * 1.0001, 0.99, n)
    o[::3] = np.exp(rng.uniform(np.log(1 / 255 * 1.0001), np.log(0.05), len(o[::3])))
    px = (rng.uniform(-1.3, 1.3, n) + 1) * 0.5 * W - 0.5
    py = (rng.uniform(-1.3, 1.3, n) + 1) * 0.5 * H - 0.5
    return np.stack([px, py, S11 / det, -S01 / det, S00 / det, o], 1)


def inputs_2d(recs, hw, depth=None):
    """fp64 records (px, py, A, B, C, o) -> the binning inputs in fp32 (ndc [1,4,N], view z [1,N], inv_cov2d [1,2,2,N],
    opacity [1,N]) and the records the raster sees (fp32 values, as fp64 [N, 6]).  depth: view z per splat (default:
    increasing with the index, so that depth order is record order)."""
    H, W = hw
    r = np.asarray(recs, np.float64)
    N = r.shape[0]
    f = np.float32
    nx = ((r[:, 0] + 0.5) / W * 2 - 1).astype(f)
    ny = ((r[:, 1] + 0.5) / H * 2 - 1).astype(f)
    ndc = np.zeros((1, 4, N), f)
    ndc[0, 0], ndc[0, 1], ndc[0, 2], ndc[0, 3] = nx, ny, 0.5, 1.0
    A, B, C, o = (r[:, k].astype(f) for k in (2, 3, 4, 5))
    inv = np.zeros((1, 2, 2, N), f)
    inv[0, 0, 0], inv[0, 0, 1], inv[0, 1, 0], inv[0, 1, 1] = A, B, B, C
    vz = (np.asarray(depth, f) if depth is not None else f(1.0) + np.arange(N, dtype=f) * f(1e-3)).reshape(1, N)
    px = ((nx + f(1)) * f(0.5)) * f(W) - f(0.5)
    py = ((ny + f(1)) * f(0.5)) * f(H) - f(0.5)
    rec32 = np.stack([px, py, A, B, C, o], 1).astype(np.float64)
    return dict(ndc=ndc, vz=vz, inv=inv, op=o.reshape(1, N), rec=rec32, nx=nx, ny=ny)


def constructed_cases(hw, tile):
    """Every constructed case -> list of dict(rec, kind, and for the grazing and off-screen cases axis, side, value)."""
    out = [dict(c, kind="grazing") for c in grazing_cases(hw, tile)]
    out += [dict(rec=r, kind="floor") for r in floor_cases(hw, tile)]
    out += [dict(rec=r, kind="needle") for r in needle_cases(hw, tile)]
    out += [dict(c, kind="offscreen") for c in offscreen_cases(hw, tile)]
    out += [dict(rec=r, kind="big") for r in big_cases(hw, tile)]
    return out
