"""Shared helpers for the parity tests: small seeded scenes pushed through the CPU oracle."""
import numpy as np

import oracle
from litegs_b200 import scene

PARAM_KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")


def small_scene(n=2000, hw=(96, 128), tile=(16, 16), sh_degree=3, seed=0, log_scale_range=(0.02, 0.08), view=0, n_views=8,
                chunk=128):
    p = scene.make_scene(n, sh_degree=sh_degree, chunk=chunk, seed=seed, log_scale_range=log_scale_range)
    cam = scene.make_camera(view, n_views, hw[1], hw[0])
    params = {k: p[k] for k in PARAM_KEYS}
    return params, (p["cluster_origin"], p["cluster_extend"]), cam


def oracle_projected(params, aabb, cam, hw, sh_degree):
    """Oracle outputs up to the inputs of binning/raster: activated+projected per-Gaussian tensors (numpy)."""
    vis, nvis, ids = oracle.frustum_culling_aabb(aabb[0], aabb[1], cam["frustumplane"])
    act = oracle.cull_compact_activate(sh_degree, ids, nvis, cam["view"], params["xyz"], params["scale"], params["rot"],
                                       params["sh_0"], params["sh_rest"], params["opacity"])
    xyz, scale, rot, color, opacity = [a.reshape(*a.shape[:-2], -1) for a in act]
    inter = oracle.project(xyz, scale, rot, cam["view"], cam["proj"], hw)
    return dict(ids=ids, nvis=nvis, vis=vis, act=act, xyz=xyz, scale=scale, rot=rot, color=color, opacity=opacity, **inter)


def tile_segments(ranges, n):
    """[start, end) of every tile's run in a tile-sorted pair list of length n, from its range table i32[1, tiles+2] (entry
    t + 1 belongs to the 0-based tile t); start = end = -1 for a tile the table leaves at -1."""
    r = np.asarray(ranges)[0].astype(np.int64)
    ntile = r.shape[0] - 2
    start = r[1:ntile + 1].copy()
    s2 = np.where(r[1:ntile + 2] >= 0, r[1:ntile + 2], np.iinfo(np.int64).max)
    nxt = np.minimum.accumulate(s2[::-1])[::-1]           # end of tile t = next populated start after t
    end = np.where(start >= 0, np.minimum(nxt[1:], n), -1)
    return start, end


def differing_tiles(ranges_a, pid_a, ranges_b, pid_b):
    """Tiles (0-based) whose depth-ordered splat lists differ between two binnings, and the number of differing pairs."""
    ntile = ranges_a.shape[1] - 2
    sa, ea = tile_segments(ranges_a, pid_a.shape[1]); sb, eb = tile_segments(ranges_b, pid_b.shape[1])
    bad, npairs = [], 0
    for t in range(ntile):
        la = pid_a[0, sa[t]:ea[t]] if sa[t] >= 0 else pid_a[0, :0]
        lb = pid_b[0, sb[t]:eb[t]] if sb[t] >= 0 else pid_b[0, :0]
        if la.shape != lb.shape or not np.array_equal(la, lb):
            bad.append(t)
            npairs += len(set(la.tolist()) ^ set(lb.tolist()))
    return np.array(bad, np.int64), npairs


def rel_err(a, b):
    """max |a-b| / max(1, |b|) -- the Tier-1 metric of SURVEY 8c."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)))) if a.size else 0.0


def scaled_err(a, b):
    """max |a-b| / max|b| -- for gradients whose magnitude is far from 1."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    m = np.max(np.abs(b)) if b.size else 0.0
    return float(np.max(np.abs(a - b)) / max(m, 1e-30)) if a.size else 0.0
