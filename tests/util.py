"""Shared helpers for the parity tests: small seeded scenes pushed through the CPU oracle, and the scaffolding the GPU tests
share."""
import math

import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, colmap, fused, scene
from tests import camera_oracle as co

PARAM_KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")
ZN, ZF = 0.01, 5000.0                                   # the near and far planes of the learnable-camera tests


@pytest.fixture
def deterministic():
    """Bit-identity checks need the raster backward's deterministic accumulation (lgs_set_deterministic): its default fp32 atomics
    make the record gradients, and so every gradient after them, reproducible only to rounding.  A test module imports this
    fixture by name."""
    _lib.call("lgs_set_deterministic", 1)
    yield
    _lib.call("lgs_set_deterministic", 0)


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


def f64_arrays(d):
    """d with its float32 arrays as float64."""
    return {k: (v.astype(np.float64) if isinstance(v, np.ndarray) and v.dtype == np.float32 else v) for k, v in d.items()}


def tiny_scene(seed=3, n=48, hw=(32, 32), chunk=16, deg=2, log_scale_range=(0.03, 0.2)):
    """An fp64 scene small enough for central differences.  The default scales go down to a third of a pixel, so that the
    antialiasing factor ranges widely."""
    p = scene.make_scene(n, sh_degree=deg, chunk=chunk, log_scale_range=log_scale_range, seed=seed)
    cam = f64_arrays(scene.make_camera(1, 8, hw[1], hw[0]))
    P = {k: p[k].astype(np.float64) for k in PARAM_KEYS}
    P["opacity"] = np.clip(P["opacity"], -1, 1.5)       # keep away from the 255/256 clamp
    P["sh_0"] *= 0.3; P["sh_rest"] *= 0.3               # keep colours inside (0,1): min(c,1) is not differentiable
    aabb = (p["cluster_origin"].astype(np.float64), p["cluster_extend"].astype(np.float64))
    return P, aabb, cam


def single_splat(std_px, hw=(64, 64), opacity=0.8, chunk=16, dt=np.float64):
    """One splat on the optical axis, isotropic with the given standard deviation in pixels before the filter, plus chunk - 1
    invisible companions (opacity far below 1/255).  -> (params, aabb, cam)."""
    H, W = hw
    recp = 1.0 / math.tan(math.radians(30.0))
    view, proj, _, planes = co.create_viewproj_forward(np.array([[1.0, 0, 0, 0, 0, 0, 0]]), np.array([recp]), H, W, 0.01, 100.0)
    z = 5.0
    fx = recp * W * 0.5
    s = std_px * z / fx
    n = chunk
    xyz = np.zeros((3, 1, n)); xyz[2] = z
    P = dict(xyz=xyz, scale=np.full((3, 1, n), math.log(s)), rot=np.tile(np.array([1.0, 0, 0, 0])[:, None, None], (1, 1, n)),
             sh_0=np.full((1, 3, 1, n), 0.5), sh_rest=np.zeros((0, 3, 1, n)), opacity=np.full((1, 1, n), -30.0))
    P["opacity"][0, 0, 0] = math.log(opacity / (1 - opacity))
    P = {k: v.astype(dt) for k, v in P.items()}
    aabb = (np.array([[0.0], [0.0], [z]], dt), np.full((3, 1), 10 * s, dt))
    cam = dict(view=view.astype(dt), proj=proj.astype(dt), frustumplane=planes.astype(dt))
    return P, aabb, cam


def lattice_cameras(n, hw, radius=3.0, fov=60.0):
    """(views [n,4,4], projs [n,4,4], hws [n,2]) of n cameras of scene.make_camera's lattice, all of size hw."""
    cams = [scene.make_camera(i, n, hw[1], hw[0], radius=radius, fov_x_deg=fov) for i in range(n)]
    return np.concatenate([c["view"] for c in cams]), np.concatenate([c["proj"] for c in cams]), np.array([hw] * n, np.int32)


def view_params(cam):
    """(qw qx qy qz tx ty tz) of a row-vector view matrix [1,4,4]: its 3x3 block is the transpose of the COLMAP rotation."""
    V = np.asarray(cam["view"], np.float64).reshape(4, 4)
    return np.concatenate([colmap.rotmat_to_qvec(V[:3, :3].T), V[3, :3]])


def rot_err_deg(a, b):
    """Angle in degrees between the rotations of two view_params."""
    qa, qb = a[:4] / np.linalg.norm(a[:4]), b[:4] / np.linalg.norm(b[:4])
    return float(np.degrees(2 * np.arccos(min(1.0, abs(float(np.dot(qa, qb)))))))


def to_torch(params, aabb, cam, dev, grad=True):
    """(params, aabb, camera) on the device -> (P dict, [origin, extent], C dict)."""
    P = {k: torch.from_numpy(params[k]).to(dev).requires_grad_(grad) for k in PARAM_KEYS}
    A = [torch.from_numpy(a).to(dev) for a in aabb]
    C = {k: torch.from_numpy(v).to(dev) for k, v in cam.items()}
    return P, A, C


def oracle_case(n, hw, tile, sh_degree, seed, view=0, scale_range=(0.02, 0.08)):
    """A seeded scene and the oracle's forward and backward for a random loss weight that is zero on the oracle's fragile pixels
    -> (params, aabb, cam, w, fragile, ref)."""
    params, aabb, cam = small_scene(n=n, hw=hw, tile=tile, sh_degree=3, seed=seed, view=view, log_scale_range=scale_range)
    rng = np.random.default_rng(seed + 100)
    w = rng.normal(size=(1, 3, hw[0], hw[1])).astype(np.float32)
    # first pass to find fragile pixels, then zero the loss weight there
    o0 = oracle.render_forward_backward(params, aabb, cam, hw, tile, sh_degree, lambda img: w)
    frag = o0["fragile"][:, : hw[0], : hw[1]]
    w = w * (~frag)[:, None]
    ref = oracle.render_forward_backward(params, aabb, cam, hw, tile, sh_degree, lambda img: w)
    return params, aabb, cam, w, frag, ref


def as_f64(out):
    """A restatement's dict with the inputs of the camera gradient (intermediates, record gradients, G_aa) in fp64, so that the
    camera gradient is summed in fp64."""
    return dict(out, inter={k: v.astype(np.float64) for k, v in out["inter"].items()},
                **{k: out[k].astype(np.float64) for k in ("d_ndc", "d_cov", "G_aa") if k in out})


def restatement_mask(st, o0, hw, tile):
    """Pixels [V,H,W] where a fused render (its state st) may differ from the restatement's o0: o0's fragile pixels and the tiles
    whose lists differ, at most two.  The contributor counts agree on every other pixel."""
    bad, _ = differing_tiles(st.ranges.cpu().numpy(), st.sorted_pid.cpu().numpy(), o0["ranges"], o0["sorted_pid"])
    assert len(bad) <= 2
    frag = o0["fragile"][:, :hw[0], :hw[1]].copy()
    gx = -(-hw[1] // tile[1])
    for t in bad:
        ty, tx = divmod(int(t), gx)
        frag[:, ty * tile[0]:(ty + 1) * tile[0], tx * tile[1]:(tx + 1) * tile[1]] = True
    last = st.last.cpu().numpy()[:, 0, :hw[0], :hw[1]]
    assert np.array_equal(last[~frag], o0["last"][:, 0, :hw[0], :hw[1]][~frag])
    return frag


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


def axis_camera(hw, t=(0.0, 0.0, 0.0)):
    """A 60-degree camera with identity rotation and view-space position = world position + t (fp32 numpy dict).  With t = 0 the
    view-space z of a point is its world z exactly."""
    H, W = hw
    recp = 1.0 / math.tan(math.radians(30.0))
    view, proj, _, planes = co.create_viewproj_forward(np.array([[1.0, 0, 0, 0, *t]]), np.array([recp]), H, W, 0.01, 100.0)
    return dict(view=view.astype(np.float32), proj=proj.astype(np.float32), frustumplane=planes.astype(np.float32))


def screen_affine(cam, hw, Z):
    """(ax, bx, ay, by) with px = ax X + bx, py = ay Y + by at depth Z (fp64 from the camera matrices)."""
    H, W = hw
    M = cam["view"][0].astype(np.float64) @ cam["proj"][0].astype(np.float64)

    def pix(X, Y):
        h = np.stack([X, Y, Z, np.ones_like(Z)], -1) @ M
        return (h[..., 0] / h[..., 3] + 1) * 0.5 * W - 0.5, (h[..., 1] / h[..., 3] + 1) * 0.5 * H - 0.5
    x0, y0 = pix(np.zeros_like(Z), np.zeros_like(Z))
    x1, y1 = pix(np.ones_like(Z), np.ones_like(Z))
    return x1 - x0, x0, y1 - y0, y0


def oracle_render_lists(packed, pid, ranges, hw, tile):
    """fp64 oracle raster of fused records packed f32[N,12] (px, py, A, B, C, o, r, g, b, ...) over the given tile lists
    (sorted_pid i32[1,L], ranges i32[1,tiles+2]) -> (img [3,Hp,Wp], T [Hp,Wp], fragile [Hp,Wp]), all f64 / bool."""
    H, W = hw
    th, tw = tile
    packed = np.asarray(packed, np.float64)
    N = packed.shape[0]
    ndc = np.zeros((1, 4, N))
    ndc[0, 0] = (packed[:, 0] + 0.5) / W * 2 - 1                   # the oracle maps ndc back to exactly the record's px, py
    ndc[0, 1] = (packed[:, 1] + 0.5) / H * 2 - 1
    inv = np.zeros((1, 2, 2, N))
    inv[0, 0, 0], inv[0, 0, 1], inv[0, 1, 0], inv[0, 1, 1] = packed[:, 2], packed[:, 3], packed[:, 3], packed[:, 4]
    col = np.ascontiguousarray(packed[:, 6:9].T[None])
    op = packed[:, 5][None]
    pid = np.ascontiguousarray(pid, np.int32).reshape(1, -1)
    if pid.shape[1] == 0:
        pid = np.zeros((1, 1), np.int32)
    oimg, oT, _, _, _, frag = oracle.rasterize_forward(pid, np.asarray(ranges, np.int32), ndc, inv, col, op, None, H, W, th, tw,
                                                       fragile_eps=2e-6)
    return oimg[0], oT[0, 0], frag[0]


def rel_err(a, b):
    """max |a-b| / max(1, |b|) -- the Tier-1 metric of SURVEY 8c."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)))) if a.size else 0.0


def scaled_err(a, b):
    """max |a-b| / max|b| -- for gradients whose magnitude is far from 1."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    m = np.max(np.abs(b)) if b.size else 0.0
    return float(np.max(np.abs(a - b)) / max(m, 1e-30)) if a.size else 0.0


def raster_case(cuda, proj, tile, staging):
    """The fused raster forward and backward against the oracle on the oracle's lists of a projected scene proj (the GPU ops
    tests' fixture), with the staging variant chosen; the backward is fed the oracle's forward state."""
    _lib.call("lgs_set_staging", 1 if staging == "bulk" else 0)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ranges, sorted_pid, _, _ = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
    oimg, oT, olast, _, _, fragile = oracle.rasterize_forward(sorted_pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None,
                                                               hw[0], hw[1], th, tw, fragile_eps=2e-6)
    out = fused.rasterize_forward(dev(sorted_pid), dev(ranges), dev(o["ndc"]), dev(o["inv_cov2d"]), dev(o["color"]), dev(o["opacity"]), None,
                                  hw[0], hw[1], th, tw, False, False, False)
    img, Tr, _, last, packed, _, _ = out
    ok = ~fragile
    assert fragile.mean() < 0.02
    assert np.array_equal(last.cpu().numpy()[:, 0][ok], olast[:, 0][ok])
    m3 = np.broadcast_to(ok[:, None], oimg.shape)
    assert rel_err(img.cpu().numpy()[m3], oimg[m3]) < 1e-4
    assert rel_err(Tr.cpu().numpy()[:, 0][ok], oT[:, 0][ok]) < 1e-4
    # backward, fed with the ORACLE's forward state so that only the backward kernel is under test
    rng = np.random.default_rng(1)
    g = rng.normal(size=oimg.shape).astype(np.float32)
    g[np.broadcast_to(fragile[:, None], g.shape)] = 0.0
    gmax = np.abs(g).max()
    ref = oracle.rasterize_backward(sorted_pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, oT, olast,
                                    g / gmax, None, gmax, hw[0], hw[1], th, tw)
    got = fused.rasterize_backward(dev(sorted_pid), dev(ranges), packed, None, dev(oT), dev(olast), dev(g / gmax), None, None,
                                   torch.tensor([gmax], device=cuda), hw[0], hw[1], th, tw, False)
    for a, b, name in zip(got[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
        assert scaled_err(a.cpu().numpy(), b) < 1e-4, (name, scaled_err(a.cpu().numpy(), b))
