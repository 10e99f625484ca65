"""Mesh extraction on the CPU: the numpy restatement (tests/mesh_oracle.py) of TSDF integration and marching tetrahedra on analytic
volumes -- closed, consistently oriented meshes of the right topology and volume, open sheets, empty volumes, the integration
rules and the pixel round trip with lgs_depth_normal's ray -- and the PLY mesh round trip."""
import math

import numpy as np
import pytest

from litegs_b200 import ply, scene
from tests import mesh_oracle as mo

F32 = np.float32


def analytic_volume(sdf, n, h, trunc):
    """tsdf = clip(sdf / trunc, -1, 1) of an analytic signed distance sampled on an n^3 lattice centred on the origin, weight 1."""
    origin = (-(n - 1) / 2 * h,) * 3
    p0, p1, p2 = (a.astype(np.float64) for a in mo.lattice_points(origin, h, (n, n, n)))
    tsdf = np.clip(sdf(p0, p1, p2) / trunc, -1, 1).astype(F32)
    return tsdf, np.ones_like(tsdf), origin


def sphere_sdf(R):
    return lambda x, y, z: np.sqrt(x * x + y * y + z * z) - R


def torus_sdf(Rmaj, r):
    return lambda x, y, z: np.sqrt((np.sqrt(x * x + y * y) - Rmaj) ** 2 + z * z) - r


def interpolation_bound(R, h):
    """Largest distance from a sphere of radius R of the zero of a linear interpolation of its distance function along a lattice
    edge (length at most sqrt(3) h): l^2 / 8 max |f''| with |f''| <= 1 / (R - l)."""
    edge = math.sqrt(3) * h
    return edge * edge / (8 * (R - edge))


def test_sphere_is_closed_manifold_with_the_right_volume():
    h, R = 0.1, 2.0                                          # R = 20 h
    tsdf, w, origin = analytic_volume(sphere_sdf(R), 48, h, 5 * h)
    v, f, c = mo.extract(tsdf, w, origin, h)
    assert c is None and len(f) > 1000
    assert mo.closed_and_oriented(f)
    chi, all_used = mo.euler(v, f)
    assert chi == 2 and all_used
    dist = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - R)
    assert dist.max() <= interpolation_bound(R, h) + 1e-5, (dist.max(), interpolation_bound(R, h))
    vol = mo.signed_volume(v, f)
    assert vol > 0 and abs(vol / (4 / 3 * math.pi * R ** 3) - 1) < 0.01, vol


def test_torus_has_euler_characteristic_zero():
    h = 0.1
    tsdf, w, origin = analytic_volume(torus_sdf(1.4, 0.6), 48, h, 5 * h)
    v, f, _ = mo.extract(tsdf, w, origin, h)
    assert mo.closed_and_oriented(f)
    assert mo.euler(v, f) == (0, True)
    assert mo.signed_volume(v, f) > 0


def test_clipped_plane_is_an_open_sheet_and_unobserved_volume_is_empty():
    h = 0.1
    tsdf, w, origin = analytic_volume(lambda x, y, z: z - 0.0137 - 0.2 * x, 20, h, 5 * h)
    v, f, _ = mo.extract(tsdf, w, origin, h)
    (uk, uc), (dk, dc), _ = mo.edge_counts(f)
    assert (dc == 1).all() and set(np.unique(uc)) == {1, 2}     # oriented, with a boundary
    assert mo.euler(v, f) == (1, True)                          # a disk
    # the normals point toward tsdf >= 0 (+z, with the slope of the plane)
    p = v[f].astype(np.float64)
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (n @ np.array([-0.2, 0.0, 1.0]) > 0).all()
    for wt in (np.zeros_like(w), w.copy()):
        if wt.any():
            wt[:, :, :] = 0.5                                   # observed, but below weight_min
        v0, f0, c0 = mo.extract(tsdf, wt, origin, h, color=np.zeros((3,) + tsdf.shape, F32))
        assert v0.shape == (0, 3) and f0.shape == (0, 3) and c0.shape == (0, 3)


def test_half_observed_sphere_is_open_where_the_weight_ends():
    h, R = 0.1, 1.5
    tsdf, w, origin = analytic_volume(sphere_sdf(R), 40, h, 5 * h)
    w[:, :, :20] = 0.0                                          # x < 0 unobserved
    v, f, _ = mo.extract(tsdf, w, origin, h)
    (uk, uc), (dk, dc), _ = mo.edge_counts(f)
    assert (dc == 1).all() and (uc == 1).any() and (uc <= 2).all()
    assert (v[:, 0] >= origin[0] + 19 * h - 1e-6).all()


def _plane_view(hw, seed=0):
    """A lattice camera and the z-depth image of a tilted plane n . X = c in its view space, computed along lgs_depth_normal's
    pixel rays in fp64 -> (view, proj, depth f32[H,W], (n, c))."""
    H, W = hw
    cam = scene.make_camera(3, 12, W, H, radius=3.0)
    V, P = cam["view"][0], cam["proj"][0]
    fx, fy = P[0, 0] * W * 0.5, P[1, 1] * H * 0.5
    n = np.array([0.2, -0.3, 1.0])
    c = 3.0
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    r = np.stack([(u - W / 2) / fx, (v - H / 2) / fy, np.ones_like(u)], -1)
    return V, P, (c / (r @ n)).astype(F32), (n, c)


def test_integration_of_an_analytic_plane():
    """T = 0: tsdf = min(1, sdf / trunc) with sdf = D(pixel) - z at every observed point (fp64 evaluation of the same rule, away
    from pixel borders); weight 0 behind the camera, outside the image, beyond the truncation band and where alpha <= alpha_min."""
    hw = (60, 80)
    H, W = hw
    Vm, Pm, D, _ = _plane_view(hw)
    h, dims, origin = 0.05, (40, 40, 40), (-1.0, -1.0, -1.0)
    trunc = 5 * h
    T = np.zeros((1, 1, H, W), F32)
    T[0, 0, :, : W // 4] = 0.6                                  # alpha 0.4 <= alpha_min on the left quarter
    vol = mo.integrate(mo.new_volume(dims, color=False), origin, h, trunc, D[None, None], T, Vm[None], Pm[None])
    p = [a.astype(np.float64) for a in mo.lattice_points(origin, h, dims)]
    X = np.stack(p + [np.ones_like(p[0])], -1) @ Vm.astype(np.float64)
    z = X[..., 2]
    fx, fy = Pm[0, 0] * W * 0.5, Pm[1, 1] * H * 0.5
    u, v = X[..., 0] / z * fx + W / 2, X[..., 1] / z * fy + H / 2
    inimg = (z > 0.01) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
    safe = inimg & (np.abs(u - np.round(u)) > 1e-3) & (np.abs(v - np.round(v)) > 1e-3)
    iu, iv = np.clip(np.floor(u), 0, W - 1).astype(int), np.clip(np.floor(v), 0, H - 1).astype(int)
    sdf = D[iv, iu].astype(np.float64) - z
    seen = safe & (iu >= W // 4) & (sdf >= -trunc + 1e-4)
    assert seen.sum() > 1000
    assert (vol["weight"][seen] == 1).all()
    np.testing.assert_allclose(vol["tsdf"][seen], np.minimum(1, sdf[seen] / trunc), atol=1e-4)
    unseen = safe & ((iu < W // 4) | (sdf < -trunc - 1e-4))
    assert unseen.sum() > 1000 and (vol["weight"][unseen] == 0).all() and (vol["tsdf"][unseen] == 1).all()
    assert (vol["weight"][~inimg & (np.abs(z) > 1e-3)] == 0).all()
    assert (~inimg).sum() > 500


def test_points_behind_outside_and_transparent_keep_weight_zero():
    hw = (20, 30)
    cam = scene.make_camera(0, 4, hw[1], hw[0])
    V, P = cam["view"][0], cam["proj"][0]
    eye = scene.fibonacci_camera(0, 4)
    fwd = -eye / np.linalg.norm(eye)
    pts = np.array([eye - fwd, eye + 1.0 * fwd + 5.0 * np.cross(fwd, [0, 1, 0]), eye + 2.0 * fwd], F32)   # behind, outside, ahead
    z, u, v = mo.project(pts[:, 0], pts[:, 1], pts[:, 2], V, P, *hw)
    assert z[0] < 0 and not (0 <= u[1] < hw[1]) and (0 <= u[2] < hw[1] and 0 <= v[2] < hw[0])
    for T_val, want in ((0.0, [0, 0, 1]), (0.5, [0, 0, 0]), (0.49, [0, 0, 1])):
        got = []                                                # each point as a one-point lattice
        for k in range(3):
            vk = mo.new_volume((1, 1, 1), color=True)
            mo.integrate(vk, pts[k], 1.0, 0.1, np.full((1, 1, *hw), 2.0, F32), np.full((1, 1, *hw), T_val, F32), V[None], P[None],
                         rgb=np.full((1, 3, *hw), 0.25, F32))
            got.append(float(vk["weight"][0, 0, 0]))
        assert got == want, (T_val, got)


def test_pixel_round_trip_with_the_depth_normal_ray():
    """A point that lgs_depth_normal's convention unprojects from pixel (u, v) at any expected depth projects back into (u, v)."""
    rng = np.random.default_rng(0)
    for hw, view in (((1080, 1920), 5), ((37, 53), 1), ((480, 640), 9)):
        H, W = hw
        cam = scene.make_camera(view, 12, W, H, radius=3.0, fov_x_deg=50.0)
        Vm, Pm = cam["view"][0], cam["proj"][0]
        u, v = rng.integers(0, W, 4000), rng.integers(0, H, 4000)
        ed = rng.uniform(0.5, 6.0, 4000)
        X = mo.unproject(u, v, ed, Vm, Pm, H, W).astype(F32)
        z, pu, pv = mo.project(X[:, 0], X[:, 1], X[:, 2], Vm, Pm, H, W)
        assert (np.floor(pu) == u).all() and (np.floor(pv) == v).all()


def test_colour_is_the_expected_colour():
    """rgb / alpha of one view, clamped to [0, 1]; two views average."""
    hw = (20, 30)
    cam = scene.make_camera(0, 4, hw[1], hw[0])
    V, P = cam["view"][0], cam["proj"][0]
    eye = scene.fibonacci_camera(0, 4)
    p = (eye - 2.0 * eye / np.linalg.norm(eye)).astype(F32)
    vk = mo.new_volume((1, 1, 1))
    T = np.full((2, 1, *hw), 0.2, F32)
    rgb = np.stack([np.full((3, *hw), 0.4, F32), np.full((3, *hw), 0.9, F32)])
    mo.integrate(vk, p, 1.0, 0.5, np.full((2, 1, *hw), 1.6, F32), T, np.stack([V, V]), np.stack([P, P]), rgb=rgb)
    assert vk["weight"][0, 0, 0] == 2
    np.testing.assert_allclose(vk["color"][:, 0, 0, 0], (0.5 + 1.0) / 2, rtol=1e-6)
    np.testing.assert_allclose(vk["tsdf"][0, 0, 0], 0.0, atol=1e-5)     # ED = 2 = z: on the surface


@pytest.mark.parametrize("colors", [False, True])
def test_mesh_ply_round_trip_is_bit_exact(tmp_path, colors):
    h, R = 0.1, 1.0
    tsdf, w, origin = analytic_volume(sphere_sdf(R), 28, h, 5 * h)
    col = np.random.default_rng(1).random((3,) + tsdf.shape).astype(F32) if colors else None
    v, f, c = mo.extract(tsdf, w, origin, h, color=col)
    path = str(tmp_path / "m.ply")
    ply.save_mesh_ply(path, v, f, c)
    v2, f2, c2 = ply.load_mesh_ply(path)
    assert v2.dtype == np.float32 and f2.dtype == np.int32
    assert v2.tobytes() == v.tobytes() and f2.tobytes() == f.tobytes()
    if colors:
        assert c2.dtype == np.uint8 and c2.tobytes() == c.tobytes()
    else:
        assert c2 is None
    head = open(path, "rb").read(400).split(b"end_header")[0].decode()
    assert "element face %d\nproperty list uchar int vertex_indices" % len(f) in head
    ply.save_mesh_ply(path, np.zeros((0, 3), F32), np.zeros((0, 3), np.int32))
    v3, f3, c3 = ply.load_mesh_ply(path)
    assert v3.shape == (0, 3) and f3.shape == (0, 3) and c3 is None
