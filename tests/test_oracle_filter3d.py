"""Mip-Splatting's 3D smoothing filter on the CPU (numpy restatement in tests/filter3d_oracle.py): the filter against a loop written
the way Mip-Splatting's compute_3D_filter is, the gradients of filtered renders against fp64 central differences, the algebra of
the filtered scale and opacity, f = 0 against no filter, and the filter_3D property of PLY files."""
import math
import os

import numpy as np
import pytest

import oracle
from litegs_b200 import ply, scene
from tests import filter3d_oracle as f3
from tests import fused_oracle as fo
from tests.util import PARAM_KEYS, f64_arrays, small_scene, tiny_scene

HW, TILE, DEG = (32, 32), (8, 8), 2


def _cameras():
    """Five cameras on one side of the scene (z < 0, looking towards +z) with different image sizes and fields of view."""
    specs = [((0.3, 0.2, -3.0), 64, 48, 60.0), ((-0.8, 0.1, -2.5), 96, 96, 45.0), ((0.5, -0.6, -3.5), 40, 80, 75.0),
             ((0.0, 0.9, -2.8), 128, 72, 50.0), ((-0.4, -0.3, -4.0), 33, 47, 90.0)]
    views, projs, hws, raw = [], [], [], []
    for eye, w, h, fov in specs:
        V = scene.look_at_view_matrix(np.array(eye), target=(0.0, 0.0, 0.5))
        P = scene.proj_matrix(w, h, fov)
        views.append(V); projs.append(P); hws.append((h, w))
        raw.append((V.astype(np.float64), w, h, fov))
    return np.stack(views), np.stack(projs), np.array(hws, np.int32), raw


def _points(seed=0, n=3000):
    """Points in front of the cameras, behind all of them (z < -5), and far to the side (outside the 1.15 margin)."""
    rng = np.random.default_rng(seed)
    front = rng.uniform(-1.5, 1.5, (3, n))
    behind = np.stack([rng.uniform(-1, 1, 200), rng.uniform(-1, 1, 200), rng.uniform(-9, -6, 200)])
    side = np.stack([rng.choice([-1, 1], 200) * rng.uniform(40, 60, 200), rng.uniform(-1, 1, 200), rng.uniform(0, 2, 200)])
    return np.concatenate([front, behind, side], axis=1).astype(np.float32)


def _mip_splatting_filter(xyz, raw):
    """compute_3D_filter as Mip-Splatting writes it, per camera, in fp64: xyz_cam = xyz @ R + T, focal_x = W / (2 tan(fov_x / 2)),
    the depth test z > 0.2 and the 15 % screen margin, the largest focal_x, unseen points set to the largest seen distance."""
    xyz = xyz.astype(np.float64).T
    distance = np.full(xyz.shape[0], 100000.0)
    valid_points = np.zeros(xyz.shape[0], bool)
    focal_length = 0.0
    for V, W, H, fov in raw:
        R, T = V[:3, :3], V[3, :3]
        xyz_cam = xyz @ R + T[None, :]
        valid_depth = xyz_cam[:, 2] > 0.2
        x, y, z = xyz_cam[:, 0], xyz_cam[:, 1], xyz_cam[:, 2]
        z = np.maximum(z, 0.001)
        focal_x = W / (2 * math.tan(math.radians(fov) / 2))
        focal_y = focal_x                                           # square pixels: fov_y follows from the aspect
        x = x / z * focal_x + W / 2.0
        y = y / z * focal_y + H / 2.0
        in_screen = (x >= -0.15 * W) & (x <= W * 1.15) & (y >= -0.15 * H) & (y <= 1.15 * H)
        valid = valid_depth & in_screen
        distance[valid] = np.minimum(distance[valid], z[valid])
        valid_points |= valid
        focal_length = max(focal_length, focal_x)
    distance[~valid_points] = distance[valid_points].max()
    return distance / focal_length * (0.2 ** 0.5), valid_points


def test_filter_matches_mip_splatting_loop():
    views, projs, hws, raw = _cameras()
    xyz = _points()
    want, seen = _mip_splatting_filter(xyz, raw)
    got = f3.compute_filter(xyz, views, projs, hws)
    assert got.dtype == np.float32 and got.shape == (xyz.shape[1],)
    n_front = 3000
    assert seen[:n_front].mean() > 0.5 and not seen[n_front:].any()          # behind every camera and outside the margin: unseen
    rel = np.abs(got.astype(np.float64) - want) / want
    print(f"3D filter vs the fp64 loop: {rel.max():.2e} relative, {(~seen).sum()} unseen points")
    assert rel.max() < 4e-6
    assert np.all(got[~seen] == got[seen].max())
    got64 = f3.compute_filter(xyz, views, projs, hws, dt=np.float64)
    assert np.abs(got64 / want - 1).max() < 1e-7          # the fp32 projection matrices' focal lengths differ in the 8th digit
    # no point seen: 0 everywhere
    assert np.all(f3.compute_filter(xyz[:, n_front:], views, projs, hws) == 0)


def test_filter_factor_algebra():
    """rho3^2 prod qf_k = prod q_k to fp64 rounding, 0 < rho3 <= 1 and s'_k >= max(s_k, f), over sixteen decades of s / f."""
    rng = np.random.default_rng(0)
    s = np.exp(rng.uniform(-9, 2, (3, 20000)))
    f = np.exp(rng.uniform(-9, 0, 20000))
    o = rng.uniform(0, 1, (1, 20000))
    sp, o3, ff = f3.filter_forward(s, f, o)
    lhs = ff["rho3"] ** 2 * ff["qf"].prod(axis=0)
    rhs = ff["q"].prod(axis=0)
    assert np.all(np.abs(lhs - rhs) <= 1e-14 * rhs)
    assert np.all(ff["rho3"] > 0) and np.all(ff["rho3"] <= 1) and np.all(o3 <= o)
    assert np.all(sp >= s) and np.all(sp >= f[None])
    # fp32: the same within single rounding
    sp32, _, ff32 = f3.filter_forward(s.astype(np.float32), f.astype(np.float32), o.astype(np.float32))
    assert np.abs(ff32["rho3"] / ff["rho3"] - 1).max() < 1e-5
    assert np.all(sp32 >= s.astype(np.float32))


def _filter_for(P, seed=0, lo=0.02, hi=0.12):
    C, S = P["xyz"].shape[-2:]
    return np.random.default_rng(seed).uniform(lo, hi, (1, C, S))


@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("true_sigmoid", [False, True])
def test_fp64_finite_differences_with_frozen_lists(true_sigmoid, antialiased):
    """scale, rot, sh and opacity of a filtered render (f held constant) equal fp64 central differences with the tile lists
    frozen.  Under the reference's sigmoid convention the opacity gradient is the true one divided by 1 - sigma."""
    P, aabb, cam = tiny_scene()
    filt = _filter_for(P)
    rng = np.random.default_rng(1)
    w = rng.normal(size=(1, 3, *HW))
    kw = dict(antialiased=antialiased, filter_3d=filt)
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, DEG, lambda img: w, true_sigmoid_grad=true_sigmoid, **kw)
    assert out["rho3"].min() < 0.5 and out["rho3"].max() > 0.8
    lists = (out["ranges"], out["sorted_pid"])
    ids = out["visible_chunk_id"]
    run = lambda Q: (fo.render_forward_backward(Q, aabb, cam, HW, TILE, DEG, lambda img: w, lists=lists, **kw)["img"] * w).sum()
    sig = 1 / (1 + np.exp(-P["opacity"]))
    checked = 0
    for name in ("scale", "rot", "sh_0", "sh_rest", "opacity"):
        g = out["grads"][name]
        for _ in range(8):
            idx = tuple(int(rng.integers(0, s)) for s in g.shape)
            full = list(idx); full[-2] = int(ids[idx[-2]]); full = tuple(full)
            h = 1e-6
            Pp = {k: v.copy() for k, v in P.items()}; Pp[name][full] += h
            Pm = {k: v.copy() for k, v in P.items()}; Pm[name][full] -= h
            fd = (run(Pp) - run(Pm)) / (2 * h)
            want = g[idx]
            if name == "opacity" and not true_sigmoid:
                want = want * (1 - sig[full])
            assert abs(fd - want) <= 1e-4 * max(1e-3, abs(fd), abs(want)), (name, idx, fd, want)
            checked += abs(fd) > 1e-6
    assert checked >= 20


@pytest.mark.parametrize("antialiased", [False, True])
def test_fp64_finite_differences_xyz_and_camera_with_frozen_J_and_dirs(antialiased):
    """xyz and the camera (view and projection matrices) of a filtered render, with J, the SH directions and the tile lists
    frozen: the analytic gradients equal central differences."""
    P, aabb, cam = tiny_scene(seed=5)
    filt = _filter_for(P, seed=1)
    rng = np.random.default_rng(2)
    w = rng.normal(size=(1, 3, *HW))
    kw = dict(antialiased=antialiased, filter_3d=filt)
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, DEG, lambda img: w, true_sigmoid_grad=True, **kw)
    freeze = dict(J=out["inter"]["J"], color=out["color"])
    lists = (out["ranges"], out["sorted_pid"])
    ids = out["visible_chunk_id"]

    def loss(Q, c=cam):
        return (fo.render_forward_backward(Q, aabb, c, HW, TILE, DEG, lambda img: w, lists=lists, freeze=freeze, **kw)["img"] * w).sum()

    g = out["grads"]["xyz"]
    h = 1e-6
    for _ in range(10):
        c, a, s = int(rng.integers(0, 3)), int(rng.integers(0, g.shape[1])), int(rng.integers(0, g.shape[2]))
        Pp = {k: v.copy() for k, v in P.items()}; Pp["xyz"][c, ids[a], s] += h
        Pm = {k: v.copy() for k, v in P.items()}; Pm["xyz"][c, ids[a], s] -= h
        fd = (loss(Pp) - loss(Pm)) / (2 * h)
        assert abs(fd - g[c, a, s]) <= 1e-4 * max(1e-3, abs(fd), abs(g[c, a, s])), (fd, g[c, a, s])
    d_view, d_proj = fo.camera_backward(P, out, cam, HW)
    for which, gc in (("view", d_view), ("proj", d_proj)):
        for k in range(4):
            for j in range(4):
                if which == "proj" and j == 2:
                    continue
                cp = {n: cam[n].copy() for n in ("view", "proj")}
                cm = {n: cam[n].copy() for n in ("view", "proj")}
                cp[which][0, k, j] += h
                cm[which][0, k, j] -= h
                fd = (loss(P, dict(cam, **cp)) - loss(P, dict(cam, **cm))) / (2 * h)
                assert abs(fd - gc[k, j]) <= 1e-4 * max(1e-3, abs(fd), abs(gc[k, j])), (which, k, j, fd, gc[k, j])


@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_zero_filter_and_no_filter_are_the_same_bits(dt, antialiased):
    """f = 0 gives the unfiltered render bit for bit, forward and gradients; with the antialiased mode off as well, both are the
    oracle's own composition.  One oracle thread: the raster backward's sums are reproducible only then."""
    hw, tile = (48, 64), (16, 16)
    params, aabb, cam = small_scene(n=800, hw=hw, seed=4)
    if dt == np.float64:
        params, aabb, cam = f64_arrays(params), tuple(a.astype(np.float64) for a in aabb), f64_arrays(cam)
    w = np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(dt)
    zero = np.zeros((1, *params["xyz"].shape[-2:]), dt)
    nt = oracle.num_threads()
    oracle.set_num_threads(1)
    try:
        a = oracle.render_forward_backward(params, aabb, cam, hw, tile, 3, lambda img: w, true_sigmoid_grad=True)
        b = fo.render_forward_backward(params, aabb, cam, hw, tile, 3, lambda img: w, true_sigmoid_grad=True, antialiased=antialiased)
        c = fo.render_forward_backward(params, aabb, cam, hw, tile, 3, lambda img: w, true_sigmoid_grad=True, antialiased=antialiased,
                                       filter_3d=zero)
    finally:
        oracle.set_num_threads(nt)
    for ref, other in [(b, c)] + ([] if antialiased else [(a, b)]):
        for k in ("img", "T", "last", "fragile", "ranges", "sorted_pid", "d_ndc", "d_cov", "d_col", "d_op", "opacity"):
            assert np.array_equal(ref[k], other[k]), k
        for k in PARAM_KEYS:
            assert np.array_equal(ref["grads"][k], other["grads"][k]), k
    assert np.all(c["rho3"] == 1)


def test_ply_round_trip_with_filter(tmp_path):
    p = scene.make_scene(300, sh_degree=1, chunk=32, seed=2)
    p["filter_3D"] = scene.cluster(np.random.default_rng(0).uniform(0.001, 0.1, (1, 300)).astype(np.float32), 32)
    path = os.path.join(tmp_path, "f.ply")
    ply.params_to_ply(path, p, p["n_points"])
    with open(path, "rb") as fh:
        header = fh.read(4096).split(b"end_header")[0].decode().split("\n")
    props = [ln.split()[-1] for ln in header if ln.startswith("property")]
    assert props[-2:] == ["rot_3", "filter_3D"]
    q = ply.params_from_ply(path, 1, 32)
    for k in PARAM_KEYS + ("filter_3D",):
        assert np.array_equal(q[k], p[k]), k
    flat = ply.load_ply(path, 1)
    assert len(flat) == 6


def test_ply_without_filter_reads_as_before(tmp_path):
    p = scene.make_scene(300, sh_degree=1, chunk=32, seed=2)
    path = os.path.join(tmp_path, "n.ply")
    ply.params_to_ply(path, p, p["n_points"])
    q = ply.params_from_ply(path, 1, 32)
    assert "filter_3D" not in q
    assert sorted(q) == sorted(PARAM_KEYS + ("cluster_origin", "cluster_extend", "n_points"))
    for k in PARAM_KEYS + ("cluster_origin", "cluster_extend"):
        assert np.array_equal(q[k], p[k]), k


def test_filtered_cluster_aabb_covers_the_widened_splats():
    """cluster_aabb with a filter: the boxes are those of the splats with scale sqrt(s^2 + f^2), and the torch form agrees."""
    import torch
    p = scene.make_scene(2000, sh_degree=0, chunk=64, seed=1)
    filt = np.random.default_rng(0).uniform(0.0, 0.05, (1, *p["xyz"].shape[-2:])).astype(np.float32)
    o0, e0 = scene.cluster_aabb(p["xyz"], p["scale"], p["rot"])
    o1, e1 = scene.cluster_aabb(p["xyz"], p["scale"], p["rot"], filter_3d=filt)
    assert np.all(e1 >= e0) and np.any(e1 > e0 * 1.01)
    widened = np.log(np.sqrt(np.exp(p["scale"].astype(np.float64)) ** 2 + filt.astype(np.float64) ** 2))
    o2, e2 = scene.cluster_aabb(p["xyz"], widened, p["rot"])
    assert np.allclose(o1, o2, atol=1e-6) and np.allclose(e1, e2, atol=1e-6)
    assert np.array_equal(scene.cluster_aabb(p["xyz"], p["scale"], p["rot"], filter_3d=np.zeros_like(filt))[1], e0)
    ot, et = scene.cluster_aabb_torch(*(torch.from_numpy(p[k]) for k in ("xyz", "scale", "rot")), filter_3d=torch.from_numpy(filt))
    assert np.allclose(ot.numpy(), o1, atol=1e-5) and np.allclose(et.numpy(), e1, atol=1e-5)
