"""Mesh extraction on the GPU (csrc/mesh.cu through litegs_b200.mesh): integration and extraction bit-identical to the numpy
restatement (tests/mesh_oracle.py) on analytic depth images, run to run and batch against single views; a 512^3 analytic sphere;
a sphere of thin opaque Gaussians rendered by render_view and fused by mesh_from_views; refusals; both examples."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from litegs_b200 import _lib, colmap, mesh, ply, scene
from litegs_b200.arguments import PipelineParams
from tests import mesh_oracle as mo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def sphere_views(n_views, hw, R, seed=0, radius=3.0):
    """n_views lattice cameras looking at a sphere of radius R at the origin: its z-depth along lgs_depth_normal's pixel rays
    (fp64), a random alpha in (0.3, 1] on the sphere (some at or below alpha_min = 0.5) -> D = alpha z, T = 1 - alpha (T = 1 off
    the sphere), rgb = alpha c with c in [0, 1.2] (clamped on the way in), views, projs; numpy f32."""
    H, W = hw
    rng = np.random.default_rng(seed)
    D, T, RGB, Vs, Ps = [], [], [], [], []
    for i in range(n_views):
        cam = scene.make_camera(i, n_views, W, H, radius=radius)
        Vm, Pm = cam["view"][0].astype(np.float64), cam["proj"][0].astype(np.float64)
        fx, fy = Pm[0, 0] * W * 0.5, Pm[1, 1] * H * 0.5
        u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
        r = np.stack([(u - W / 2) / fx, (v - H / 2) / fy, np.ones_like(u)], -1)
        Rinv = np.linalg.inv(Vm[:3, :3])
        c = -Vm[3, :3] @ Rinv
        d = r @ Rinv
        a, b, cc = (d * d).sum(-1), 2 * d @ c, c @ c - R * R
        disc = b * b - 4 * a * cc
        hit = disc > 0
        z = np.where(hit, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
        alpha = np.where(hit, rng.uniform(0.3, 1.0, (H, W)), 0.0)
        col = rng.uniform(0.0, 1.2, (3, H, W))
        D.append((alpha * z)[None]); T.append((1 - alpha)[None]); RGB.append(alpha[None] * col)
        Vs.append(Vm); Ps.append(Pm)
    return tuple(np.stack(x).astype(F32) for x in (D, T, RGB, Vs, Ps))


def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


GRID = dict(origin=(-1.2, -1.1, -1.3), h=0.08, dims=(31, 29, 33))


def _gpu_volume(batches, color=True):
    vol = mesh.TSDFVolume(GRID["origin"], GRID["h"], GRID["dims"], color=color)
    for D, T, C, V, P in batches:
        vol.integrate(*_dev(D, T, V, P), rgb=_dev(C)[0] if color else None)
    return vol


def _oracle_volume(batches, color=True):
    vol = mo.new_volume(GRID["dims"], color=color)
    for D, T, C, V, P in batches:
        mo.integrate(vol, GRID["origin"], GRID["h"], 5 * GRID["h"], D, T, V, P, rgb=C if color else None)
    return vol


def _batches():
    D, T, C, V, P = sphere_views(13, (72, 96), 0.9, seed=4)
    cut = [(0, 5), (5, 6), (6, 13)]
    return [(D[a:b], T[a:b], C[a:b], V[a:b], P[a:b]) for a, b in cut]


@pytest.mark.parametrize("color", [True, False])
def test_integration_is_the_restatement_bit_for_bit(cuda, color):
    """Three batches (5, 1 and 7 views): tsdf, weight and colour bit-identical to the restatement, to a second run and to 13
    single-view launches."""
    batches = _batches()
    ref = _oracle_volume(batches, color)
    a, b = _gpu_volume(batches, color), _gpu_volume(batches, color)
    single = _gpu_volume([tuple(x[i:i + 1] for x in bt) for bt in batches for i in range(bt[0].shape[0])], color)
    w = ref["weight"]
    print(f"integration: {int((w > 0).sum())} of {w.size} lattice points observed, weight up to {int(w.max())}")
    assert (w > 0).mean() > 0.2 and w.max() >= 3
    for name in ("tsdf", "weight") + (("color",) if color else ()):
        got = getattr(a, name).cpu().numpy()
        assert got.tobytes() == ref[name].tobytes(), (name, np.abs(got - ref[name]).max())
        assert torch.equal(getattr(a, name), getattr(b, name)) and torch.equal(getattr(a, name), getattr(single, name)), name
    assert not color and a.color is None or (ref["color"] > 0).any()


@pytest.mark.parametrize("weight_min", [1.0, 3.0])
def test_extraction_is_the_restatement(cuda, weight_min):
    """Vertices, faces and colours equal to the restatement's arrays in the canonical order."""
    batches = _batches()
    ref = _oracle_volume(batches)
    vol = _gpu_volume(batches)
    v, f, c = vol.extract(weight_min=weight_min)
    rv, rf, rc = mo.extract(ref["tsdf"], ref["weight"], GRID["origin"], GRID["h"], color=ref["color"], weight_min=weight_min)
    print(f"extraction (weight_min {weight_min}): {len(rv)} vertices, {len(rf)} faces")
    assert len(rf) > 300
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and c.dtype == torch.uint8
    assert v.cpu().numpy().tobytes() == rv.tobytes()
    assert np.array_equal(f.cpu().numpy(), rf)
    assert np.array_equal(c.cpu().numpy(), rc)
    v2, f2, c2 = vol.extract(weight_min=weight_min)
    assert torch.equal(v, v2) and torch.equal(f, f2) and torch.equal(c, c2)


def test_empty_and_unobserved_volumes(cuda):
    vol = mesh.TSDFVolume((0, 0, 0), 0.1, (8, 9, 10))
    for out in (vol.extract(), vol.extract(weight_min=0.0)):
        v, f, c = out
        assert v.shape == (0, 3) and f.shape == (0, 3) and c.shape == (0, 3) and v.is_cuda
    v, f, c = mesh.TSDFVolume((0, 0, 0), 0.1, (1, 1, 1), color=False).extract()
    assert v.shape == (0, 3) and c is None


def _sphere_volume(n, h, R, color=False):
    origin = (-(n - 1) / 2 * h,) * 3
    vol = mesh.TSDFVolume(origin, h, (n, n, n), color=color)
    ax = [torch.arange(n, device="cuda", dtype=torch.float32).mul_(F32(h)).add_(F32(o)).double() for o in origin]
    r = torch.sqrt(ax[0][None, None, :] ** 2 + ax[1][None, :, None] ** 2 + ax[2][:, None, None] ** 2)
    vol.tsdf.copy_(((r - R) / vol.sdf_trunc).clamp_(-1, 1).float())
    vol.weight.fill_(1.0)
    return vol


def interpolation_bound(R, h):
    edge = math.sqrt(3) * h
    return edge * edge / (8 * (R - edge))


def test_full_size_sphere(cuda):
    """512^3 lattice, R = 200 h: closed, consistently oriented, chi = 2, every vertex within the interpolation bound."""
    n, h = 512, 0.01
    R = 200 * h
    vol = _sphere_volume(n, h, R)
    torch.cuda.synchronize()
    v, f, _ = vol.extract()
    v, f = v.cpu().numpy(), f.cpu().numpy()
    assert mo.closed_and_oriented(f)
    chi, used = mo.euler(v, f)
    dist = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - R)
    vol_ratio = mo.signed_volume(v, f) / (4 / 3 * math.pi * R ** 3)
    print(f"512^3 sphere: {len(v)} vertices, {len(f)} faces, chi {chi}, max distance {dist.max() / h:.2e} h "
          f"(bound {interpolation_bound(R, h) / h:.2e} h), volume ratio {vol_ratio:.6f}")
    assert chi == 2 and used
    assert dist.max() <= interpolation_bound(R, h) + 1e-6
    assert abs(vol_ratio - 1) < 1e-3


def gaussian_sphere(n=30000, rho=1.0, colour=(0.8, 0.5, 0.2), chunk=128):
    """Thin, opaque, camera-independent Gaussians tangent to a sphere of radius rho: centres on a Fibonacci lattice, tangent
    scale 0.015, normal scale 0.0005, opacity sigmoid(5); the rotation is the half turn about the bisector of z and the normal,
    which maps the third axis to the normal whichever way the rotation matrix is read."""
    pts = np.stack([scene.fibonacci_camera(i, n, rho) for i in range(n)], 1)
    nrm = pts / rho
    a = nrm + np.array([0.0, 0.0, 1.0])[:, None]
    a /= np.linalg.norm(a, axis=0, keepdims=True)
    rot = np.concatenate([np.zeros((1, n)), a])
    order = scene.morton_order(pts)
    sh0 = (np.asarray(colour)[:, None] - 0.5) / colmap.SH_C0
    raw = dict(xyz=pts, scale=np.log(np.array([[0.015], [0.015], [0.0005]])) * np.ones((1, n)), rot=rot,
               sh_0=np.repeat(sh0[None], n, axis=2), sh_rest=np.zeros((15, 3, n)), opacity=np.full((1, n), 5.0))
    P = {k: torch.from_numpy(scene.cluster(np.ascontiguousarray(v[..., order]).astype(F32), chunk)).cuda() for k, v in raw.items()}
    return P


def test_gaussian_sphere_end_to_end(cuda):
    """A sphere (R = 40 h) of thin opaque Gaussians from 24 lattice cameras through render_view and mesh_from_views: a closed
    mesh with chi = 2, vertices near the sphere and coloured like the Gaussians."""
    rho = 1.0
    h = rho / 40
    P = gaussian_sphere(rho=rho)
    hw = (400, 400)
    cams = [{k: torch.from_numpy(x).cuda() for k, x in scene.make_camera(i, 24, hw[1], hw[0], radius=3.0).items()} for i in range(24)]
    vol = mesh.bounding_volume(None, bounds=(-1.3, -1.3, -1.3, 1.3, 1.3, 1.3), resolution=105)
    assert abs(vol.voxel_size - h) < 1e-9
    mesh.mesh_from_views(P, cams, hw, PipelineParams(tile_size=(8, 16)), vol, batch=16)
    v, f, c = vol.extract()
    v, f, c = v.cpu().numpy(), f.cpu().numpy(), c.cpu().numpy()
    chi, used = mo.euler(v, f)
    dist = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - rho) / h
    cerr = np.abs(c.astype(np.float64) - np.array([0.8, 0.5, 0.2]) * 255).max()
    print(f"Gaussian sphere R = 40 h, 24 views {hw}: {len(v)} vertices, {len(f)} faces, chi {chi}, closed "
          f"{mo.closed_and_oriented(f)}; distance to the sphere max {dist.max():.3f} h, mean {dist.mean():.3f} h; colour error "
          f"max {cerr:.2f} / 255")
    assert mo.closed_and_oriented(f) and chi == 2 and used
    # measured on an H100: max 0.964 h, mean 0.264 h, colour 0.50 / 255
    assert dist.max() <= 1.25 and dist.mean() <= 0.35
    assert cerr <= 2.0
    assert mo.signed_volume(v, f) > 0


def test_refusals(cuda):
    vol = mesh.TSDFVolume((0, 0, 0), 0.1, (4, 4, 4))
    D, T, C, V, P = _dev(*sphere_views(2, (8, 10), 0.1))
    with pytest.raises(RuntimeError, match="float32 CUDA"):
        vol.integrate(D.double(), T, V, P, rgb=C)
    with pytest.raises(RuntimeError, match="float32 CUDA"):
        vol.integrate(D.cpu(), T, V, P, rgb=C)
    with pytest.raises(RuntimeError, match=r"trans must be \[2,1,8,10\]"):
        vol.integrate(D, T[..., :9], V, P, rgb=C)
    with pytest.raises(RuntimeError, match=r"views must be \[2,4,4\]"):
        vol.integrate(D, T, V[:, :3], P, rgb=C)
    with pytest.raises(RuntimeError, match=r"rgb must be \[2,3,8,10\]"):
        vol.integrate(D, T, V, P, rgb=C[:, :2])
    with pytest.raises(RuntimeError, match="rgb is required"):
        vol.integrate(D, T, V, P)
    with pytest.raises(RuntimeError, match="alpha_min"):
        vol.integrate(D, T, V, P, rgb=C, alpha_min=1.0)
    with pytest.raises(RuntimeError, match="2\\^31 - 1"):
        mesh.TSDFVolume((0, 0, 0), 0.1, (2048, 1024, 1024))
    with pytest.raises(RuntimeError, match="CUDA device"):
        mesh.TSDFVolume((0, 0, 0), 0.1, (4, 4, 4), device="cpu")
    # totals of 2^31 are refused before anything is written: by the host check and by the entry point itself
    with pytest.raises(RuntimeError, match="below 2\\^31"):
        mesh.check_totals(1 << 31, 0)
    N = 64
    u8 = [torch.zeros(N, dtype=torch.uint8, device=cuda) for _ in range(2)]
    i64 = [torch.zeros(N, dtype=torch.int64, device=cuda) for _ in range(2)]
    for nv, nf in ((1 << 31, 0), (0, 1 << 31)):
        with pytest.raises(_lib.LiteGSB200Error, match="below 2\\^31"):
            _lib.call("lgs_mesh_emit", vol.tsdf.data_ptr(), None, 4, 4, 4, 0.0, 0.0, 0.0, 0.1, u8[0].data_ptr(), u8[1].data_ptr(),
                      i64[0].data_ptr(), i64[1].data_ptr(), nv, nf, None, None, None, None)


def _run(args, cwd):
    r = subprocess.run([sys.executable, *args], cwd=cwd, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_extract_mesh_example(cuda, tmp_path):
    """examples/extract_mesh.py on a cloud that examples/render_ply.py --make wrote."""
    model = str(tmp_path / "cloud.ply")
    _run([os.path.join(ROOT, "examples", "render_ply.py"), "--make", model, "--out", str(tmp_path / "renders"), "--views", "1",
          "--width", "64", "--height", "48"], tmp_path)
    out = str(tmp_path / "mesh.ply")
    log = _run([os.path.join(ROOT, "examples", "extract_mesh.py"), "--ply", model, "--views", "12", "--width", "320", "--height", "240",
                "--resolution", "128", "--out", out], tmp_path)
    print(log.strip())
    v, f, c = ply.load_mesh_ply(out)
    assert len(v) > 0 and len(f) > 0 and c is not None and f.max() < len(v)
    assert f"{len(v)} vertices" in log and f"{len(f)} faces" in log


def test_train_colmap_mesh(cuda, tmp_path):
    """train_colmap.py --make DIR --iters 50 --depth-normal-weight 0.1 --mesh out.ply writes a mesh load_mesh_ply reads back."""
    out = str(tmp_path / "out.ply")
    log = _run([os.path.join(ROOT, "examples", "train_colmap.py"), "--make", str(tmp_path / "ds"), "--iters", "50",
                "--depth-normal-weight", "0.1", "--mesh", out], tmp_path)
    print(log.strip().splitlines()[-1])
    v, f, c = ply.load_mesh_ply(out)
    assert len(f) > 0 and c is not None and f.max() < len(v)
