"""CPU tests of the camera path's restatement (tests/camera_oracle.py): create_viewproj against the COLMAP camera builder, finite
differences and the reference's fixture; the camera gradient of a render against fp64 central differences with J, the SH
directions, the tile lists and the colours frozen, and the translation identity sum_i d xyz_i = V3x3 . d_view[3, :3]."""
import os

import numpy as np
import pytest

import oracle
from litegs_b200 import colmap, scene
from tests import camera_oracle as co
from tests.util import tiny_scene

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "viewproj.npz")
ZN, ZF = 0.01, 5000.0


def _params(n, seed, unit=True):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    if not unit:
        q *= rng.uniform(0.6, 1.5, size=(n, 1))
    return np.concatenate([q, rng.normal(size=(n, 3))], axis=1)


def test_forward_equals_the_colmap_camera():
    """A centred pinhole with fx = fy: view, proj and planes as colmap.camera_from_colmap / scene.frustum_planes build them."""
    H, W = 1080, 1920
    p = _params(3, 0)
    fx = 1400.0
    recp = np.array([fx / (W * 0.5)])
    view, proj, vp, planes = co.create_viewproj_forward(p, recp, H, W, ZN, ZF)
    for v in range(3):
        cam = colmap.camera_from_colmap(p[v, :4], p[v, 4:], [fx, fx, W / 2, H / 2], W, H, ZN, ZF)
        assert np.allclose(view[v], cam["view"][0], atol=1e-6)
        assert np.allclose(proj[v], cam["proj"][0], rtol=1e-6, atol=1e-9)
        assert np.allclose(planes[v], scene.frustum_planes(cam["view"][0], cam["proj"][0]), rtol=1e-5, atol=1e-5)


def _loss_of_params(p, recp, H, W, G):
    view, proj, vp, _ = co.create_viewproj_forward(p, recp, H, W, ZN, ZF)
    return float(np.sum(view * G[0]) + np.sum(proj * G[1]) + np.sum(vp * G[2]))


@pytest.mark.parametrize("unit", [True, False])
def test_backward_is_the_finite_difference_times_norm(unit):
    """fp64 central differences of <G, (view, proj, viewproj)>: equal at |q| = 1, |q| x the finite difference otherwise
    (the normalisation backward runs on the already normalised quaternion, GR/compact.cu:279-285)."""
    H, W = 96, 128                    # integer aspect quotient == 1 (128 // 96): the fov check is the next test
    p = _params(2, 1, unit)
    recp = np.array([1.3])
    rng = np.random.default_rng(2)
    G = [rng.normal(size=(2, 4, 4)) for _ in range(3)]
    gp, _ = co.create_viewproj_backward(G[0], G[1], G[2], p, recp, H, W, ZN, ZF)
    h = 1e-6
    for v in range(2):
        for k in range(7):
            pp, pm = p.copy(), p.copy()
            pp[v, k] += h; pm[v, k] -= h
            fd = (_loss_of_params(pp, recp, H, W, G) - _loss_of_params(pm, recp, H, W, G)) / (2 * h)
            want = fd * (np.linalg.norm(p[v, :4]) if k < 4 else 1.0)
            assert abs(gp[v, k] - want) <= 1e-6 * max(1.0, abs(want)), (v, k, gp[v, k], want)


def test_fov_gradient_uses_the_integer_aspect_ratio():
    """d recp = d proj[0][0] + d proj[1][1] * (img_w // img_h) (GR/compact.cu:276): at 1920x1080 the factor is 1, not 16/9."""
    H, W = 1080, 1920
    p = _params(1, 3)
    recp = np.array([1.7])
    G = [np.zeros((1, 4, 4)), np.zeros((1, 4, 4)), np.zeros((1, 4, 4))]
    G[1][0, 1, 1] = 1.0
    _, gr = co.create_viewproj_backward(G[0], G[1], G[2], p, recp, H, W, ZN, ZF)
    assert gr[0] == 1.0
    h = 1e-6
    fd = (_loss_of_params(p, recp + h, H, W, G) - _loss_of_params(p, recp - h, H, W, G)) / (2 * h)
    assert abs(fd - W / H) < 1e-6                   # the true derivative, which the reference does not return
    G[1][0, 0, 0] = 2.0
    _, gr = co.create_viewproj_backward(G[0], G[1], G[2], p, recp, 1080, 3000, ZN, ZF)
    assert gr[0] == 2.0 + 2.0                       # 3000 // 1080 == 2


def test_oracle_matches_the_reference_fixture():
    """tests/golden/viewproj.npz: the reference's create_viewproj kernels on an H100 (tests/golden/make_golden_viewproj.py)."""
    g = np.load(GOLD)
    H, W = 1080, 1920
    view, proj, vp, planes = co.create_viewproj_forward(g["view_params"], g["recp"], H, W, ZN, ZF)
    for k, a in (("view", view), ("proj", proj), ("viewproj", vp), ("frustumplane", planes)):
        assert np.allclose(a, g[k], rtol=1e-5, atol=1e-5 * np.abs(g[k]).max()), k
    gp, _ = co.create_viewproj_backward(g["g_view"], g["g_proj"], g["g_viewproj"], g["view_params"], g["recp"], H, W, ZN, ZF)
    assert np.abs(gp - g["grad_view_params"]).max() <= 1e-4 * np.abs(g["grad_view_params"]).max()
    _, gr = co.create_viewproj_backward(g["g_view"][:1], g["g_proj"][:1], g["g_viewproj"][:1], g["view_params"][:1], g["recp"], H, W, ZN, ZF)
    assert abs(gr[0] - g["grad_recp_v1"][0]) <= 1e-4 * max(1.0, abs(g["grad_recp_v1"][0]))
    assert np.any(np.abs(np.linalg.norm(g["view_params"][:, :4], axis=1) - 1) > 0.1)      # the fixture covers |q| != 1


def _render_case(seed=5):
    P, aabb, cam = tiny_scene(seed=seed, log_scale_range=(0.05, 0.2))
    hw, tile = (32, 32), (8, 8)
    w = np.random.default_rng(2).normal(size=(1, 3, 32, 32))
    out = oracle.render_forward_backward(P, aabb, cam, hw, tile, 2, lambda img: w, true_sigmoid_grad=True)
    return P, aabb, cam, hw, tile, w, out


def test_camera_gradient_matches_finite_differences_with_frozen_J_and_dirs():
    """The convention of the position gradient (test_fp64_finite_differences_xyz_with_frozen_J_and_dirs) applied to the camera:
    J, SH directions, tile lists, colours and opacities frozen; the mean (MVP) and Sigma2 = (T V3x3 J)^T (T V3x3 J) + 0.3 I follow
    the perturbed matrices.  All 16 d_view entries and the d_proj entries that are not identically zero."""
    P, aabb, cam, hw, tile, w, out = _render_case()
    inter = out["inter"]
    ids = out["visible_chunk_id"]
    xyz = np.concatenate([P["xyz"][:, ids, :].reshape(3, -1), np.ones((1, inter["view_pos"].shape[2]))])

    def loss(view, proj):
        vp, ndc = oracle.mvp_transform_forward(xyz, view, proj)
        cov = oracle.createCov2dDirectly_forward(inter["J"], view, inter["T"])
        _, _, inv = oracle.eigh_and_inv_2x2matrix_forward(cov)
        img, *_ = oracle.rasterize_forward(out["sorted_pid"], out["ranges"], ndc, inv, out["color"], out["opacity"], None, hw[0], hw[1], *tile)
        return (np.clip(img[..., :hw[0], :hw[1]], 0, 1) * w).sum()

    d_view, d_proj, _ = co.camera_backward(P, out, cam, hw)
    assert np.abs(d_view).max() > 0 and np.abs(d_proj).max() > 0
    h = 1e-6
    checked = 0
    for which, g in (("view", d_view), ("proj", d_proj)):
        for k in range(4):
            for j in range(4):
                if which == "proj" and j == 2:
                    assert g[k, j] == 0          # ndc z is not used by the rasteriser
                    continue
                cp = {n: cam[n].copy() for n in ("view", "proj")}
                cm = {n: cam[n].copy() for n in ("view", "proj")}
                cp[which][0, k, j] += h
                cm[which][0, k, j] -= h
                fd = (loss(cp["view"], cp["proj"]) - loss(cm["view"], cm["proj"])) / (2 * h)
                assert abs(fd - g[k, j]) <= 1e-4 * max(1e-3, abs(fd), abs(g[k, j])), (which, k, j, fd, g[k, j])
                checked += 1
    assert checked == 28


def test_translation_identity_in_fp64():
    """Moving the camera by t moves every Gaussian by -t and Sigma2 does not change while J is frozen: sum_i d xyz_i equals
    V3x3 . d_view[3, :3] (row-vector convention: sum_j V[k][j] d_view[3][j])."""
    for seed in (5, 6):
        P, aabb, cam, hw, tile, w, out = _render_case(seed)
        d_view, _, parts = co.camera_backward(P, out, cam, hw)
        s = out["grads"]["xyz"].reshape(3, -1).sum(axis=1)
        rhs = cam["view"][0, :3, :3] @ d_view[3, :3]
        assert np.abs(s).max() > 0
        assert np.abs(s - rhs).max() <= 1e-9 * np.abs(s).max(), (s, rhs)
        assert np.all(parts["sigma_view"][:, 3, :] == 0) and np.abs(parts["sigma_view"]).max() > 0
