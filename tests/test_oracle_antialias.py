"""The antialiased mode on the CPU (fp64 restatement in tests/aa_oracle.py, composed by tests/fused_oracle.py): its gradients
against central finite differences, the off switch, the range of rho, the integrated alpha of one splat and the consistency of
renders across resolutions."""
import math

import numpy as np
import pytest

import oracle
from litegs_b200 import scene
from tests import aa_oracle as aa
from tests import camera_oracle as co
from tests import fused_oracle as fo
from tests.util import PARAM_KEYS, f64_arrays, single_splat, small_scene, tiny_scene


HW, TILE, DEG = (32, 32), (8, 8), 2


@pytest.mark.parametrize("true_sigmoid", [False, True])
def test_fp64_finite_differences_with_frozen_lists(true_sigmoid):
    """scale, rot, sh and opacity: the analytic gradients of the antialiased render equal fp64 central differences of the same
    render with the tile lists frozen.  Under the reference's convention (true_sigmoid False) the opacity gradient is the true
    one divided by 1 - sigma (SURVEY Q15), and the check divides it out."""
    P, aabb, cam = tiny_scene()
    rng = np.random.default_rng(1)
    w = rng.normal(size=(1, 3, *HW))
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, DEG, lambda img: w, true_sigmoid_grad=true_sigmoid, antialiased=True)
    assert out["rho"].min() < 0.5 and out["rho"].max() > 0.8           # sub-pixel and larger splats both present
    lists = (out["ranges"], out["sorted_pid"])
    ids = out["visible_chunk_id"]
    run = lambda Q: (fo.render_forward_backward(Q, aabb, cam, HW, TILE, DEG, lambda img: w, antialiased=True, lists=lists)["img"] * w).sum()
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


def test_fp64_finite_differences_xyz_with_frozen_J_and_dirs():
    """xyz: with J, the SH directions and the tile lists frozen, the analytic d xyz of the antialiased render equals central
    differences.  J frozen makes Sigma2 and so rho independent of the position: the gradient flows through the NDC mean only."""
    P, aabb, cam = tiny_scene(seed=5)
    rng = np.random.default_rng(2)
    w = rng.normal(size=(1, 3, *HW))
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, DEG, lambda img: w, true_sigmoid_grad=True, antialiased=True)
    freeze = dict(J=out["inter"]["J"], color=out["color"])
    lists = (out["ranges"], out["sorted_pid"])
    ids = out["visible_chunk_id"]
    g = out["grads"]["xyz"]

    def loss(Q):
        return (fo.render_forward_backward(Q, aabb, cam, HW, TILE, DEG, lambda img: w, antialiased=True, lists=lists,
                                           freeze=freeze)["img"] * w).sum()

    for _ in range(10):
        c, a, s = int(rng.integers(0, 3)), int(rng.integers(0, g.shape[1])), int(rng.integers(0, g.shape[2]))
        h = 1e-6
        Pp = {k: v.copy() for k, v in P.items()}; Pp["xyz"][c, ids[a], s] += h
        Pm = {k: v.copy() for k, v in P.items()}; Pm["xyz"][c, ids[a], s] -= h
        fd = (loss(Pp) - loss(Pm)) / (2 * h)
        assert abs(fd - g[c, a, s]) <= 1e-4 * max(1e-3, abs(fd), abs(g[c, a, s])), (fd, g[c, a, s])


def test_camera_gradient_matches_finite_differences_with_frozen_J_and_dirs():
    """The camera gradient with the antialiasing term (fused_oracle.camera_backward) against central differences of the view and
    projection matrices, J, SH directions and tile lists frozen."""
    P, aabb, cam = tiny_scene(seed=5)
    w = np.random.default_rng(2).normal(size=(1, 3, *HW))
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, DEG, lambda img: w, true_sigmoid_grad=True, antialiased=True)
    freeze = dict(J=out["inter"]["J"], color=out["color"])
    lists = (out["ranges"], out["sorted_pid"])
    d_view, d_proj = fo.camera_backward(P, out, cam, HW)

    def loss(view, proj):
        c = dict(cam, view=view, proj=proj)
        return (fo.render_forward_backward(P, aabb, c, HW, TILE, DEG, lambda img: w, antialiased=True, lists=lists,
                                           freeze=freeze)["img"] * w).sum()

    h = 1e-6
    for which, g in (("view", d_view), ("proj", d_proj)):
        for k in range(4):
            for j in range(4):
                if which == "proj" and j == 2:
                    continue
                cp = {n: cam[n].copy() for n in ("view", "proj")}
                cm = {n: cam[n].copy() for n in ("view", "proj")}
                cp[which][0, k, j] += h
                cm[which][0, k, j] -= h
                fd = (loss(cp["view"], cp["proj"]) - loss(cm["view"], cm["proj"])) / (2 * h)
                assert abs(fd - g[k, j]) <= 1e-4 * max(1e-3, abs(fd), abs(g[k, j])), (which, k, j, fd, g[k, j])
    # the antialiasing term is there: without it the view gradient is different
    d_view0, _, _ = co.camera_backward(P, out, cam, HW)
    assert np.abs(d_view - d_view0).max() > 1e-3 * np.abs(d_view).max()


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_off_means_unchanged(dt):
    """antialiased=False: the composition in fused_oracle returns the oracle's own outputs bit for bit.  One oracle thread: the
    raster backward's per-splat sums are run-to-run reproducible only then."""
    hw, tile = (48, 64), (16, 16)
    params, aabb, cam = small_scene(n=800, hw=hw, seed=4)
    if dt == np.float64:
        params, aabb, cam = f64_arrays(params), tuple(a.astype(np.float64) for a in aabb), f64_arrays(cam)
    w = np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(dt)
    nt = oracle.num_threads()
    oracle.set_num_threads(1)
    try:
        a = oracle.render_forward_backward(params, aabb, cam, hw, tile, 3, lambda img: w, true_sigmoid_grad=True)
        b = fo.render_forward_backward(params, aabb, cam, hw, tile, 3, lambda img: w, true_sigmoid_grad=True, antialiased=False)
    finally:
        oracle.set_num_threads(nt)
    for k in ("img", "T", "last", "fragile", "ranges", "sorted_pid", "d_ndc", "d_cov", "d_col", "d_op"):
        assert np.array_equal(a[k], b[k]), k
    for k in PARAM_KEYS:
        assert np.array_equal(a["grads"][k], b["grads"][k]), k
    assert np.all(b["rho"] == 1) and np.all(b["G_aa"] == 0)


def test_rho_range():
    """0 <= rho <= 1 everywhere, rho -> 1 for splats much larger than the filter, rho -> 0 for vanishing ones; the fp32 and
    fp64 factors agree."""
    rng = np.random.default_rng(0)
    M = rng.normal(size=(6, 5000)) * np.exp(rng.uniform(-8, 4, size=5000))
    o = rng.uniform(0, 1, size=(1, 5000))
    oe, rho, _ = aa.antialias_forward(M, o)
    assert np.all(rho >= 0) and np.all(rho <= 1) and np.all(oe <= o)
    smin = np.linalg.svd(M.T.reshape(-1, 3, 2), compute_uv=False).min(axis=1)     # smallest singular value of M
    big = smin > 10
    assert big.any() and np.all(rho[big] > 0.99)
    tiny = np.abs(M).max(axis=0) < 1e-3
    assert tiny.any() and np.all(rho[tiny] < 1e-2)
    # isotropic: rho = s^2 / (s^2 + 0.3)
    for s in (0.1, 0.5, 1.0, 3.0, 30.0):
        Mi = np.array([[s], [0.0], [0.0], [s], [0.0], [0.0]])
        assert abs(aa.antialias_forward(Mi, np.ones((1, 1)))[1][0] - s * s / (s * s + 0.3)) < 1e-12
    _, rho32, _ = aa.antialias_forward(M.astype(np.float32), o.astype(np.float32))
    assert np.abs(rho32 - rho).max() < 1e-4             # det_o cancels in fp32 for needle-like splats: 3.6e-5 at worst here
    # degenerate (rank-1) M: det_o = 0, rho = 0, and the backward gives no gradient
    Md = np.array([[1.0], [2.0], [0.0], [0.0], [0.0], [0.0]])
    oe, rho, f = aa.antialias_forward(Md, np.ones((1, 1)))
    d_o, G = aa.antialias_backward(f, np.ones((1, 1)), np.ones((1, 1)))
    assert rho[0] == 0 and d_o[0, 0] == 0 and np.all(G == 0)


@pytest.mark.parametrize("std_px", [0.35, 0.7, 1.5, 3.0])
def test_integrated_alpha_of_one_splat(std_px):
    """With the compensation, a splat's alpha summed over the pixels equals the integral of the unfiltered Gaussian, o 2 pi
    sqrt(det Sigma) (less the part below the alpha < 1/256 cut-off), at every size.  Without it, a 0.35 px splat covers more than
    three times that."""
    hw = (64, 64)
    P, aabb, cam = single_splat(std_px, hw)
    for on in (True, False):
        out = fo.render_forward_backward(P, aabb, cam, hw, (16, 16), 0, lambda img: np.zeros_like(img), antialiased=on)
        o_act = 1 / (1 + np.exp(-P["opacity"].reshape(1, -1)))
        _, rho, f = aa.antialias_forward(aa.cov_M(out["inter"], cam["view"]), o_act)
        o, oe = float(o_act[0, 0]), float(o_act[0, 0] * rho[0])
        assert abs(math.sqrt(f["det_o"][0]) - std_px ** 2) < 1e-9 * std_px ** 2
        got = float((1 - out["T"]).sum())
        if on:
            want = 2 * math.pi * o * math.sqrt(f["det_o"][0]) * (1 - 1 / (256 * oe))
            print(f"integrated alpha at {std_px} px: {got:.5f}, predicted {want:.5f} ({(got / want - 1) * 100:+.3f} %)")
            assert abs(got / want - 1) < 0.01
        elif std_px == 0.35:
            want = 2 * math.pi * o * math.sqrt(f["det_o"][0]) * (1 - 1 / (256 * oe))
            assert got / want > 3.0


def test_resolution_consistency():
    """Sub-pixel Gaussians rendered at 4x the resolution and average-pooled 4x4 land closer (L1) to the 1x render in the
    antialiased mode than without it: without the compensation the 1x render draws each splat at the filter's size with its
    full opacity, too bright and too thick."""
    lo, k = (48, 64), 4
    hi = (lo[0] * k, lo[1] * k)
    p = scene.make_scene(1500, sh_degree=0, chunk=64, seed=9, log_scale_range=(0.002, 0.006))
    P = {key: p[key] for key in PARAM_KEYS}
    aabb = (p["cluster_origin"], p["cluster_extend"])
    err = {}
    for on in (False, True):
        imgs = {}
        for hw in (lo, hi):
            cam = scene.make_camera(0, 8, hw[1], hw[0])
            out = fo.render_forward_backward(P, aabb, cam, hw, (16, 16), 0, lambda img: np.zeros_like(img), antialiased=on)
            imgs[hw] = out["img"][0].astype(np.float64)
        pooled = imgs[hi].reshape(3, lo[0], k, lo[1], k).mean(axis=(2, 4))
        err[on] = float(np.abs(pooled - imgs[lo]).mean())
    print(f"resolution consistency: L1(pool(4x), 1x) = {err[False]:.5f} off, {err[True]:.5f} antialiased")
    # first run: 0.16378 off, 0.00280 antialiased (ratio 0.017); the margin leaves a factor of six
    assert err[True] < 0.1 * err[False]
