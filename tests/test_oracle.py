"""CPU tests of the oracle itself: an independent dense numpy restatement on tiny cases, fp64 finite
differences for every differentiable leaf, fp32-vs-fp64 agreement, and the integer invariants of binning.
(The oracle's pin against the reference's own kernels lives in tests/test_golden.py.)"""
import numpy as np
import pytest

import oracle
from litegs_b200 import scene
from tests.util import f64_arrays, oracle_projected, small_scene, tiny_scene


def _tiny(seed=3):
    return tiny_scene(seed=seed, log_scale_range=(0.05, 0.2))


def test_dense_numpy_rasterizer_agrees():
    """Per-pixel front-to-back compositing written independently in numpy (Appendix A items 12)."""
    hw, tile = (24, 32), (8, 8)
    params, aabb, cam = small_scene(n=300, hw=hw, tile=tile, sh_degree=1, seed=2, log_scale_range=(0.05, 0.15))
    o = oracle_projected(f64_arrays(params), tuple(a.astype(np.float64) for a in aabb), f64_arrays(cam), hw, 1)
    ranges, pid, _, _ = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
    img, T, last, *_ = oracle.rasterize_forward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, hw[0], hw[1], *tile)
    H, W = hw
    gx = W // tile[1]
    mu_x = (o["ndc"][0, 0] + 1) * 0.5 * W - 0.5
    mu_y = (o["ndc"][0, 1] + 1) * 0.5 * H - 0.5
    A, B, C = o["inv_cov2d"][0, 0, 0], o["inv_cov2d"][0, 0, 1], o["inv_cov2d"][0, 1, 1]
    for (y, x) in [(0, 0), (5, 17), (23, 31), (12, 8), (7, 7), (16, 24)]:
        t = (y // tile[0]) * gx + x // tile[1] + 1
        s, e = ranges[0, t], ranges[0, t + 1]
        Tp, col, n = 1.0, np.zeros(3), 0
        if s >= 0:
            for i in pid[0, s:e]:
                if Tp <= 1 / 8192:
                    break
                n += 1
                dx, dy = mu_x[i] - x, mu_y[i] - y
                a = o["opacity"][0, i] * np.exp(-0.5 * (A[i] * dx * dx + 2 * B[i] * dx * dy + C[i] * dy * dy))
                if a < 1 / 256:
                    continue
                a = min(a, 255 / 256)
                col += o["color"][0, :, i] * a * Tp
                Tp *= 1 - a
        assert np.allclose(img[0, :, y, x], np.minimum(col, 1), atol=1e-12)
        assert abs(T[0, 0, y, x] - Tp) < 1e-12 and last[0, 0, y, x] == n


def test_fp64_finite_differences_all_leaves_but_xyz():
    P, aabb, cam = _tiny()
    rng = np.random.default_rng(1)
    w = rng.normal(size=(1, 3, 32, 32))
    run = lambda Q: oracle.render_forward_backward(Q, aabb, cam, (32, 32), (8, 8), 2, lambda img: w, true_sigmoid_grad=True)
    out = run(P)
    ids = out["visible_chunk_id"]
    for name in ("scale", "rot", "sh_0", "sh_rest", "opacity"):
        g = out["grads"][name]
        for _ in range(6):
            idx = tuple(int(rng.integers(0, s)) for s in g.shape)
            full = list(idx); full[-2] = int(ids[idx[-2]]); full = tuple(full)
            h = 1e-6
            Pp = {k: v.copy() for k, v in P.items()}; Pp[name][full] += h
            Pm = {k: v.copy() for k, v in P.items()}; Pm[name][full] -= h
            fd = ((run(Pp)["img"] * w).sum() - (run(Pm)["img"] * w).sum()) / (2 * h)
            assert abs(fd - g[idx]) <= 1e-4 * max(1e-3, abs(fd), abs(g[idx])), (name, fd, g[idx])


def test_fp64_finite_differences_xyz_with_frozen_J_and_dirs():
    """The reference drops d colour/d position and treats J as constant (SURVEY Appendix A items 2, 5, 14):
    the analytic d xyz is the derivative through the NDC mean only.  Check exactly that."""
    P, aabb, cam = _tiny(seed=5)
    hw, tile = (32, 32), (8, 8)
    rng = np.random.default_rng(2)
    w = rng.normal(size=(1, 3, 32, 32))
    out = oracle.render_forward_backward(P, aabb, cam, hw, tile, 2, lambda img: w, true_sigmoid_grad=True)
    base = oracle_projected(P, aabb, cam, hw, 2)

    def loss_with_xyz(xyz_flat):
        vp, ndc = oracle.mvp_transform_forward(xyz_flat, cam["view"], cam["proj"])
        img, *_ = oracle.rasterize_forward(out["sorted_pid"], out["ranges"], ndc, base["inv_cov2d"], base["color"], base["opacity"],
                                           None, hw[0], hw[1], *tile)
        return (np.clip(img, 0, 1) * w).sum()

    g = out["grads"]["xyz"].reshape(3, -1)
    for _ in range(10):
        c, i = int(rng.integers(0, 3)), int(rng.integers(0, g.shape[1]))
        h = 1e-6
        xp = base["xyz"].copy(); xp[c, i] += h
        xm = base["xyz"].copy(); xm[c, i] -= h
        fd = (loss_with_xyz(xp) - loss_with_xyz(xm)) / (2 * h)
        assert abs(fd - g[c, i]) <= 1e-4 * max(1e-3, abs(fd), abs(g[c, i])), (fd, g[c, i])


def test_reference_opacity_gradient_quirk_is_sigma_not_sigma_one_minus_sigma():
    P, aabb, cam = _tiny()
    w = np.ones((1, 3, 32, 32))
    a = oracle.render_forward_backward(P, aabb, cam, (32, 32), (8, 8), 2, lambda img: w, true_sigmoid_grad=False)["grads"]["opacity"]
    b = oracle.render_forward_backward(P, aabb, cam, (32, 32), (8, 8), 2, lambda img: w, true_sigmoid_grad=True)["grads"]["opacity"]
    sig = 1 / (1 + np.exp(-P["opacity"]))
    m = np.abs(b) > 1e-12
    assert np.allclose(a[m] * (1 - sig[m]), b[m], rtol=1e-9)      # SURVEY Q15


def test_fp32_and_fp64_oracles_agree():
    hw, tile = (48, 64), (16, 16)
    params, aabb, cam = small_scene(n=800, hw=hw, seed=4)
    w = np.random.default_rng(0).normal(size=(1, 3, *hw))
    a = oracle.render_forward_backward(params, aabb, cam, hw, tile, 3, lambda img: w.astype(np.float32))
    b = oracle.render_forward_backward(f64_arrays(params), tuple(x.astype(np.float64) for x in aabb), f64_arrays(cam), hw, tile, 3, lambda img: w)
    if a["sorted_pid"].shape == b["sorted_pid"].shape and np.array_equal(a["sorted_pid"], b["sorted_pid"]):
        ok = ~(a["fragile"] | b["fragile"])[:, None, : hw[0], : hw[1]]
        ok = np.broadcast_to(ok, a["img"].shape)
        assert np.abs(a["img"][ok] - b["img"][ok]).max() < 2e-5


@pytest.mark.parametrize("tile", [(8, 16), (16, 16), (12, 16), (8, 8)])
def test_binning_invariants(tile):
    hw = (72, 100)
    params, aabb, cam = small_scene(n=1500, hw=hw, seed=7)
    o = oracle_projected(params, aabb, cam, hw, 3)
    ranges, pid, visible, keys = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
    _, _, alloc = oracle.get_allocate_size(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], hw[0], hw[1], *tile)
    gx, gy = -(-hw[1] // tile[1]), -(-hw[0] // tile[0])
    assert keys.shape[1] == alloc.sum() and (keys > 0).all() and keys.max() <= gx * gy
    assert (np.diff(keys[0]) >= 0).all()                              # sorted by tile
    z = o["view_pos"][0, 2]
    for t in range(1, gx * gy + 1):
        s, e = ranges[0, t], ranges[0, t + 1]
        if s < 0 or e <= s:          # an empty tile right after a populated one carries that tile's end marker
            assert not (keys[0] == t).any()
            continue
        assert (keys[0, s:e] == t).all() and e - s == (keys[0] == t).sum() and (np.diff(z[pid[0, s:e]]) >= 0).all()   # depth ascending inside a tile
    # each splat appears in exactly alloc[i] tiles, and only visible splats appear
    counts = np.bincount(pid[0], minlength=alloc.shape[1])
    assert np.array_equal(counts, alloc[0]) and np.array_equal(visible[0], alloc[0] != 0)
    # tile membership is conservative: the splat centre's tile is listed whenever it is on screen
    px = (o["ndc"][0, 0] + 1) * 0.5 * hw[1] - 0.5; py = (o["ndc"][0, 1] + 1) * 0.5 * hw[0] - 0.5
    for i in np.nonzero(alloc[0])[0][:200]:
        if 0 <= px[i] < hw[1] and 0 <= py[i] < hw[0]:
            t = int(py[i] // tile[0]) * gx + int(px[i] // tile[1]) + 1
            s, e = ranges[0, t], ranges[0, t + 1]
            assert s >= 0 and i in pid[0, s:e]


def test_tile_range_reference_quirk_and_fix():
    keys = np.array([[0, 0, 2, 2, 5, 5, 5]], np.int32)
    q = oracle.tileRange(keys, 8, fix_last=False)
    f = oracle.tileRange(keys, 8, fix_last=True)
    assert q[0, 2] == 2 and q[0, 3] == 4 and q[0, 5] == 4 and q[0, 6] == -1        # last populated tile left open (SURVEY Q3)
    assert f[0, 6] == 7 and np.array_equal(np.delete(q, 6, 1), np.delete(f, 6, 1))


def test_valid_length_limits_every_op():
    hw = (48, 64)
    params, aabb, cam = small_scene(n=600, hw=hw, seed=1)
    o = oracle_projected(params, aabb, cam, hw, 3)
    N = o["xyz"].shape[1]
    vl = np.array([N // 3], np.int32)
    vp, ndc = oracle.mvp_transform_forward(o["xyz"], cam["view"], cam["proj"], vl)
    assert np.all(vp[..., N // 3:] == 0) and np.any(vp[..., : N // 3] != 0)
    _, _, al = oracle.get_allocate_size(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], hw[0], hw[1], 8, 16, vl)
    assert al[:, N // 3:].sum() == 0


def test_scene_conventions():
    cam = scene.make_camera(0, 8, 128, 96)
    o = np.array([[0.0], [0.0], [0.0], [1.0]], np.float32)
    vp, ndc = oracle.mvp_transform_forward(o, cam["view"], cam["proj"])
    assert abs(vp[0, 2, 0] - 3.0) < 1e-5 and abs(ndc[0, 0, 0]) < 1e-5 and abs(ndc[0, 1, 0]) < 1e-5
    p = scene.make_scene(1000, sh_degree=0)
    vis, num, ids = oracle.frustum_culling_aabb(p["cluster_origin"], p["cluster_extend"], cam["frustumplane"])
    assert num[0] == p["cluster_origin"].shape[1]                   # the unit cube is inside the frustum at distance 3


def test_err_square_reference_recurrence_properties():
    """orc_raster_err_square_ref (GR/raster.cu:779-784): with 8x8 tiles a lane owns ONE pixel pair, so the lane-running
    recurrence degenerates to the per-pixel sum of squares; with more pairs per lane it is larger or equal wherever the
    running sums keep their sign, and it never is negative."""
    import oracle
    from tests.util import oracle_projected, small_scene
    hw = (64, 96)
    params, aabb, cam = small_scene(n=1500, hw=hw)
    o = oracle_projected(params, aabb, cam, hw, 3)
    rng = np.random.default_rng(0)
    for tile in ((8, 8), (8, 16), (16, 16)):
        th, tw = tile
        ranges, pid, _, _ = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
        img, T, last, _, _, _ = oracle.rasterize_forward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, hw[0], hw[1], th, tw)
        g = rng.normal(size=img.shape).astype(np.float32)
        args = (pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, T, last, g, None, 1.0, hw[0], hw[1], th, tw)
        e_ref = oracle.rasterize_backward(*args, enable_statistic=True, err_mode="reference")[5]
        e_pix = oracle.rasterize_backward(*args, enable_statistic=True, err_mode="pixel")[5]
        assert e_ref.min() >= 0 and e_pix.max() > 0
        if tile == (8, 8):
            assert np.abs(e_ref - e_pix).max() <= 1e-5 * e_pix.max()
        else:
            assert np.abs(e_ref - e_pix).max() > 1e-3 * e_pix.max()      # a different statistic, not a rounding variant
