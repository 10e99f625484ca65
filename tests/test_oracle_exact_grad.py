"""The exact gradient mode on the CPU (numpy restatement in tests/exact_grad_oracle.py, composed by tests/fused_oracle.py): the J
backward and the SH direction backward on their own against fp64 central differences, the position and camera gradients of a
render against central differences of the real function (only the tile lists frozen; J and the colours follow the perturbation),
the default convention failing that check on the same scenes, and what the mode leaves unchanged."""
import numpy as np
import pytest

import oracle
from litegs_b200 import scene
from tests import camera_oracle as co
from tests import exact_grad_oracle as ex
from tests import fused_oracle as fo
from tests.util import PARAM_KEYS, tiny_scene

HW, TILE = (32, 32), (8, 8)
TOL = 1e-4


def _close(fd, g):
    return abs(fd - g) <= TOL * max(1e-3, abs(fd), abs(g))


def _ratio(fd, g):
    """How many times the tolerance a gradient misses a finite difference by."""
    return abs(fd - g) / (TOL * max(1e-3, abs(fd), abs(g)))


def _J_points(rng):
    """View-space points inside the clamp, on both clamp branches, and on both sides of the 0.01 depth floor, each at least 20 %
    away from a kink, with per-point focal terms."""
    n = 200
    p00 = rng.uniform(0.8, 2.5, 5 * n)
    p11 = rng.uniform(0.8, 2.5, 5 * n)
    tz = np.concatenate([rng.uniform(0.3, 6.0, 3 * n), rng.uniform(0.002, 0.008, n), rng.uniform(0.0125, 0.05, n)])
    lx, ly = tz / p00 * 1.3, tz / p11 * 1.3
    frac = lambda lo, hi, k: rng.uniform(lo, hi, k) * rng.choice([-1, 1], k)
    fx = np.concatenate([frac(0, 0.8, n), rng.uniform(1.2, 3, n), -rng.uniform(1.2, 3, n), frac(0, 3, 2 * n)])
    fy = np.concatenate([frac(0, 0.8, n), -rng.uniform(1.2, 3, n), rng.uniform(1.2, 3, n), frac(0, 3, 2 * n)])
    fx = np.where(np.abs(np.abs(fx) - 1) < 0.2, fx * 1.5, fx)
    fy = np.where(np.abs(np.abs(fy) - 1) < 0.2, fy * 1.5, fy)
    return np.stack([fx * lx, fy * ly, tz]), p00, p11


def test_J_backward_matches_finite_differences():
    rng = np.random.default_rng(0)
    v, p00, p11 = _J_points(rng)
    H, W = 1080, 1920
    dJ = rng.normal(size=(4, v.shape[1]))
    # fused_J is elementwise: perturb every point at once and difference the per-point losses
    loss = lambda v_, a, b: sum(dJ[i] * j for i, j in enumerate(ex.fused_J(v_, a, b, H, W)))
    dv, dp00, dp11 = ex.J_backward(v, p00, p11, H, W, *dJ)
    worst = 0.0
    for which in range(5):
        h = 1e-7 * (v[2] if which < 3 else 1.0)
        vp, vm, ap, am, bp, bm = v.copy(), v.copy(), p00.copy(), p00.copy(), p11.copy(), p11.copy()
        if which < 3:
            vp[which] += h; vm[which] -= h
        elif which == 3:
            ap += h; am -= h
        else:
            bp += h; bm -= h
        fd = (loss(vp, ap, bp) - loss(vm, am, bm)) / (2 * h)
        g = dv[which] if which < 3 else dp00 if which == 3 else dp11
        err = np.abs(fd - g) / np.maximum(1.0, np.abs(fd))
        assert err.max() <= 1e-5, (which, int(err.argmax()), fd[err.argmax()], g[err.argmax()])
        worst = max(worst, err.max())
    # the clamp branches have no tx (ty) and no P00 (P11) term
    n = 200
    assert np.all(dv[0, n:3 * n] == 0) and np.all(dv[1, n:3 * n] == 0)
    print(f"J backward vs fp64 central differences: {worst:.1e} relative")


@pytest.mark.parametrize("deg", [1, 2, 3])
def test_direction_backward_matches_finite_differences(deg):
    rng = np.random.default_rng(deg)
    n = 300
    K = (deg + 1) ** 2
    p = rng.uniform(-2, 2, (3, n))
    Vm = scene.look_at_view_matrix(np.array([0.3, -0.5, -4.0]), target=(0.1, 0.2, 0.3)).astype(np.float64)
    sh = rng.normal(size=(K, 3, n))
    dcol = rng.normal(size=(3, n))
    cc = ex.camera_center(Vm)

    def loss(p_):
        d = p_ - cc[:, None]
        u = d / np.sqrt((d * d).sum(axis=0) + 1e-12)
        return (np.einsum("kn,kcn->cn", ex.sh_basis(deg, u), sh) * dcol).sum()

    g = ex.direction_backward(deg, p, Vm, sh, dcol)
    h = 1e-6
    for i in range(n):
        for k in range(3):
            pp, pm = p.copy(), p.copy()
            pp[k, i] += h; pm[k, i] -= h
            fd = (loss(pp) - loss(pm)) / (2 * h)
            assert abs(fd - g[k, i]) <= 1e-7 * max(1.0, abs(fd)), (i, k, fd, g[k, i])
    # the basis restated here is the oracle's: the colours of cull_compact_activate come out of it
    u = rng.normal(size=(3, 5)); u /= np.linalg.norm(u, axis=0)
    assert ex.sh_basis(deg, u).shape == (K, 5)


def _scene(deg, filtered):
    P, aabb, cam = tiny_scene(seed=5, deg=max(deg, 1))
    if deg == 0:
        P["sh_rest"] = P["sh_rest"][:0]
    filt = np.random.default_rng(1).uniform(0.02, 0.12, (1, *P["xyz"].shape[-2:])) if filtered else None
    return P, aabb, cam, filt


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("deg", [0, 3])
def test_fp64_finite_differences_xyz_and_camera(deg, antialiased, filtered):
    """d xyz, all 16 d_view entries and d_proj (column 2 excepted: NDC z is not used) of the exact mode equal fp64 central
    differences of the render with only the tile lists frozen.  The default convention misses the same differences by at least
    ten times the tolerance somewhere."""
    P, aabb, cam, filt = _scene(deg, filtered)
    rng = np.random.default_rng(2)
    w = rng.normal(size=(1, 3, *HW))
    kw = dict(antialiased=antialiased, filter_3d=filt)
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, true_sigmoid_grad=True, exact_grad=True, **kw)
    off = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, true_sigmoid_grad=True, **kw)
    lists = (out["ranges"], out["sorted_pid"])
    ids = out["visible_chunk_id"]

    def loss(Q, c=cam):
        return (fo.render_forward_backward(Q, aabb, c, HW, TILE, deg, lambda img: w, lists=lists, **kw)["img"] * w).sum()

    h = 1e-6
    worst = miss = 0.0
    g, g0 = out["grads"]["xyz"], off["grads"]["xyz"]
    for _ in range(10):
        c, a, s = int(rng.integers(0, 3)), int(rng.integers(0, g.shape[1])), int(rng.integers(0, g.shape[2]))
        Pp = {k: v.copy() for k, v in P.items()}; Pp["xyz"][c, ids[a], s] += h
        Pm = {k: v.copy() for k, v in P.items()}; Pm["xyz"][c, ids[a], s] -= h
        fd = (loss(Pp) - loss(Pm)) / (2 * h)
        assert _close(fd, g[c, a, s]), ("xyz", fd, g[c, a, s])
        worst, miss = max(worst, _ratio(fd, g[c, a, s])), max(miss, _ratio(fd, g0[c, a, s]))
    d_view, d_proj = fo.camera_backward(P, out, cam, HW, exact_grad=True)
    v0, p0 = fo.camera_backward(P, off, cam, HW)
    for which, gc, gd in (("view", d_view, v0), ("proj", d_proj, p0)):
        for k in range(4):
            for j in range(4):
                if which == "proj" and j == 2:
                    assert gc[k, j] == 0
                    continue
                cp = {n: cam[n].copy() for n in ("view", "proj")}
                cm = {n: cam[n].copy() for n in ("view", "proj")}
                cp[which][0, k, j] += h
                cm[which][0, k, j] -= h
                fd = (loss(P, dict(cam, **cp)) - loss(P, dict(cam, **cm))) / (2 * h)
                assert _close(fd, gc[k, j]), (which, k, j, fd, gc[k, j])
                worst, miss = max(worst, _ratio(fd, gc[k, j])), max(miss, _ratio(fd, gd[k, j]))
    print(f"deg {deg} aa {antialiased} filter {filtered}: exact within {worst:.3f} x the tolerance, the default convention "
          f"misses by {miss:.0f} x")
    assert miss >= 10


def test_mode_changes_only_xyz_and_keeps_the_translation_identity():
    """Exact on vs off: the same image, lists and scale, rot, opacity, sh gradients (the mode only adds to d xyz);
    sum_i d xyz_i = V3x3 . d_view[3, :3] to 1e-9 in fp64, with the antialiased mode and the filter on as well.  With the other
    modes off as well, off is the oracle's own composition and camera_oracle's camera gradient, bit for bit."""
    for deg, aa_on, filtered in ((3, False, False), (3, True, True), (1, True, False)):
        P, aabb, cam, filt = _scene(deg, filtered)
        w = np.random.default_rng(3).normal(size=(1, 3, *HW))
        kw = dict(true_sigmoid_grad=True, antialiased=aa_on, filter_3d=filt)
        nt = oracle.num_threads()
        oracle.set_num_threads(1)               # the oracle's raster backward sums are reproducible with one thread
        try:
            on = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, exact_grad=True, **kw)
            off = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, **kw)
            ref = None if aa_on or filtered else oracle.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w,
                                                                                 true_sigmoid_grad=True)
        finally:
            oracle.set_num_threads(nt)
        for k in ("img", "ranges", "sorted_pid", "T", "last"):
            assert np.array_equal(on[k], off[k]), k
        for k in ("scale", "rot", "opacity", "sh_0", "sh_rest"):
            assert np.array_equal(on["grads"][k], off["grads"][k]), k
        assert not np.array_equal(on["grads"]["xyz"], off["grads"]["xyz"])
        d_view, _ = fo.camera_backward(P, on, cam, HW, exact_grad=True)
        s = on["grads"]["xyz"].reshape(3, -1).sum(axis=1)
        rhs = cam["view"][0, :3, :3] @ d_view[3, :3]
        assert np.abs(s).max() > 0
        assert np.abs(s - rhs).max() <= 1e-9 * np.abs(s).max(), (s, rhs)
        # off: the oracle's own composition, unchanged
        if ref is not None:
            for k in ("img", "T", "last", "ranges", "sorted_pid", "d_ndc", "d_cov", "d_op"):
                assert np.array_equal(ref[k], off[k]), k
            for k in PARAM_KEYS:
                assert np.array_equal(ref["grads"][k], off["grads"][k]), k
            v0, p0 = fo.camera_backward(P, off, cam, HW)
            va, pa, _ = co.camera_backward(P, ref, cam, HW)
            assert np.array_equal(v0, va) and np.array_equal(p0, pa)


def test_level_a_render_refuses_the_flag():
    """The op-by-op render() has no exact gradient mode: it refuses pp.exact_grad rather than return the frozen-J gradients."""
    from litegs_b200 import render
    from litegs_b200.arguments import PipelineParams
    with pytest.raises(RuntimeError, match="exact_grad"):
        render.render(*([None] * 10), 3, (8, 8), PipelineParams(exact_grad=True))
