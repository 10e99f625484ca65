"""Depth-normal consistency on the CPU (numpy restatement in tests/depth_normal_oracle.py): analytic planes, fp64 central
differences of every D, T and N element, the invariances and the masks of the definition, and the gradient through the render
(tests/fused_oracle.py) against fp64 central differences of the parameters."""
import numpy as np
import pytest

from tests import depth_normal_oracle as dn
from tests import fused_oracle as fo
from tests.util import tiny_scene


def _plane_case(H, W, fx, fy, normal, dist, rng, alpha_min=0.5):
    """ED of the plane {X : n.X = -dist} (n unit, camera-facing) seen through the pixel rays, and D = alpha ED with alpha varying
    per pixel above alpha_min -> (D, T, proj).  The rays are those of the focal lengths the f32 projection matrix holds."""
    P = dn.proj_matrix(fx, fy, H, W).astype(np.float64)
    fx, fy = P[0, 0, 0] * W / 2, P[0, 1, 1] * H / 2
    rx, ry = (np.arange(W) + 0.5 - W / 2) / fx, (np.arange(H) + 0.5 - H / 2) / fy      # pixel centres of the rasteriser
    r = np.stack(np.broadcast_arrays(rx[None, :], ry[:, None], np.ones((H, W))))
    ed = -dist / np.einsum("k,khw->hw", normal, r)
    assert np.all(ed > 0)
    alpha = rng.uniform(alpha_min + 0.05, 1.0, (H, W))
    return alpha * ed, 1 - alpha, P


PLANES = [(np.array([0.0, 0.0, -1.0]), 2.0), (np.array([0.3, -0.2, -1.0]), 5.0), (np.array([-0.6, 0.4, -1.0]), 0.7),
          (np.array([0.1, 0.8, -1.0]), 40.0)]
CAMERAS = [(24, 32, 30.0, 28.0), (37, 53, 60.0, 60.0), (64, 48, 150.0, 120.0)]


@pytest.mark.parametrize("H,W,fx,fy", CAMERAS)
def test_analytic_planes(H, W, fx, fy):
    """n_d is the plane's camera-facing unit normal within 1e-12 at every interior pixel, and L = 0 when N is that normal times any
    positive per-pixel factor."""
    rng = np.random.default_rng(H)
    for nrm, dist in PLANES:
        nrm = nrm / np.linalg.norm(nrm)
        D, T, P = _plane_case(H, W, fx, fy, nrm, dist, rng)
        N = nrm[:, None, None] * rng.uniform(0.01, 3.0, (1, H, W))
        o = dn.forward_backward(D, T, N, P, weight=0.7, dtype=np.float64)
        assert o["mask"][1:-1, 1:-1].all() and not o["mask"][0].any() and not o["mask"][:, -1].any()
        err = np.abs(o["nd"] - nrm[:, None, None])[:, o["mask"]].max()
        assert err < 1e-12, err
        assert abs(o["loss"]) < 1e-12 and np.abs(o["l"]).max() < 1e-12


def _random_case(rng, H=12, W=16, dt=np.float64):
    """A smooth random depth field with every threshold kept away: alpha in (0.6, 0.95), |N| in (0.3, 1.7)."""
    P = dn.proj_matrix(20.0, 18.0, H, W).astype(np.float64)
    y, x = np.mgrid[0:H, 0:W]
    ed = 3.0 + 0.4 * np.sin(0.5 * x + 0.2) * np.cos(0.3 * y) + 0.05 * x + 0.1 * rng.normal(size=(H, W))
    alpha = rng.uniform(0.6, 0.95, (H, W))
    N = rng.normal(size=(3, H, W))
    N *= rng.uniform(0.3, 1.7, (1, H, W)) / np.linalg.norm(N, axis=0, keepdims=True)
    return (alpha * ed).astype(dt), (1 - alpha).astype(dt), N.astype(dt), P


def test_fp64_central_differences():
    """Every D, T and N element's gradient matches fp64 central differences (relative 1e-7 of the largest gradient)."""
    rng = np.random.default_rng(0)
    D, T, N, P = _random_case(rng)
    w, up = 0.7, 1.3
    o = dn.forward_backward(D, T, N, P, weight=w, upstream=up, dtype=np.float64)
    assert o["lmask"].sum() == (12 - 2) * (16 - 2)
    L = lambda D_, T_, N_: up * dn.loss_only(D_, T_, N_, P, weight=w)
    for name, X, G in (("D", D, o["dD"]), ("T", T, o["dT"]), ("N", N, o["dN"])):
        fd = np.zeros_like(X)
        for idx in np.ndindex(X.shape):
            h = 1e-6 * max(1.0, abs(X[idx]))
            Xp, Xm = X.copy(), X.copy()
            Xp[idx] += h
            Xm[idx] -= h
            args_p = dict(D=D, T=T, N=N); args_p[name] = Xp
            args_m = dict(D=D, T=T, N=N); args_m[name] = Xm
            fd[idx] = (L(args_p["D"], args_p["T"], args_p["N"]) - L(args_m["D"], args_m["T"], args_m["N"])) / (2 * h)
        err = np.abs(fd - G).max() / np.abs(G).max()
        assert err < 1e-7, (name, err)


def test_invariances():
    """Scaling D by k > 0 leaves L unchanged and sum D dD = 0; scaling N_p leaves L unchanged and N_p . dN_p = 0; 0 <= l_p <= 2;
    a pixel's own depth does not enter its n_d."""
    rng = np.random.default_rng(1)
    D, T, N, P = _random_case(rng, 20, 24)
    o = dn.forward_backward(D, T, N, P, dtype=np.float64)
    for k in (0.01, 3.0, 250.0):
        assert abs(dn.loss_only(k * D, T, N, P) - o["loss"]) < 1e-14
    assert abs((D * o["dD"]).sum()) < 1e-12 * np.abs(D * o["dD"]).sum()
    s = rng.uniform(0.1, 10.0, (1, *D.shape))
    assert abs(dn.loss_only(D, T, N * s, P) - o["loss"]) < 1e-14
    assert np.abs((N * o["dN"]).sum(0)).max() < 1e-14 * np.abs(o["dN"]).max() * np.abs(N).max() * 10
    assert o["l"].min() >= 0 and o["l"].max() <= 2 and o["l"].max() > 1
    D2 = D.copy()
    D2[7, 9] *= 1.5
    assert np.array_equal(dn.forward_backward(D2, T, N, P, dtype=np.float64)["nd"][:, 7, 9], o["nd"][:, 7, 9])


def test_masks():
    """Border pixels, pixels with alpha <= alpha_min at themselves or a neighbour and pixels with |N| <= 1e-6 contribute nothing;
    an H or W below 3 gives L = 0 and zero gradients."""
    rng = np.random.default_rng(2)
    D, T, N, P = _random_case(rng, 20, 24)
    T[5, 6] = 0.5                     # alpha = 0.5: not above alpha_min
    T[12, 3] = 0.9
    N[:, 15, 15] = 1e-7
    o = dn.forward_backward(D, T, N, P, dtype=np.float64)
    lm = o["lmask"]
    assert not lm[0].any() and not lm[-1].any() and not lm[:, 0].any() and not lm[:, -1].any()
    for y, x in ((5, 6), (12, 3)):
        for dy, dx in ((0, 0), (0, 1), (0, -1), (1, 0), (-1, 0)):
            assert not lm[y + dy, x + dx] and o["l"][y + dy, x + dx] == 0
        assert lm[y + 1, x + 1]           # a diagonal neighbour is not part of the stencil
    assert o["mask"][15, 15] and not lm[15, 15] and np.all(o["dN"][:, 15, 15] == 0)
    assert lm.sum() == 18 * 22 - 5 - 5 - 1
    for H, W in ((2, 9), (9, 2), (1, 1), (2, 2)):
        Dm, Tm, Nm, Pm = _random_case(rng, H, W)
        om = dn.forward_backward(Dm, Tm, Nm, Pm, dtype=np.float64)
        assert om["loss"] == 0 and not np.any(om["dD"]) and not np.any(om["dT"]) and not np.any(om["dN"]) and not np.any(om["nd"])


def test_fp32_restatement_follows_fp64():
    """The fp32 order (differences written as (ED+ - ED-) r- + ED+ (r+ - r-)) keeps n_d within 1e-3 of fp64 on a distant, slightly
    tilted plane at 1080 x 1920, where differences of the points themselves would cancel."""
    H, W = 1080, 1920
    rng = np.random.default_rng(3)
    nrm = np.array([0.05, -0.1, -1.0]); nrm /= np.linalg.norm(nrm)
    D, T, P = _plane_case(H, W, 1600.0, 1600.0, nrm, 30.0, rng)
    o = dn.forward_backward(D.astype(np.float32), T.astype(np.float32), None, P, dtype=np.float32)
    assert o["mask"][1:-1, 1:-1].all()
    err = np.abs(o["nd"] - nrm[:, None, None].astype(np.float32))[:, o["mask"]].max()
    assert err < 1e-3, err


HW, TILE = (32, 32), (8, 8)


def test_gradient_through_the_render():
    """The consistency loss on the fused path's D, T and N (SH degree 0, tile lists, shortest axes, facing signs and J frozen): the
    xyz, scale, rot and opacity gradients match fp64 central differences within 1e-4."""
    P, aabb, cam = tiny_scene(seed=5, deg=1, n=96, log_scale_range=(0.1, 0.35))
    P["sh_rest"] = P["sh_rest"][:0]
    P["opacity"] = np.abs(P["opacity"]) + 1.0
    am, w = 0.3, 2.0
    zero = lambda img: np.zeros_like(img)
    base = fo.render_forward_backward(P, aabb, cam, HW, TILE, 0, zero, render_depth=True, render_normal=True, true_sigmoid_grad=True)
    lists, frame, J = (base["ranges"], base["sorted_pid"]), base["frame"], base["inter"]["J"]
    alpha = 1 - base["T"][0, 0, :HW[0], :HW[1]]
    assert np.abs(alpha - am).min() > 1e-4                    # no mask decision within reach of a perturbation

    def terms(o):
        return dn.forward_backward(o["depth"], o["T"][..., :HW[0], :HW[1]], o["normal"], cam["proj"], weight=w, alpha_min=am,
                                   dtype=np.float64)

    t0 = terms(base)
    assert t0["lmask"].sum() > 100, t0["lmask"].sum()
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, 0, zero, render_depth=True, render_normal=True, true_sigmoid_grad=True,
                                     lists=lists, normal_freeze=frame, freeze=dict(J=J),
                                     d_depth_fn=lambda D_, T_: (t0["dD"][None, None], t0["dT"][None, None]),
                                     d_normal_fn=lambda N_, T_: (t0["dN"][None], None))

    def run(Q):
        o = fo.render_forward_backward(Q, aabb, cam, HW, TILE, 0, zero, render_depth=True, render_normal=True, lists=lists,
                                       normal_freeze=frame, freeze=dict(J=J))
        t = terms(o)
        assert np.array_equal(t["lmask"], t0["lmask"])
        return t["loss"]

    rng = np.random.default_rng(4)
    ids = base["visible_chunk_id"]
    h = 1e-6
    for name in ("xyz", "scale", "rot", "opacity"):
        g = out["grads"][name]
        assert np.abs(g).max() > 0
        for _ in range(6):
            idx = tuple(int(rng.integers(0, s)) for s in g.shape)
            full = list(idx); full[-2] = int(ids[idx[-2]]); full = tuple(full)
            Pp = {k: x.copy() for k, x in P.items()}; Pp[name][full] += h
            Pm = {k: x.copy() for k, x in P.items()}; Pm[name][full] -= h
            fd = (run(Pp) - run(Pm)) / (2 * h)
            assert abs(fd - g[idx]) <= 1e-4 * max(1e-3 * np.abs(g).max(), abs(fd), abs(g[idx])), (name, idx, fd, g[idx])
