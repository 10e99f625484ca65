"""The normal mode on the CPU (numpy restatement in tests/normal_oracle.py, composed by tests/fused_oracle.py): the gradients of a
loss in the colour, the normal N and the expected normal N / (1 - T) against fp64 central differences with the tile lists, the
shortest axes and the facing signs frozen, in the default and the exact convention; the properties of the definition."""
import numpy as np
import pytest

import oracle
from tests import fused_oracle as fo
from tests import normal_oracle as nm
from tests.util import tiny_scene

HW, TILE = (32, 32), (8, 8)
TOL = 1e-4


def _close(fd, g):
    return abs(fd - g) <= TOL * max(1e-3, abs(fd), abs(g))


def _scene(deg, filtered):
    P, aabb, cam = tiny_scene(seed=5, deg=max(deg, 1))
    if deg == 0:
        P["sh_rest"] = P["sh_rest"][:0]
    filt = np.random.default_rng(1).uniform(0.02, 0.12, (1, *P["xyz"].shape[-2:])) if filtered else None
    return P, aabb, cam, filt


def _normal_loss(u, v, mask):
    """Loss in N and in the expected normal EN = N / (1 - T) over mask, and its (dL/dN, dL/dT)."""
    def loss(N, T):
        a = np.where(mask, 1 / np.where(mask, 1 - T, 1), 0)
        return (u * N).sum() + (v * N * a).sum()
    def grad(N, T):
        a = np.where(mask, 1 / np.where(mask, 1 - T, 1), 0)
        return u + v * a, (v * N * a * a).sum(1, keepdims=True)
    return loss, grad


@pytest.mark.parametrize("depth", [False, True])
@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("deg", [0, 3])
def test_fp64_finite_differences(deg, antialiased, filtered, depth):
    """Colour + N + N/(1-T) (+ a depth loss): scale, rot, opacity (both sigmoid conventions across the cases), sh; xyz and all 16
    d_view entries in the default convention (J, SH directions frozen) and the exact one; the normal term adds nothing to d_proj."""
    P, aabb, cam, filt = _scene(deg, filtered)
    rng = np.random.default_rng(7)
    w = rng.normal(size=(1, 3, *HW))
    u, v = rng.normal(size=(1, 3, *HW)), rng.normal(size=(1, 3, *HW))
    uz = rng.normal(size=(1, 1, *HW))
    true_sigmoid = bool(antialiased)
    kw = dict(antialiased=antialiased, filter_3d=filt, render_depth=depth)
    base = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_normal=True, **kw)
    mask = (1 - base["T"][..., :HW[0], :HW[1]]) > 0.2
    nloss, ngrad = _normal_loss(u, v, mask)
    dz_fn = (lambda D, T: (uz, None)) if depth else None
    lists = (base["ranges"], base["sorted_pid"])
    frame = base["frame"]
    ids = base["visible_chunk_id"]
    assert np.abs(base["normal"]).max() > 0.1

    def run(Q, c=cam, freeze=None):
        o = fo.render_forward_backward(Q, aabb, c, HW, TILE, deg, lambda img: w, render_normal=True, lists=lists, freeze=freeze,
                                       normal_freeze=frame, **kw)
        T = o["T"][..., :HW[0], :HW[1]]
        return (o["img"] * w).sum() + nloss(o["normal"], T) + ((uz * o["depth"]).sum() if depth else 0.0)

    h = 1e-6
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_normal=True, d_normal_fn=ngrad,
                                     d_depth_fn=dz_fn, true_sigmoid_grad=true_sigmoid, **kw)
    assert np.abs(out["dn"]).max() > 0
    sig = 1 / (1 + np.exp(-P["opacity"]))
    for name in ("scale", "rot", "opacity", "sh_0", "sh_rest"):
        g = out["grads"][name]
        if g.size == 0:
            continue
        for _ in range(3):
            idx = tuple(int(rng.integers(0, s)) for s in g.shape)
            full = list(idx); full[-2] = int(ids[idx[-2]]); full = tuple(full)
            Pp = {k: x.copy() for k, x in P.items()}; Pp[name][full] += h
            Pm = {k: x.copy() for k, x in P.items()}; Pm[name][full] -= h
            fd = (run(Pp) - run(Pm)) / (2 * h)
            want = g[idx] * ((1 - sig[full]) if name == "opacity" and not true_sigmoid else 1.0)
            assert _close(fd, want), (name, idx, fd, want)
    for exact in (False, True):
        o = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_normal=True, d_normal_fn=ngrad,
                                       d_depth_fn=dz_fn, true_sigmoid_grad=True, exact_grad=exact, **kw)
        freeze = None if exact else dict(J=o["inter"]["J"], color=o["color"])
        g = o["grads"]["xyz"]
        for _ in range(5):
            c, a, s = int(rng.integers(0, 3)), int(rng.integers(0, g.shape[1])), int(rng.integers(0, g.shape[2]))
            Pp = {k: x.copy() for k, x in P.items()}; Pp["xyz"][c, ids[a], s] += h
            Pm = {k: x.copy() for k, x in P.items()}; Pm["xyz"][c, ids[a], s] -= h
            fd = (run(Pp, freeze=freeze) - run(Pm, freeze=freeze)) / (2 * h)
            assert _close(fd, g[c, a, s]), ("xyz", exact, fd, g[c, a, s])
        d_view, d_proj = fo.camera_backward(P, o, cam, HW, sh_degree=deg, exact_grad=exact)
        d_view0, d_proj0 = fo.camera_backward(P, dict(o, dn=None), cam, HW, sh_degree=deg, exact_grad=exact)
        assert np.array_equal(d_proj, np.asarray(d_proj0, np.float64))      # the normal term adds nothing to d_proj
        for k in range(4):
            for j in range(4):
                cp, cm = cam["view"].copy(), cam["view"].copy()
                cp[0, k, j] += h
                cm[0, k, j] -= h
                fd = (run(P, dict(cam, view=cp), freeze) - run(P, dict(cam, view=cm), freeze)) / (2 * h)
                assert _close(fd, d_view[k, j]), ("view", exact, k, j, fd, d_view[k, j])


def _opaque_tilted(P, rot):
    keep = np.zeros(P["opacity"].shape, bool)
    keep[0, 0, 0] = True
    Q = {k: x.copy() for k, x in P.items()}
    Q["opacity"] = np.where(keep, 6.0, -40.0)
    Q["scale"][:, 0, 0] = np.log([0.5, 0.4, 0.05])           # axis 2 is the shortest
    Q["rot"][:, 0, 0] = rot
    return Q


def test_opaque_tilted_splat_gives_its_normal():
    """One large opaque tilted splat: N / (1 - T) equals its n wherever it was blended, |n| = 1 and n faces the camera."""
    P, aabb, cam, _ = _scene(0, False)
    Q = _opaque_tilted(P, np.array([0.9, 0.3, -0.2, 0.1]))
    out = fo.render_forward_backward(Q, aabb, cam, HW, TILE, 0, lambda img: np.zeros_like(img), render_normal=True)
    a = 1 - out["T"][..., :HW[0], :HW[1]]
    m = a[0, 0] > 1e-3
    assert m.sum() > 50
    fr = out["frame"]
    i0 = int(np.argmax(out["opacity"][0]))
    n0 = fr["n"][:, i0]
    assert fr["a"][i0] == 2
    en = out["normal"][0][:, m] / a[0, 0][m]
    assert np.abs(en - n0[:, None]).max() <= 1e-12
    v = out["inter"]["view_pos"][0, :3, i0]
    assert float(n0 @ v) <= 0 and abs(np.linalg.norm(n0) - 1) <= 1e-6
    assert abs(n0[1]) > 0.05 or abs(n0[0]) > 0.05                   # tilted: not the optical axis


def test_rotation_about_the_shortest_axis_leaves_N_unchanged():
    """Rotating a splat about its own shortest axis changes R's other rows but not row a, so N is unchanged."""
    P, aabb, cam, _ = _scene(0, False)
    q = np.array([0.9, 0.3, -0.2, 0.1]); q /= np.linalg.norm(q)
    R = nm.quat_R(q[:, None])[:, 0].reshape(3, 3)
    ax = R[2]                                                        # world direction of the shortest axis (axis 2)
    t = 0.7
    qa = np.array([np.cos(t / 2), *(np.sin(t / 2) * ax)])
    # composing with a rotation about the axis itself: R' = R Ra^T keeps the row R[2] (R[2] Ra^T = R[2])
    r1, v1 = q[0], q[1:]
    r2, v2 = qa[0], -qa[1:]
    q2 = np.array([r1 * r2 - v1 @ v2, *(r1 * v2 + r2 * v1 + np.cross(v1, v2))])
    R2 = nm.quat_R(q2[:, None])[:, 0].reshape(3, 3)
    if not np.allclose(R2[2], R[2], atol=1e-12):                     # the other composition order
        q2 = np.array([r2 * r1 - v2 @ v1, *(r2 * v1 + r1 * v2 + np.cross(v2, v1))])
        R2 = nm.quat_R(q2[:, None])[:, 0].reshape(3, 3)
    assert np.allclose(R2[2], R[2], atol=1e-12) and not np.allclose(R2[0], R[0], atol=1e-3)
    o1 = fo.render_forward_backward(_opaque_tilted(P, q), aabb, cam, HW, TILE, 0, lambda img: np.zeros_like(img), render_normal=True)
    o2 = fo.render_forward_backward(_opaque_tilted(P, q2), aabb, cam, HW, TILE, 0, lambda img: np.zeros_like(img), render_normal=True)
    # the ellipse turns with the long axes, so compare the expected normal where both renders blended the splat (it is the only
    # one the alpha test lets through)
    a1, a2 = 1 - o1["T"][0, 0, :HW[0], :HW[1]], 1 - o2["T"][0, 0, :HW[0], :HW[1]]
    m = (a1 > 1e-3) & (a2 > 1e-3)
    assert m.sum() > 20
    e1, e2 = o1["normal"][0][:, m] / a1[m], o2["normal"][0][:, m] / a2[m]
    assert np.abs(e1 - e2).max() <= 1e-10


def test_unit_normals_and_tie_rule():
    """|n| = 1 within 1e-6 for every Gaussian (fp32 restatement); the first index wins a tie of the raw log-scales."""
    rng = np.random.default_rng(2)
    q = rng.normal(size=(4, 2000)).astype(np.float32)
    s = rng.normal(size=(3, 2000)).astype(np.float32)
    s[:, :10] = 0.5
    s[2, 10:20] = s[1, 10:20]
    V = np.eye(4, dtype=np.float32)
    V[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    v = rng.normal(size=(3, 2000)).astype(np.float32)
    fr = nm.normal_frame(s, q, V, v)
    assert np.abs(np.linalg.norm(fr["n"].astype(np.float64), axis=0) - 1).max() <= 1e-6
    assert np.all(fr["a"][:10] == 0)
    assert np.all(fr["a"][10:20] == np.where(s[1, 10:20] < s[0, 10:20], 1, 0))
    assert np.all((fr["n"] * v).sum(0) <= 1e-6)


def test_fp32_sign_is_the_stated_expression():
    """The fp32 facing sign of the ordered restatement equals a scalar float32 evaluation of
    ((n_c0 v0 + n_c1 v1) + n_c2 v2) > 0, with n_c[j] = (n_w0 V[0][j] + n_w1 V[1][j]) + n_w2 V[2][j], including near-zero cases."""
    rng = np.random.default_rng(4)
    n = 3000
    q = rng.normal(size=(4, n)).astype(np.float32)
    s = rng.normal(size=(3, n)).astype(np.float32)
    V = np.eye(4, dtype=np.float32)
    V[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    fr0 = nm.normal_frame(s, q, V, np.ones((3, n), np.float32))
    # positions almost in each splat's tangent plane, so that many dot products sit within a few ulps of zero
    t = rng.normal(size=(3, n)).astype(np.float32)
    nc = fr0["nc"]
    v = (t - nc * (nc * t).sum(0)).astype(np.float32) + rng.normal(size=(3, n)).astype(np.float32) * np.float32(1e-7)
    fr = nm.normal_frame(s, q, V, v)
    f = np.float32
    near = 0
    for i in range(n):
        nw = [f(x) for x in fr["nw"][:, i]]
        c = [f(f(f(nw[0] * V[0, j]) + f(nw[1] * V[1, j])) + f(nw[2] * V[2, j])) for j in range(3)]
        d = f(f(f(c[0] * v[0, i]) + f(c[1] * v[1, i])) + f(c[2] * v[2, i]))
        assert fr["sg"][i] == (f(-1) if d > 0 else f(1)), i
        near += abs(float(d)) < 1e-6
    assert near > 100


def test_translation_identity():
    """n does not depend on the camera translation: with a normal loss, sum d xyz = V3x3 . d_view[3, 0:3] (fp64, 1e-9)."""
    P, aabb, cam, _ = _scene(3, False)
    rng = np.random.default_rng(9)
    w, u = rng.normal(size=(1, 3, *HW)), rng.normal(size=(1, 3, *HW))
    for exact in (False, True):
        o = fo.render_forward_backward(P, aabb, cam, HW, TILE, 3, lambda img: w, render_normal=True,
                                       d_normal_fn=lambda N, T: (u, None), true_sigmoid_grad=True, exact_grad=exact)
        d_view, _ = fo.camera_backward(P, o, cam, HW, sh_degree=3, exact_grad=exact)
        V3 = np.asarray(cam["view"], np.float64).reshape(4, 4)[:3, :3]
        gsum = o["grads"]["xyz"].astype(np.float64).reshape(3, -1).sum(1)
        assert np.abs(gsum - V3 @ d_view[3, :3]).max() <= 1e-9 * max(1.0, np.abs(gsum).max()), (exact, gsum, V3 @ d_view[3, :3])


def test_off_and_normals_without_loss_are_the_existing_composition():
    """render_normal=False returns the oracle's own composition's bits where the other modes allow it; normals on with no normal
    loss change no output either."""
    nt = oracle.num_threads()
    oracle.set_num_threads(1)
    try:
        for deg, aa_on, filtered, depth in ((3, False, False, False), (3, True, True, True), (0, True, False, True)):
            P, aabb, cam, filt = _scene(deg, filtered)
            w = np.random.default_rng(3).normal(size=(1, 3, *HW))
            kw = dict(true_sigmoid_grad=True, antialiased=aa_on, filter_3d=filt, render_depth=depth)
            ref = None if aa_on or filtered or depth else oracle.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w,
                                                                                          true_sigmoid_grad=True)
            off = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, **kw)
            on = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_normal=True, **kw)
            for k in ("img", "T", "last", "ranges", "sorted_pid", "d_ndc", "d_cov", "d_op"):
                assert (ref is None or np.array_equal(ref[k], off[k])) and np.array_equal(on[k], off[k]), k
            for k in on["grads"]:
                assert (ref is None or np.array_equal(ref["grads"][k], off["grads"][k])) and np.array_equal(on["grads"][k], off["grads"][k]), k
            assert not np.any(on["dn"])
    finally:
        oracle.set_num_threads(nt)
