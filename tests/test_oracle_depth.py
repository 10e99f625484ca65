"""The depth mode on the CPU (numpy restatement in tests/depth_oracle.py, composed by tests/fused_oracle.py): the gradients of a
loss in D and of a loss in the expected depth ED = D / (1 - T) against fp64 central differences with the tile lists frozen, in the
default convention (J and the SH directions frozen as well) and in the exact mode (nothing else frozen); what the mode leaves
unchanged."""
import numpy as np
import pytest

import oracle
from tests import depth_oracle as dp
from tests import fused_oracle as fo
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


def _losses(kind, u, mask):
    """(loss of (D, T), d_depth_fn) for a loss in D or in ED = D / (1 - T) over the pixels of mask."""
    if kind == "D":
        return (lambda D, T: (u * D).sum()), (lambda D, T: (u, None))
    def loss(D, T):
        return (np.where(mask, u * D / np.where(mask, 1 - T, 1), 0)).sum()
    def grad(D, T):
        a = np.where(mask, 1 / np.where(mask, 1 - T, 1), 0)
        return u * a, u * D * a * a
    return loss, grad


@pytest.mark.parametrize("kind", ["D", "ED"])
@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("deg", [0, 3])
def test_fp64_finite_differences(deg, antialiased, filtered, kind):
    """Colour loss plus a depth loss: scale, rot, opacity (under both sigmoid conventions across the cases) and sh in the default
    convention; xyz and all 16 d_view entries with J and the SH directions frozen (default convention) and unfrozen (exact mode);
    d_proj column 2 stays zero."""
    P, aabb, cam, filt = _scene(deg, filtered)
    rng = np.random.default_rng(7)
    w = rng.normal(size=(1, 3, *HW))
    u = rng.normal(size=(1, 1, *HW))
    true_sigmoid = bool(antialiased)
    kw = dict(antialiased=antialiased, filter_3d=filt)
    base = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_depth=True, **kw)
    mask = (1 - base["T"][..., :HW[0], :HW[1]]) > 0.2
    dloss, dgrad = _losses(kind, u, mask)
    lists = (base["ranges"], base["sorted_pid"])
    ids = base["visible_chunk_id"]
    assert np.abs(base["depth"]).max() > 1.0           # no clamp: depths well above 1 are present

    def run(Q, c=cam, freeze=None):
        o = fo.render_forward_backward(Q, aabb, c, HW, TILE, deg, lambda img: w, render_depth=True, lists=lists, freeze=freeze, **kw)
        return (o["img"] * w).sum() + dloss(o["depth"], o["T"][..., :HW[0], :HW[1]])

    h = 1e-6
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_depth=True, d_depth_fn=dgrad,
                                     true_sigmoid_grad=true_sigmoid, **kw)
    assert np.abs(out["dz"]).max() > 0
    sig = 1 / (1 + np.exp(-P["opacity"]))
    for name in ("scale", "rot", "opacity", "sh_0", "sh_rest"):
        g = out["grads"][name]
        if g.size == 0:
            continue
        for _ in range(3):
            idx = tuple(int(rng.integers(0, s)) for s in g.shape)
            full = list(idx); full[-2] = int(ids[idx[-2]]); full = tuple(full)
            Pp = {k: v.copy() for k, v in P.items()}; Pp[name][full] += h
            Pm = {k: v.copy() for k, v in P.items()}; Pm[name][full] -= h
            fd = (run(Pp) - run(Pm)) / (2 * h)
            want = g[idx] * ((1 - sig[full]) if name == "opacity" and not true_sigmoid else 1.0)
            assert _close(fd, want), (name, idx, fd, want)
    for exact in (False, True):
        o = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_depth=True, d_depth_fn=dgrad,
                                       true_sigmoid_grad=True, exact_grad=exact, **kw)
        freeze = None if exact else dict(J=o["inter"]["J"], color=o["color"])
        g = o["grads"]["xyz"]
        for _ in range(5):
            c, a, s = int(rng.integers(0, 3)), int(rng.integers(0, g.shape[1])), int(rng.integers(0, g.shape[2]))
            Pp = {k: v.copy() for k, v in P.items()}; Pp["xyz"][c, ids[a], s] += h
            Pm = {k: v.copy() for k, v in P.items()}; Pm["xyz"][c, ids[a], s] -= h
            fd = (run(Pp, freeze=freeze) - run(Pm, freeze=freeze)) / (2 * h)
            assert _close(fd, g[c, a, s]), ("xyz", exact, fd, g[c, a, s])
        d_view, d_proj = fo.camera_backward(P, o, cam, HW, sh_degree=deg, exact_grad=exact)
        assert np.all(d_proj[:, 2] == 0)
        for k in range(4):
            for j in range(4):
                cp, cm = cam["view"].copy(), cam["view"].copy()
                cp[0, k, j] += h
                cm[0, k, j] -= h
                fd = (run(P, dict(cam, view=cp), freeze) - run(P, dict(cam, view=cm), freeze)) / (2 * h)
                assert _close(fd, d_view[k, j]), ("view", exact, k, j, fd, d_view[k, j])


def test_depth_of_one_opaque_splat_is_its_z():
    """A single large opaque splat: ED = D / (1 - T) equals its view-space z wherever it was blended, and sum w = 1 - T."""
    P, aabb, cam, _ = _scene(0, False)
    keep = np.zeros(P["opacity"].shape, bool)
    keep[0, 0, 0] = True
    P["opacity"] = np.where(keep, 6.0, -40.0)
    P["scale"] = np.where(keep[None], np.log(0.5), P["scale"])
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, 0, lambda img: np.zeros_like(img), render_depth=True)
    a = 1 - out["T"][..., :HW[0], :HW[1]]
    m = a > 1e-3
    assert m.sum() > 50
    z = out["inter"]["view_pos"][0, 2]
    z0 = z[np.argmax(out["opacity"][0])]
    ed = out["depth"][m] / a[m]
    assert np.abs(ed - z0).max() <= 1e-12 * z0, (ed, z0)


def test_off_and_depth_without_loss_are_the_existing_composition():
    """render_depth=False returns the oracle's own composition's bits where the other modes allow it; depth on with no depth loss
    changes no output either."""
    nt = oracle.num_threads()
    oracle.set_num_threads(1)               # the oracle's raster backward sums are reproducible with one thread
    try:
        _off_and_on_without_loss()
    finally:
        oracle.set_num_threads(nt)


def _off_and_on_without_loss():
    for deg, aa_on, filtered in ((3, False, False), (3, True, True), (0, True, False)):
        P, aabb, cam, filt = _scene(deg, filtered)
        w = np.random.default_rng(3).normal(size=(1, 3, *HW))
        kw = dict(true_sigmoid_grad=True, antialiased=aa_on, filter_3d=filt)
        ref = None if aa_on or filtered else oracle.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w,
                                                                             true_sigmoid_grad=True)
        off = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, **kw)
        on = fo.render_forward_backward(P, aabb, cam, HW, TILE, deg, lambda img: w, render_depth=True, **kw)
        for k in ("img", "T", "last", "ranges", "sorted_pid", "d_ndc", "d_cov", "d_op"):
            assert np.array_equal(on[k], off[k]), k
            if ref is not None:
                assert np.array_equal(ref[k], off[k]), k
        for k in on["grads"]:
            assert np.array_equal(on["grads"][k], off["grads"][k]), k
            if ref is not None:
                assert np.array_equal(ref["grads"][k], off["grads"][k]), k
        assert not np.any(on["dz"])


def test_weights_sum_to_one_minus_T():
    """sum w = 1 - T (the identity that makes D / (1 - T) the expected depth), from the oracle's composite of z = 1."""
    P, aabb, cam, _ = _scene(3, False)
    out = fo.render_forward_backward(P, aabb, cam, HW, TILE, 3, lambda img: np.zeros_like(img), render_depth=True)
    inter = out["inter"]
    ones = np.ones(inter["view_pos"].shape[-1])
    sw = dp.depth_forward(out["sorted_pid"], out["ranges"], inter["ndc"], inter["inv_cov2d"], out["opacity"], ones, *HW, *TILE)
    assert np.abs(sw - (1 - out["T"])).max() <= 1e-12
