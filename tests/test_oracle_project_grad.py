"""The fp64 projection-backward reference (tests/project_grad_oracle.py) against finite differences, on the constructed cases.

For each family and mode set, L(theta) = sum g_rec . rec(theta) with the reference's record gradient and its held quantities (J and
the SH direction in the default convention, the normal's axis and sign) is differentiated by fp64 differences in every slot of
every Gaussian's parameters and of its own copy of the camera matrices, and must equal the analytic gradient within 1e-7 of the
component's magnitude |J|^T |g| (plus the differences' own rounding: the record carries kappa ulps, kappa the conditioning of the conic and the
antialiasing factor) at one of three step sizes.  Differences are central unless a step would flip a J clamp decision the reference took (exact
mode, the fp32 tie rule): then they are one-sided, on the side that keeps it.  Both stencils are fourth order.  Also the opacity-logit factor.
"""
import numpy as np
import pytest
import torch

from tests import project_grad_oracle as pg

CASES = pg.constructed_cases()
MODES = {"default": dict(), "exact": dict(exact=True), "all": dict(exact=True, aa=True, f3d=True, depth=True, normal=True)}


def _slots(P, view, proj):
    """(name, index) of every scalar input slot, per Gaussian: xyz, scale, rot, sh, sig, then the camera copies."""
    for k in pg.PARAMS:
        for idx in np.ndindex(np.asarray(P[k]).shape[:-1]):
            yield k, idx
    for k in ("view", "proj"):
        for idx in np.ndindex(4, 4):
            yield k, idx


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("family", list(CASES))
def test_reference_matches_finite_differences(family, mode):
    case = CASES[family]
    kw = MODES[mode]
    deg = 3
    p = case["params"]
    N = p["xyz"].shape[1]
    rng = np.random.default_rng(N + len(mode))
    m = rng.normal(size=(N, 12))
    gn = np.concatenate([rng.normal(size=(N, 3)), np.zeros((N, 1))], 1)
    view, proj = (np.asarray(x, np.float64) for x in case["cam"])
    filt = p["filt"] if kw.get("f3d") else None
    ref = pg.backward(p, view, proj, case["hw"], deg, m, gn=gn if kw.get("normal") else None, filt=filt, aa=kw.get("aa", False),
                      exact=kw.get("exact", False), depth=kw.get("depth", False), true_sigmoid=True)
    base = {k: np.asarray(p[k], np.float64) for k in ("xyz", "scale", "rot", "sh")}
    base["sig"] = torch.sigmoid(torch.as_tensor(np.asarray(p["opacity"], np.float64))).numpy()
    base["view"] = np.repeat(view[None], N, 0)
    base["proj"] = np.repeat(proj[None], N, 0)
    pred = None if ref["pred"] is None else ref["pred"].numpy()
    lkw = dict(filt=filt, aa=kw.get("aa", False), fixed=ref["fixed"], normal=ref["normal"])

    def L(q):
        return pg.loss(q, q["view"], q["proj"], case["hw"], deg, ref["g"], **lkw)

    analytic = dict(ref["grads"], view=ref["cam_each"][:, 0], proj=ref["cam_each"][:, 1])
    mags = dict(ref["mag"], view=ref["mag_cam_each"][:, 0], proj=ref["mag_cam_each"][:, 1])
    worst, one_sided = 0.0, 0
    L0, _ = L(base)
    it = ref["it"]
    det = it["c00"] * it["c11"] - it["c01"] ** 2
    kappa = (np.abs(it["c00"] * it["c11"]) + it["c01"] ** 2) / np.abs(det)              # ulps of the conic per ulp of its inputs
    if kw.get("aa"):
        a00, a11 = it["c00"] - 0.3, it["c11"] - 0.3
        kappa = kappa + (np.abs(a00 * a11) + it["c01"] ** 2) / np.maximum(np.abs(a00 * a11 - it["c01"] ** 2), 1e-300)
    Lab = kappa * np.abs(ref["g"] * ref["rec"]).sum(0)
    for k, idx in _slots(base, view, proj):
        cam = k in ("view", "proj")
        sel = (slice(None),) + idx if cam else idx + (slice(None),)
        x0 = base[k][sel]
        best = None
        for rel in (1e-3, 1e-4, 1e-5):                                       # the best of three steps: truncation vs rounding
            h = rel * np.maximum(np.abs(x0), 1e-2)
            vals = {}
            for s in (-4, -3, -2, -1, 1, 2, 3, 4):
                q = dict(base)
                q[k] = base[k].copy()
                q[k][sel] = x0 + s * h
                vals[s] = L(q)
            f = lambda s: vals[s][0] if s else L0
            fd = (8 * (f(1) - f(-1)) - (f(2) - f(-2))) / (12 * h)           # fourth order
            if pred is not None:
                keep = lambda sg: np.all([np.all(vals[sg * i][1] == pred, 0) for i in (1, 2, 3, 4)], 0)
                plus, minus = keep(1), keep(-1)
                one = lambda sg: sg * (-25 * f(0) + 48 * f(sg) - 36 * f(2 * sg) + 16 * f(3 * sg) - 3 * f(4 * sg)) / (12 * h)
                fd = np.where(plus & minus, fd, np.where(plus, one(1), one(-1)))
                assert np.all(plus | minus), (k, idx)
                if rel == 1e-5:
                    one_sided += int((~(plus & minus)).sum())
            a = analytic[k][sel] if cam else analytic[k][idx]
            mg = mags[k][sel] if cam else mags[k][idx]
            r = np.abs(fd - a) / np.maximum(1e-7 * mg + 1e-15 * Lab / h, 1e-300)   # the stencils' rounding: kappa ulps of sum |g rec| / h
            best = r if best is None else np.minimum(best, r)
        worst = max(worst, float(best.max()))
        assert np.all(best <= 1.0), (k, idx, best.max(), np.argmax(best))
    if family == "j_clamp" and mode != "default":
        assert one_sided > 0, "the clamp ties are differentiated one-sided"


def test_clamp_tie_goes_to_the_position():
    """At x = l exactly (the fp32 limit), the reference's decision is the kernel's: the gradient goes to x, not to the limit."""
    case = CASES["j_clamp"]
    p = case["params"]
    ref = pg.backward(p, *case["cam"], case["hw"], 0, np.ones((16, 12)), exact=True)
    pred = ref["pred"].numpy()
    # per axis and sign: inside, tie, beyond, far beyond
    for k, row in ((0, 0), (1, 2)):
        for sign, base in ((1, 8 * k), (-1, 8 * k + 4)):
            upper, lower = pred[row], pred[row + 1]
            hit = upper if sign > 0 else lower
            assert list(hit[base:base + 4]) == [False, False, True, True], (k, sign, hit[base:base + 4])


def test_opacity_logit_factor():
    """The reference's true-sigmoid factor against the closed form e^-|x| / (1 + e^-|x|)^2, and the fp32 forms: sig * u with
    u = 1 / (1 + e^x) stays within 1e-6 of it from 0 up to x = 16 (and within a few ulps of u / sig below 0), while sig * (1 - sig) from the rounded sig is off by more than 1 %
    at x = 16 (the cancellation the kernels used to have)."""
    x = np.array([-5.5, 0.0, 10.0, 13.0, 15.0, 16.0])
    f = pg.sigmoid_factor(x, True).numpy()
    want = np.exp(-np.abs(x)) / (1 + np.exp(-np.abs(x))) ** 2
    assert np.allclose(f, want, rtol=1e-13, atol=0)
    old = np.array([pg.fp32_true_sigmoid(v, False) for v in x], np.float64)
    new = np.array([pg.fp32_true_sigmoid(v, True) for v in x], np.float64)
    assert np.all(np.abs(new - want)[x >= 0] <= 1e-6 * want[x >= 0])
    assert np.all(np.abs(new - want) <= 4 * 2.0 ** -24 * want * (1 + np.exp(-x)))    # below 0, sig = 1 - u has ulps of u / sig
    assert np.abs(old[-1] - want[-1]) > 1e-2 * want[-1]
    assert np.array_equal(pg.sigmoid_factor(x, False).numpy(), torch.sigmoid(torch.as_tensor(x)).numpy())


def _conic_fp32(p, view, proj, hw):
    """The conic (A, B, C) [3,N] in fp32 numpy by the kernel's formulas (lgs_normalize_quat, lgs_quat_R, lgs_ray_J, lgs_cov_M,
    lgs_cov2d, lgs_inv2x2), for Gaussians in front of an axis camera, whose view position is the world position."""
    f = np.float32
    H, W = hw
    q = np.asarray(p["rot"], f)
    rn = f(1) / np.sqrt((q * q).sum(0) + f(1e-12))
    r, x, y, z = q * rn
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)]),
                  np.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)]),
                  np.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)])]).astype(f)     # [3,3,N]
    s = np.exp(np.asarray(p["scale"], f))
    tx, ty, tz = np.asarray(p["xyz"], f)
    P = np.asarray(proj, f)
    fx, fy = P[0, 0] * f(W) * f(0.5), P[1, 1] * f(H) * f(0.5)
    rz = f(1) / np.maximum(tz, f(1e-2))
    z0 = np.zeros_like(tz)
    J = np.stack([np.stack([fx * rz, z0]), np.stack([z0, fy * rz]), np.stack([-fx * tx * rz * rz, -fy * ty * rz * rz])])   # [3,2,N]
    V3 = np.asarray(view, f)[:3, :3]
    VJ = np.einsum("ak,kcn->acn", V3, J).astype(f)
    M = np.einsum("akn,kcn->acn", (R * s[:, None, :]).astype(f), VJ).astype(f)
    c00 = (M[0, 0] * M[0, 0] + M[1, 0] * M[1, 0] + M[2, 0] * M[2, 0]) + f(0.3)
    c01 = M[0, 0] * M[0, 1] + M[1, 0] * M[1, 1] + M[2, 0] * M[2, 1]
    c11 = (M[0, 1] * M[0, 1] + M[1, 1] * M[1, 1] + M[2, 1] * M[2, 1]) + f(0.3)
    dr = f(1) / (c00 * c11 - c01 * c01)
    return np.stack([c11 * dr, -c01 * dr, c00 * dr]).astype(np.float64)


def test_conversion_magnitude_bounds_the_fp32_conic():
    """conversion_magnitude on the needles: zero wherever c01 is above its own rounding, and for the 0-degree needles, whose
    rotation (1, 0, 0, 0) is exact; non-zero for the needles along the screen's y axis; and above the position error that an fp32
    conic by the kernel's formulas carries through lgs_record_grad's conversion."""
    case = pg.constructed_cases()["needles_sizes"]
    p, (view, proj), hw = case["params"], case["cam"], case["hw"]
    N = p["xyz"].shape[1]
    m = np.random.default_rng(0).normal(size=(N, 12))
    out = pg.conversion_magnitude(p, view, proj, hw, m)
    ang = [0, 10, 30, 45, 60, 90, 135]
    along_y = [i for i in range(14) if ang[i % 7] == 90]
    assert np.array_equal(np.flatnonzero(out["where"]), along_y)
    assert np.all(out["xyz"][:, [0, 7]] == 0.0) and np.all(out["cam_each"][[0, 7]] == 0.0)
    assert np.all(out["xyz"][:2, along_y] > 0.0)
    th, Vm, P = pg.leaves(dict(p, sh=p["sh"][:1]), view, proj)
    rec, _ = pg.record(th, Vm, P, hw, 0)
    jx, = torch.autograd.grad(rec[0].sum(), th["xyz"], retain_graph=True)
    jy, = torch.autograd.grad(rec[1].sum(), th["xyz"])
    d = np.abs(_conic_fp32(p, view, proj, hw) - rec[2:5].detach().numpy())
    dgx = d[0] * np.abs(m[:, 0]) + d[1] * np.abs(m[:, 1])
    dgy = d[1] * np.abs(m[:, 0]) + d[2] * np.abs(m[:, 1])
    err = jx.abs().numpy() * dgx + jy.abs().numpy() * dgy
    assert np.all(err[:, along_y] <= out["xyz"][:, along_y]), (err[:, along_y], out["xyz"][:, along_y])
    assert np.all(err[:, along_y].max(1)[:2] > 0.05 * out["xyz"][:2, along_y].max(1))     # the bound is not vacuous
