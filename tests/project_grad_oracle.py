"""fp64 reference of the fused projection backward, one Gaussian at a time (torch fp64 on the CPU, autograd for the derivatives).

``record`` maps the raw parameters of each Gaussian and one camera to its record, following project_chain and the mode steps of
litegs_b200/csrc/fused.cu in the kernel's order: (px, py, A, B, C, o_rec, r, g, b, z, n0, n1, n2).  It is written from the
definitions (exp, the 3D filter, the normalised quaternion, MVP, S.R, J, M = T.V3.J, the inverse of M^T M + 0.3 I, the antialiasing
factor, the SH colour, the shortest-axis normal), not from the kernel's fp32 expression order, so an fp32 expression that
cancels shows up as a difference instead of being shared.

Conventions, as the kernel differentiates them (DESIGN.md section 1):
- default: J and the SH view direction are held constant (``fixed`` carries them, computed at the evaluation point);
- exact: neither is held; each clamp of J passes the gradient to the operand it returned, at a tie the position;
- normal: the shortest axis and the facing sign are held constant (the axis is the first index among equal raw log-scales);
- the 3D filter's f is a constant; the opacity is an input as sigma = sigmoid(logit), and the logit gradient is
  d sigma * sigma(1 - sigma) with ``true_sigmoid`` or the reference's d sigma * sigma (DESIGN.md section 7, D3) without.

``backward`` takes the record gradient in the kernel's input form (the 12 raw-moment slots of common.cuh and the normal row),
turns it into record-space gradients with the fp64 record, and returns the per-Gaussian parameter gradients, the camera gradient
and the magnitude |J|^T |g| of every component (J the per-Gaussian Jacobian of the record map), which scales the GPU bars.
"""
import numpy as np
import torch

F64 = torch.float64
REC = ("px", "py", "A", "B", "C", "o", "r", "g", "b", "z", "n0", "n1", "n2")
PARAMS = ("xyz", "scale", "rot", "sh", "sig")
SH_C = (0.28209479177387814, 0.4886025119029199, 1.0925484305920792, 0.31539156525252005, 0.5462742152960396, 0.5900435899266435,
        2.890611442640554, 0.4570457994644658, 0.3731763325901154, 1.445305721320277)


def sh_basis(deg, d):
    """Real SH basis [K,N] at unit directions d [3,N], in the coefficient order of sh.cuh."""
    x, y, z = d
    c = SH_C
    b = [torch.full_like(x, c[0])]
    if deg > 0:
        b += [-c[1] * y, c[1] * z, -c[1] * x]
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        b += [c[2] * x * y, -c[2] * y * z, c[3] * (2 * zz - xx - yy), -c[2] * x * z, c[4] * (xx - yy)]
    if deg > 2:
        b += [-c[5] * y * (3 * xx - yy), c[6] * x * y * z, -c[7] * y * (4 * zz - xx - yy), c[8] * z * (2 * zz - 3 * xx - 3 * yy),
              -c[7] * x * (4 * zz - xx - yy), c[9] * z * (xx - yy), -c[5] * x * (xx - 3 * yy)]
    return torch.stack(b)


def _clamp_pos(t, l, pred=None):
    """max(min(t, l), -l) as fused_J writes it: the gradient goes to the operand returned, at a tie to t.  pred: the two decisions
    (t > l, min(t, l) < -l) to take instead of comparing here."""
    up = t > l if pred is None else pred[0]
    m = torch.where(up, l, t)
    return torch.where(m < -l if pred is None else pred[1], -l, m)


def clamp_decisions_fp32(v, P):
    """fused_J's clamp decisions [4,N] made in fp32, with the limit l = (tz / p) * 1.3 rounded as the kernel rounds it, from the
    fp32-rounded view position (exactly the kernel's under an axis camera, whose view position is the world position)."""
    f = lambda a: np.asarray(a, np.float64).astype(np.float32)
    tz = f(v[2])
    out = []
    for t, p in ((f(v[0]), f(P[:, 0, 0])), (f(v[1]), f(P[:, 1, 1]))):
        l = (tz / p) * np.float32(1.3)
        out += [t > l, np.minimum(t, l) < -l]
    return torch.as_tensor(np.stack(out))


def camera_J(v, P, hw, pred=None):
    """J [N,3,2] of view positions v [4,N] under P [N,4,4] (fused_J); pred: clamp decisions [4,N] (clamp_decisions_fp32) or None."""
    H, W = hw
    p00, p11 = P[:, 0, 0], P[:, 1, 1]
    fx, fy = p00 * W * 0.5, p11 * H * 0.5
    tz = v[2]
    tx = _clamp_pos(v[0], tz / p00 * 1.3, None if pred is None else pred[0:2])
    ty = _clamp_pos(v[1], tz / p11 * 1.3, None if pred is None else pred[2:4])
    rz = 1.0 / torch.where(tz < 1e-2, torch.full_like(tz, 1e-2), tz)
    z0 = torch.zeros_like(tz)
    return torch.stack([torch.stack([fx * rz, z0], -1), torch.stack([z0, fy * rz], -1),
                        torch.stack([-fx * tx * rz * rz, -fy * ty * rz * rz], -1)], 1)


def branches(v, P):
    """The clamp decisions of J in fp64 as bool [4,N]: (x > l, min(x, l) < -l, the same for y)."""
    tz = v[2]
    out = []
    for t, p in ((v[0], P[:, 0, 0]), (v[1], P[:, 1, 1])):
        l = tz / p * 1.3
        out += [t > l, torch.where(t > l, l, t) < -l]
    return torch.stack(out)


def quat_R(qn):
    r, x, y, z = qn
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], -1),
                        torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], -1),
                        torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], -1)], 1)   # [N,3,3]


def shortest_axis(s_raw):
    """normal_frame's axis: argmin of the raw log-scales [3,N], the first index on a tie."""
    ax = (s_raw[1] < s_raw[0]).long()
    return torch.where(s_raw[2] < torch.where(ax == 1, s_raw[1], s_raw[0]), torch.full_like(ax, 2), ax)


def record(th, Vm, P, hw, deg, *, filt=None, aa=False, fixed=None, normal=None, pred=None):
    """Records [13,N] (REC order) and the intermediates.  th: xyz [3,N], scale [3,N] raw log-scales, rot [4,N] raw quaternions,
    sh [K,3,N] (row 0 = sh_0), sig [N] = sigmoid(logit); Vm, P [N,4,4] (one copy per Gaussian, so the camera Jacobian is per
    Gaussian).  filt: f [N] or None.  fixed: dict(J, dirn) held constant, or None for the exact convention.  normal: (ax, sg)
    held constant, or None (n rows are zero).  pred: the clamp decisions of J, or None to make them here in fp64."""
    H, W = hw
    p, q = th["xyz"], th["rot"]
    s = s_unf = torch.exp(th["scale"])
    o = th["sig"]
    if filt is not None:
        f2 = filt * filt
        qf = s * s + f2
        o = o * torch.sqrt(torch.prod(s * s / qf, 0))
        s = torch.sqrt(qf)
    qn = q / torch.sqrt((q * q).sum(0) + 1e-12)
    pt = torch.cat([p, torch.ones_like(p[:1])])
    v = torch.einsum("in,nik->kn", pt, Vm)
    h = torch.einsum("in,nik->kn", v, P)
    R = quat_R(qn)
    J = camera_J(v, P, hw, pred) if fixed is None else fixed["J"]
    VJ = torch.einsum("nak,nkc->nac", Vm[:, :3, :3], J)
    M = torch.einsum("nak,nkc->nac", R * s.T[:, :, None], VJ)
    Sg = torch.einsum("nac,nad->ncd", M, M)
    c00, c01, c11 = Sg[:, 0, 0] + 0.3, Sg[:, 0, 1], Sg[:, 1, 1] + 0.3
    det = c00 * c11 - c01 * c01
    A, B, C = c11 / det, -c01 / det, c00 / det
    r2 = (Sg[:, 0, 0] * Sg[:, 1, 1] - c01 * c01) / det                # rho^2 of the antialiasing factor
    o3 = o
    if aa:
        o = o * torch.sqrt(torch.clamp(r2, min=0.0))
    ndc = h[:2] / h[3]
    px = (ndc[0] + 1) * 0.5 * W - 0.5
    py = (ndc[1] + 1) * 0.5 * H - 0.5
    if fixed is None:
        cc = -torch.einsum("nk,nmk->mn", Vm[:, 3, :3], Vm[:, :3, :3])
        d = p - cc
        dirn = d / torch.sqrt((d * d).sum(0) + 1e-12)
    else:
        dirn = fixed["dirn"]
    col = torch.einsum("kn,kcn->cn", sh_basis(deg, dirn), th["sh"]) + 0.5
    if normal is not None:
        ax, sg = normal
        nw = R[torch.arange(R.shape[0]), ax]                           # [N,3] row ax
        n = sg[None] * torch.einsum("nk,nkj->jn", nw, Vm[:, :3, :3])
    else:
        n = torch.zeros_like(p)
    rec = torch.cat([torch.stack([px, py, A, B, C, o]), col, v[2:3], n])
    return rec, dict(v=v, J=J, dirn=dirn, R=R, M=M, VJ=VJ, c00=c00, c01=c01, c11=c11, r2=r2, s=s, s_unf=s_unf, qn=qn, o3=o3,
                     rn=1.0 / torch.sqrt((q * q).sum(0) + 1e-12))


def record_grad(rec, m, gn=None, depth=False, sc=1.0):
    """Record-space gradient [13,N] of the kernel's input: m [N,12] raw-moment slots (common.cuh), gn [N,4] or None."""
    A, B, C, o = rec[2], rec[3], rec[4], rec[5]
    m = torch.as_tensor(np.asarray(m, np.float64)).T
    g = torch.zeros_like(rec)
    g[0] = -(A * m[0] + B * m[1])
    g[1] = -(B * m[0] + C * m[1])
    g[2], g[3], g[4] = -0.5 * m[2], -m[3], -0.5 * m[4]
    g[5] = torch.where(o > 0, m[8] / torch.where(o > 0, o, torch.ones_like(o)), torch.zeros_like(o))
    g[6:9] = m[5:8]
    if depth:
        g[9] = m[10]
    if gn is not None:
        g[10:13] = torch.as_tensor(np.asarray(gn, np.float64)).T[:3]
    return g * sc


def leaves(params, view, proj):
    """fp64 leaf tensors from numpy: params dict xyz [3,N], scale [3,N], rot [4,N], sh [K,3,N], opacity [N] (logits);
    view, proj [4,4] -> (th, Vm [N,4,4], P [N,4,4])."""
    t = lambda a: torch.as_tensor(np.asarray(a, np.float64)).clone()
    N = np.asarray(params["opacity"]).shape[-1]
    th = {k: t(params[k]).requires_grad_() for k in ("xyz", "scale", "rot", "sh")}
    th["sig"] = torch.sigmoid(t(params["opacity"])).detach().requires_grad_()
    Vm = t(view).reshape(1, 4, 4).repeat(N, 1, 1).requires_grad_()
    P = t(proj).reshape(1, 4, 4).repeat(N, 1, 1).requires_grad_()
    return th, Vm, P


def frozen(th, Vm, P, hw, deg, *, filt=None, aa=False, exact=False, normal=False):
    """The quantities each convention holds constant, taken at the evaluation point: (fixed, normal) for ``record``."""
    with torch.no_grad():
        _, it = record(th, Vm, P, hw, deg, filt=filt, aa=aa)
    fixed = None if exact else dict(J=it["J"].detach(), dirn=it["dirn"].detach())
    nrm = None
    if normal:
        ax = shortest_axis(th["scale"].detach())
        nc = torch.einsum("nk,nkj->jn", it["R"][torch.arange(ax.shape[0]), ax], Vm.detach()[:, :3, :3])
        sg = torch.where((nc * it["v"][:3]).sum(0) > 0, -1.0, 1.0).to(F64)
        nrm = (ax, sg)
    return fixed, nrm


def sigmoid_factor(logit, true_sigmoid):
    """d sigma -> d logit factor: sigma(1 - sigma) formed as sigma * u with u = 1 / (1 + e^x), or the D3 factor sigma."""
    x = torch.as_tensor(np.asarray(logit, np.float64))
    u = 1.0 / (1.0 + torch.exp(x))
    sig = torch.sigmoid(x)
    return sig * u if true_sigmoid else sig


def backward(params, view, proj, hw, deg, m, *, gn=None, filt=None, aa=False, exact=False, depth=False, true_sigmoid=False, sc=1.0):
    """The fp64 projection backward of every Gaussian.  -> dict(grads={xyz, scale, rot, sh, opacity, sig (d sigma)}, cam [2,4,4] (d_view, d_proj),
    mag= the same keys with |J|^T |g| (cam summed over the Gaussians), cam_each [N,2,4,4], mag_cam_each, rec [13,N], g [13,N],
    it= the intermediates), all numpy fp64, and the held quantities (fixed, normal) and J's clamp decisions (pred, exact mode:
    made in fp32 as the kernel makes them)."""
    th, Vm, P = leaves(params, view, proj)
    f = None if filt is None else torch.as_tensor(np.asarray(filt, np.float64))
    fixed, nrm = frozen(th, Vm, P, hw, deg, filt=f, aa=aa, exact=exact, normal=gn is not None)
    with torch.no_grad():
        pred = clamp_decisions_fp32(record(th, Vm, P, hw, deg)[1]["v"].numpy(), P.numpy()) if exact else None
    rec, it = record(th, Vm, P, hw, deg, filt=f, aa=aa, fixed=fixed, normal=nrm, pred=pred)
    g = record_grad(rec.detach(), m, gn, depth, sc)
    ins = [th[k] for k in PARAMS] + [Vm, P]
    grad = [torch.zeros_like(x) for x in ins]
    mag = [torch.zeros_like(x) for x in ins]
    for c in range(rec.shape[0]):
        if not bool((g[c] != 0).any()) or not rec[c].requires_grad:
            continue
        jc = torch.autograd.grad(rec[c].sum(), ins, retain_graph=True, allow_unused=True)
        for i, j in enumerate(jc):
            if j is None:
                continue
            gc = g[c].reshape(*([1] * (j.dim() - 1)), -1) if i < len(PARAMS) else g[c].reshape(-1, 1, 1)
            grad[i] += gc * j
            mag[i] += gc.abs() * j.abs()
    fac = sigmoid_factor(params["opacity"], true_sigmoid)
    n = lambda x: x.detach().numpy()
    grads = dict(xyz=n(grad[0]), scale=n(grad[1]), rot=n(grad[2]), sh=n(grad[3]), opacity=n(grad[4] * fac), sig=n(grad[4]))
    mags = dict(xyz=n(mag[0]), scale=n(mag[1]), rot=n(mag[2]), sh=n(mag[3]), opacity=n(mag[4] * fac), sig=n(mag[4]))
    cam_each = np.stack([n(grad[5]), n(grad[6])], 1)
    mag_cam_each = np.stack([n(mag[5]), n(mag[6])], 1)
    mags["cam"] = mag_cam_each.sum(0)
    return dict(grads=grads, mag=mags, cam=cam_each.sum(0), cam_each=cam_each, mag_cam_each=mag_cam_each, rec=n(rec), g=n(g),
                it={k: n(v) for k, v in it.items()}, fixed=fixed, normal=nrm, pred=pred, proj=np.asarray(proj, np.float64))


def loss(params, view, proj, hw, deg, g, *, filt=None, aa=False, fixed=None, normal=None):
    """L = sum g . rec with the given record gradient g [13,N] and held quantities: the scalar the finite differences differentiate.
    params as in ``leaves`` but with the opacity given as sigma ("sig")."""
    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    th = {k: t(params[k]) for k in PARAMS}
    N = th["sig"].shape[-1]
    Vm = t(view).reshape(-1, 4, 4).expand(N, 4, 4) if np.asarray(view).size == 16 else t(view)
    P = t(proj).reshape(-1, 4, 4).expand(N, 4, 4) if np.asarray(proj).size == 16 else t(proj)
    f = None if filt is None else t(filt)
    with torch.no_grad():
        rec, it = record(th, Vm, P, hw, deg, filt=f, aa=aa, fixed=fixed, normal=normal)
    return (torch.as_tensor(g) * rec).sum(0).numpy(), branches(it["v"], P).numpy()


def fp32_true_sigmoid(x, fixed_form):
    """The kernel's fp32 opacity-logit factor: sig(1 - sig) from sig = 1 - 1/(1 + e^x) (the parent's form), or sig * u."""
    x = np.float32(x)
    u = np.float32(1.0) / (np.float32(1.0) + np.exp(x, dtype=np.float32))
    sig = np.float32(1.0) - u
    return sig * u if fixed_form else sig * (np.float32(1.0) - sig)


# ----------------------------------------------------------------------------------------------------------------------------
# Constructed cases: Gaussians placed directly under an axis camera (tests/util.py) or one rotated camera, each family at the edges
# where the projection backward can go wrong.  Every case is fp32 numpy: xyz [3,N], scale [3,N], rot [4,N], sh [16,3,N],
# opacity [N], filt [N], and the camera (view, proj [4,4]) and image size.
# ----------------------------------------------------------------------------------------------------------------------------
HW = (128, 192)


def _cams():
    from tests import camera_oracle as co
    from tests.util import axis_camera
    H, W = HW
    ax = axis_camera(HW)
    q = np.array([0.9, 0.2, -0.3, 0.25])
    view, proj, _, _ = co.create_viewproj_forward(np.array([[*(q / np.linalg.norm(q)), 0.4, -0.3, 0.5]]),
                                                  np.array([1.0 / np.tan(np.radians(30.0))]), H, W, 0.01, 100.0)
    return dict(axis=(ax["view"][0], ax["proj"][0]), rotated=(view[0].astype(np.float32), proj[0].astype(np.float32)))


def _zq(theta):
    """Quaternion (r, x, y, z) of a rotation by theta about the view axis."""
    return np.array([np.cos(theta / 2), 0.0, 0.0, np.sin(theta / 2)])


def _gaussians(xyz, sig_world, rot, logit, rng, filt=None):
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3).T
    N = xyz.shape[1]
    s = np.asarray(sig_world, np.float64).reshape(N, 3).T
    return dict(xyz=xyz.astype(np.float32), scale=np.log(s).astype(np.float32), rot=np.asarray(rot, np.float64).reshape(N, 4).T.astype(np.float32),
                sh=(0.3 * rng.normal(size=(16, 3, N))).astype(np.float32), opacity=np.asarray(logit, np.float32).reshape(N),
                filt=(0.4 * s.min(0) if filt is None else np.asarray(filt, np.float64)).astype(np.float32))


def _px(cam, z):
    """World units per pixel at depth z under a camera of this module (the x focal length)."""
    view, proj = cam
    return z / (proj[0, 0] * HW[1] * 0.5)


def constructed_cases():
    """name -> dict(params, cam=(view, proj), hw): the families of the projection-backward edge cases."""
    rng = np.random.default_rng(7)
    cams = _cams()
    ax = cams["axis"]
    out = {}
    rq = lambda n: rng.normal(size=(n, 4))
    # J clamp: view-space x/z and y/z just inside, exactly at (in fp32, as fused_J forms the limit) and beyond 1.3/P00 (1.3/P11), on
    # both sides of both axes; the splats are large enough to reach the image
    xyz, s = [], []
    z = np.float32(2.0)
    for k, p in ((0, ax[1][0, 0]), (1, ax[1][1, 1])):
        l32 = float(np.float32(np.float32(z / np.float32(p)) * np.float32(1.3)))
        for sign in (1.0, -1.0):
            for t in (l32 * (1 - 1e-3), l32, l32 * (1 + 1e-3), l32 * 1.6):
                c = [0.05, -0.04, float(z)]
                c[k] = sign * t
                xyz.append(c)
                s.append([0.4, 0.3, 0.35])
    out["j_clamp"] = dict(params=_gaussians(xyz, s, rq(len(xyz)), np.full(len(xyz), 0.5), rng), cam=ax)
    # guarded inverse: screen-sized needles (sigma_long 150-600 px, 0.5 px wide) at 45 and 30 degrees, both sides of the det1 switch
    z = 4.0
    u = _px(ax, z)
    xyz, s, q = [], [], []
    for ang in (np.pi / 4, np.pi / 6, -np.pi / 4):
        for L in (150, 250, 330, 360, 450, 600):
            xyz.append([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), z])
            s.append([L * u, 0.5 * u, 0.5 * u])
            q.append(_zq(ang))
    out["det1"] = dict(params=_gaussians(xyz, s, q, np.full(len(xyz), 1.0), rng), cam=ax)
    # needles of 100:1 and 1000:1 at several angles, sub-pixel splats at the 0.3 px^2 floor, sigma about the image size
    xyz, s, q = [], [], []
    for ratio in (100, 1000):
        for ang in np.radians([0, 10, 30, 45, 60, 90, 135]):
            xyz.append([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), z])
            s.append([20 * u, 20 * u / ratio, 20 * u / ratio])
            q.append(_zq(ang))
    for spx in (0.01, 0.1, 0.3, 0.55, 150, 250):
        xyz.append([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), z])
        s.append([spx * u, spx * u * 1.1, spx * u * 0.9])
        q.append(rng.normal(size=4))
    out["needles_sizes"] = dict(params=_gaussians(xyz, s, q, np.full(len(xyz), 0.3), rng), cam=ax)
    # opacity logits from just above 1/255 up to +16
    logit = np.array([np.log((1 / 255) / (1 - 1 / 255)) + 0.01, -3, -1, 0, 2, 5, 8, 10, 12, 13, 14, 15, 15.5, 16])
    n = len(logit)
    xyz = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.full(n, z)], 1)
    out["opacity"] = dict(params=_gaussians(xyz, np.full((n, 3), 5 * u) * [1, 0.7, 0.5], rq(n), logit, rng), cam=ax)
    # quaternion norms 1e-3 .. 1e3
    norms = np.array([1e-3, 1e-2, 0.1, 1, 10, 100, 1e3, 1e-3, 1e3])
    n = len(norms)
    q = rq(n)
    q = q / np.linalg.norm(q, axis=1, keepdims=True) * norms[:, None]
    xyz = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.full(n, z)], 1)
    out["quaternions"] = dict(params=_gaussians(xyz, np.full((n, 3), 6 * u) * [1, 0.5, 0.25], q, np.full(n, 0.5), rng), cam=ax)
    # log-scales -12 .. +3, with exact ties (the normal mode's first-index rule)
    ls = np.array([[-12, -12, -3], [-5, -5, -5], [0, 0, 1], [3, 1, 1], [-2, -4, -4], [-4, -2, -4], [-4, -4, -2], [-1, -3, -3], [-3, -1, -1],
                   [-12, -8, -6], [1, 2, 3], [-6, -6.5, -6.5], [-2.5, -2.5, -2.5]], np.float64)
    n = len(ls)
    xyz = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.full(n, z)], 1)
    out["log_scales"] = dict(params=_gaussians(xyz, np.exp(ls), rq(n), np.full(n, 0.5), rng), cam=ax)
    # antialiasing factor rho from 1 down below 1e-3 (round splats of 30 px down to 0.003 px, and thin ones)
    xyz, s, q = [], [], []
    for spx in (30, 3, 1, 0.3, 0.1, 0.03, 0.01, 0.003):
        xyz.append([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), z])
        s.append([spx * u, spx * u, spx * u])
        q.append(rng.normal(size=4))
    for w in (0.1, 0.01, 0.001):
        xyz.append([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), z])
        s.append([8 * u, w * u, w * u])
        q.append(_zq(0.4))
    out["antialias"] = dict(params=_gaussians(xyz, s, q, np.full(len(xyz), 1.5), rng), cam=ax)
    # 3D filter f = 0, f ~ s and f >> s
    n = 9
    sw = np.full((n, 3), 3 * u) * [1, 0.6, 0.3]
    f = np.array([0, 0, 0, 0.3 * 3 * u, 0.6 * 3 * u, 3 * u, 30 * u, 100 * u, 300 * u])
    xyz = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.full(n, z)], 1)
    out["filter3d"] = dict(params=_gaussians(xyz, sw, rq(n), np.full(n, 0.5), rng, filt=f), cam=ax)
    # depth just above the 0.2 cull
    zs = np.array([0.2001, 0.2005, 0.201, 0.21, 0.25])
    n = len(zs)
    xyz = np.stack([rng.uniform(-0.02, 0.02, n), rng.uniform(-0.02, 0.02, n), zs], 1)
    out["near_depth"] = dict(params=_gaussians(xyz, np.full((n, 3), 2e-3) * [1, 0.8, 0.6], rq(n), np.full(n, 0.5), rng), cam=ax)
    # the rotated camera: ordinary splats and needles in front of it
    view, proj = cams["rotated"]
    n = 24
    Vi = np.linalg.inv(view.astype(np.float64))
    vs = np.stack([rng.uniform(-1, 1, n), rng.uniform(-0.7, 0.7, n), rng.uniform(1.5, 5, n), np.ones(n)], 1)
    xyz = (vs @ Vi)[:, :3]
    sw = np.exp(rng.uniform(-5, -2, (n, 3)))
    sw[: n // 3, 1:] /= 300
    out["rotated_camera"] = dict(params=_gaussians(xyz, sw, rq(n), rng.uniform(-4, 10, n), rng), cam=cams["rotated"])
    for c in out.values():
        c["hw"] = HW
    return out


def _dq_abs(qn, dT):
    """The quaternion backward of project_backward_kernel with every term taken in absolute value: qn [4,N], dT [N,9] -> [4,N]."""
    r, x, y, z = np.abs(qn)
    t = dT.T
    return np.stack([2 * z * (t[1] + t[3]) + 2 * y * (t[6] + t[2]) + 2 * x * (t[5] + t[7]),
                     2 * y * (t[3] + t[1]) + 2 * z * (t[6] + t[2]) + 2 * r * (t[5] + t[7]) + 4 * x * (t[8] + t[4]),
                     2 * x * (t[3] + t[1]) + 2 * r * (t[6] + t[2]) + 2 * z * (t[5] + t[7]) + 4 * y * (t[8] + t[0]),
                     2 * r * (t[1] + t[3]) + 2 * x * (t[6] + t[2]) + 2 * y * (t[5] + t[7]) + 4 * z * (t[4] + t[0])])


def chain_magnitude(ref, view, hw, *, aa=False, filt=None, normal=False, exact=False):
    """The absolute terms of the kernel's own backward for the scale and rotation gradients, and in exact mode for the position
    gradient's J term -> dict(scale [3,N], rot [4,N], xyz [3,N]).

    The kernel forms these gradients in stages: the conic gradient G = -inv dInv inv (plus the antialiasing term), dM = 2 M G,
    dT = dM (V3 J)^T scaled by s, then ds and the quaternion backward and its normalisation.  Each stage is a few fp32 operations,
    so its rounding is a few ulps of the sum of the absolute values of its terms, and that reaches the output through the later
    stages.  This restates the stages with every product and sum taken in absolute value, from the fp64 intermediates.  Where the
    terms cancel (the rotation gradient of a splat symmetric about an axis, the long-axis scale of a screen-sized needle) the
    gradient and |J|^T |g| are small while these terms are not.  The J term of exact mode follows fused_J_axis_backward the
    same way: dVJ = T^T dM, dJ = V3^T dVJ, then d t, d rz and d tz of each axis, back through V3 to the position."""
    it, g = ref["it"], np.abs(ref["g"])
    A, B, C = np.abs(ref["rec"][2:5])
    N = A.shape[0]
    inv = np.stack([np.stack([A, B], -1), np.stack([B, C], -1)], 1)                    # |inv| [N,2,2]
    dinv = np.stack([np.stack([g[2], g[3] / 2], -1), np.stack([g[3] / 2, g[4]], -1)], 1)
    G = inv @ dinv @ inv
    if aa:
        c00, c01, c11, r2 = it["c00"], it["c01"], it["c11"], it["r2"]
        det_b = np.abs(c00 * c11 - c01 * c01)
        rho = np.sqrt(np.maximum(r2, 0.0))
        d_r2 = np.where(rho > 0, g[5] * np.abs(it["o3"]) / (2 * np.where(rho > 0, rho, 1.0)), 0.0)
        d_do, d_db = d_r2 / det_b, d_r2 * np.abs(r2) / det_b
        a00, a11 = np.abs(c00 - 0.3), np.abs(c11 - 0.3)
        G[:, 0, 0] += d_do * a11 + d_db * np.abs(c11)
        G[:, 1, 1] += d_do * a00 + d_db * np.abs(c00)
        G[:, 0, 1] += np.abs(c01) * (d_do + d_db)
        G[:, 1, 0] += np.abs(c01) * (d_do + d_db)
    dM = 2 * np.abs(it["M"]) @ G                                                          # [N,3,2]
    dT = dM @ np.abs(it["VJ"]).transpose(0, 2, 1)                                        # [N,3,3]
    R, s = np.abs(it["R"]), np.abs(it["s"])
    ds = (R * dT).sum(-1).T                                                              # [3,N]
    dTs = (dT * s.T[:, :, None]).reshape(N, 9)
    sc = s * ds
    if filt is not None:
        s0, f2 = it["s_unf"], np.asarray(filt, np.float64) ** 2
        qf = s0 * s0 + f2
        sc = s0 * ds * s0 / s + g[5] * np.abs(it["o3"]) * f2 / qf
    qn, rn = np.asarray(it["qn"]), np.asarray(it["rn"])
    dq = _dq_abs(qn, dTs)
    rot = rn * (dq + (dq * np.abs(qn)).sum(0) * np.abs(qn))
    if normal:
        ax = np.asarray(ref["normal"][0])
        dnw = np.abs(np.asarray(view, np.float64).reshape(4, 4)[:3, :3]) @ g[10:13]          # [3,N]
        dRn = np.zeros((N, 3, 3))
        dRn[np.arange(N), ax] = dnw.T
        dqn = _dq_abs(qn, dRn.reshape(N, 9))
        rot = rot + rn * (dqn + (dqn * np.abs(qn)).sum(0) * np.abs(qn))
    out = dict(scale=sc, rot=rot, xyz=np.zeros((3, N)))
    if exact:
        V = np.asarray(view, np.float64).reshape(4, 4)
        P = np.asarray(ref["proj"], np.float64)
        dVJ = np.einsum("nar,na,nac->nrc", R, s.T, dM)                                  # sum_a |R[a][r]| s_a dM[a][c]
        aV = np.abs(V[:3, :3])
        dJd = [aV[:, 0] @ dVJ[:, :, 0].T, aV[:, 1] @ dVJ[:, :, 1].T]
        dJ2 = [aV[:, 2] @ dVJ[:, :, 0].T, aV[:, 2] @ dVJ[:, :, 1].T]
        v = it["v"]
        tz = np.maximum(v[2], 1e-2)
        rz = 1.0 / tz
        dt, dtz = [], np.zeros(N)
        for a, (p_, n_) in enumerate(((P[0, 0], hw[1]), (P[1, 1], hw[0]))):
            f = abs(p_) * n_ * 0.5
            l = np.abs(v[2] / p_ * 1.3)
            th = np.minimum(np.abs(v[a]), l)
            dt.append(dJ2[a] * f * rz * rz)
            dtz += rz * rz * (dJd[a] * f + 2 * dJ2[a] * f * th * rz) + dJ2[a] * f * rz * rz * 1.3 / abs(p_)
        out["xyz"] = aV @ np.stack([dt[0], dt[1], dtz])
    return out


def fragile(ref, view, *, exact=False, aa=False):
    """Gaussians whose branch decisions are within rounding of flipping -> bool [N]: rho > 0 (antialiased mode) when det(M^T M) is
    within 4 ulps of its terms, and a J clamp (exact mode) within 4 ulps of its limit unless the camera is an axis camera, whose
    view position is the world position exactly, so that the reference makes the kernel's fp32 decision."""
    it = ref["it"]
    u = 2.0 ** -24
    out = np.zeros(it["r2"].shape, bool)
    if aa:
        a00, a11, c01 = it["c00"] - 0.3, it["c11"] - 0.3, it["c01"]
        out |= np.abs(a00 * a11 - c01 * c01) <= 4 * u * (np.abs(a00 * a11) + c01 * c01)
    V = np.asarray(view, np.float64).reshape(4, 4)
    if exact and not np.array_equal(V, np.eye(4)):
        v, P = it["v"], np.asarray(ref["proj"], np.float64)
        for t, p in ((v[0], P[0, 0]), (v[1], P[1, 1])):
            l = np.abs(v[2] / p * 1.3)
            out |= np.abs(np.abs(t) - l) <= 4 * u * l
    return out
