"""Numpy restatement of the depth-normal consistency term (DESIGN.md section 1, "Depth-normal consistency"; csrc/geometry.cu), in
fp32 with the kernel's order of operations or in fp64.

``forward_backward(D, T, N, proj, ...)`` takes one view's D, T [H,W] (or [1,1,H,W]) and N [3,H,W] (or [1,3,H,W], or None) and
returns the normal n_d, the masks, the per-pixel terms, the loss and its gradients.
"""
import numpy as np


def intrinsics(proj, H, W, dt=np.float32):
    """(fx, fy) = ((P[0][0] W) 0.5, (P[1][1] H) 0.5) in dt, as lgs_ray_J."""
    P = np.asarray(proj, np.float64).reshape(4, 4).astype(dt)
    return (P[0, 0] * dt(W)) * dt(0.5), (P[1, 1] * dt(H)) * dt(0.5)


def rays(H, W, fx, fy, dt=np.float32):
    """(rx [W], ry [H]): r(u, v) = (rx[u], ry[v], 1), rx[u] = ((u + 0.5) - W/2) / fx."""
    rx = ((np.arange(W).astype(dt) + dt(0.5)) - dt(0.5) * dt(W)) / dt(fx)
    ry = ((np.arange(H).astype(dt) + dt(0.5)) - dt(0.5) * dt(H)) / dt(fy)
    return rx.astype(dt), ry.astype(dt)


def proj_matrix(fx, fy, H, W, znear=0.01, zfar=100.0):
    """A row-vector projection matrix with P[0][0] = 2 fx / W and P[1][1] = 2 fy / H, f32[1,4,4]."""
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1] = 2 * fx / W, 2 * fy / H
    P[2, 2], P[2, 3] = zfar / (zfar - znear), 1.0
    P[3, 2] = -zfar * znear / (zfar - znear)
    return P[None].astype(np.float32)


def _cross(p, q):
    return np.stack([p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]])


def _dot(p, q):
    return p[0] * q[0] + p[1] * q[1] + p[2] * q[2]


def forward_backward(D, T, N, proj, weight=1.0, upstream=1.0, alpha_min=0.5, dtype=np.float32):
    """-> dict(nd [3,H,W], mask [H,W] (where n_d is defined), lmask [H,W] (where l_p counts), l [H,W], loss (fp64 sum of l times
    weight / (H W)), and with N: dD, dT [H,W], dN [3,H,W] = upstream * dL/d(D, T, N), the masks held constant)."""
    dt = dtype
    D = np.asarray(D).reshape(np.shape(D)[-2:]).astype(dt)
    T = np.asarray(T).reshape(np.shape(T)[-2:]).astype(dt)
    H, W = D.shape
    fx, fy = intrinsics(proj, H, W, dt)
    rx, ry = rays(H, W, fx, fy, dt)
    hx, hy = dt(2) / fx, dt(2) / fy
    am = dt(alpha_min)
    alpha = dt(1) - T
    valid = alpha > am
    with np.errstate(divide="ignore", invalid="ignore"):
        E = np.where(valid, D / np.where(valid, alpha, dt(1)), dt(0)).astype(dt)
    out = dict(nd=np.zeros((3, H, W), dt), mask=np.zeros((H, W), bool), lmask=np.zeros((H, W), bool), l=np.zeros((H, W), dt), loss=0.0)
    if N is not None:
        out.update(dD=np.zeros((H, W), dt), dT=np.zeros((H, W), dt), dN=np.zeros((3, H, W), dt))
    if H < 3 or W < 3:
        return out
    c_ = (slice(1, H - 1), slice(1, W - 1))
    eL, eR, eT, eB = E[1:-1, :-2], E[1:-1, 2:], E[:-2, 1:-1], E[2:, 1:-1]
    m = valid[c_] & valid[1:-1, :-2] & valid[1:-1, 2:] & valid[:-2, 1:-1] & valid[2:, 1:-1]
    rxL, rxc = rx[None, :-2], rx[None, 1:-1]
    ryc, ryT = ry[1:-1, None], ry[:-2, None]
    dx, dy = eR - eL, eB - eT
    a = np.stack([dx * rxL + eR * hx, dx * ryc, dx])                 # (ED+ - ED-) r- + ED+ (r+ - r-)
    b = np.stack([dy * rxc, dy * ryT + eB * hy, dy])
    c = _cross(b, a)
    cc = _dot(c, c)
    m &= cc > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        ic = np.where(m, dt(1) / np.sqrt(np.where(m, cc, dt(1))), dt(0)).astype(dt)
    n = (c * ic).astype(dt)
    out["nd"][:, 1:-1, 1:-1] = n
    out["mask"][c_] = m
    if N is None:
        return out
    N = np.asarray(N).reshape(3, H, W).astype(dt)
    q = N[:, 1:-1, 1:-1]
    nn = _dot(q, q)
    lm = m & (nn > dt(1e-12))
    iN = np.where(lm, dt(1) / np.sqrt(np.where(lm, nn, dt(1))), dt(0)).astype(dt)
    mq = q * iN
    cs = _dot(n, mq)
    l = np.where(lm, dt(1) - cs, dt(0)).astype(dt)
    out["lmask"][c_] = lm
    out["l"][c_] = l
    out["loss"] = float(weight) * float(l.astype(np.float64).sum()) / (H * W)
    s = dt(float(weight) * float(upstream) / (H * W))
    sN, sc = s * iN, s * ic
    out["dN"][:, 1:-1, 1:-1] = np.where(lm, sN * (cs * mq - n), dt(0))
    gc = np.where(lm, sc * (cs * n - mq), dt(0)).astype(dt)
    GA, GB = np.zeros((3, H + 2, W + 2), dt), np.zeros((3, H + 2, W + 2), dt)     # one zero pixel around the image
    GA[:, 2:-2, 2:-2] = _cross(gc, b)
    GB[:, 2:-2, 2:-2] = _cross(a, gc)
    G = (GA[:, 1:-1, :-2] - GA[:, 1:-1, 2:]) + (GB[:, :-2, 1:-1] - GB[:, 2:, 1:-1])
    gE = (G[0] * rx[None, :] + G[1] * ry[:, None]) + G[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        dD = np.where(valid, gE / np.where(valid, alpha, dt(1)), dt(0)).astype(dt)
    out["dD"] = dD
    out["dT"] = (dD * E).astype(dt)
    return out


def loss_only(D, T, N, proj, weight=1.0, alpha_min=0.5, dtype=np.float64):
    return forward_backward(D, T, N, proj, weight=weight, alpha_min=alpha_min, dtype=dtype)["loss"]

