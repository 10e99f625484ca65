"""CPU restatement of the antialiased mode in numpy (fp32 or fp64), for the antialiasing tests.

The mode (DESIGN.md section 1) scales each splat's opacity by rho = sqrt(det(M^T M) / det(M^T M + 0.3 I)), M = T.V3x3.J, so
that the filtered splat's integrated alpha equals the unfiltered Gaussian's.  Its forward and backward sit between the oracle's
stages: after ``oracle.project`` and before binning, and in the backward between the raster gradient and the projection /
activation backward; tests/fused_oracle.py puts them there.  The oracle library itself has no antialiased mode.

numpy evaluates every elementwise operation below once, correctly rounded and without contraction, in the order written: the
same order as ``antialias_factor`` in fused.cu, so the fp32 opacity here is the kernel's bit for bit given the same M.
"""
import numpy as np


def cov_M(inter, view_matrix):
    """M = T.V3x3.J of every Gaussian [6,N] (M[a*2+c]), in the oracle's summation order (oracle_core.h: cov_M)."""
    T, J = inter["T"], inter["J"][0]
    dt = T.dtype
    Vm = np.asarray(view_matrix, dt).reshape(4, 4)
    VJ = [[None] * 2 for _ in range(3)]
    for a in range(3):
        for c in range(2):
            t = np.zeros(T.shape[-1], dt)
            for k in range(3):
                t = t + Vm[a, k] * J[k, c]
            VJ[a][c] = t
    M = np.zeros((6, T.shape[-1]), dt)
    for a in range(3):
        for c in range(2):
            t = np.zeros(T.shape[-1], dt)
            for k in range(3):
                t = t + T[a, k] * VJ[k][c]
            M[a * 2 + c] = t
    return M


def antialias_forward(M, opacity):
    """(o_eff, rho, factors) from M [6,N] and the activated opacity [1,N]."""
    dt = M.dtype.type
    a00 = (M[0] * M[0] + M[2] * M[2]) + M[4] * M[4]
    a01 = (M[0] * M[1] + M[2] * M[3]) + M[4] * M[5]
    a11 = (M[1] * M[1] + M[3] * M[3]) + M[5] * M[5]
    c00, c11 = a00 + dt(0.3), a11 + dt(0.3)
    a01sq = a01 * a01
    det_o = a00 * a11 - a01sq
    det_b = c00 * c11 - a01sq
    r2 = det_o / det_b
    rho = np.sqrt(np.maximum(r2, dt(0)))
    o_eff = (opacity * rho).astype(M.dtype)
    return o_eff, rho, dict(a00=a00, a01=a01, a11=a11, c00=c00, c11=c11, det_o=det_o, det_b=det_b, r2=r2, rho=rho)


def antialias_backward(f, opacity, g):
    """g = d o_eff [1,N] -> (d o [1,N] (the activated opacity), G [2,2,N] (d of the filtered 2D covariance))."""
    rho = f["rho"]
    live = rho > 0
    safe = np.where(live, rho, 1)
    d_r2 = np.where(live, g[0] * opacity[0] / (2 * safe), 0)
    d_det_o = d_r2 / f["det_b"]
    d_det_b = -d_r2 * f["r2"] / f["det_b"]
    d_a01_half = -f["a01"] * (d_det_o + d_det_b)
    G = np.zeros((2, 2, rho.shape[0]), g.dtype)
    G[0, 0] = d_det_o * f["a11"] + d_det_b * f["c11"]
    G[1, 1] = d_det_o * f["a00"] + d_det_b * f["c00"]
    G[0, 1] = G[1, 0] = d_a01_half
    return (g * rho).astype(g.dtype), G
