"""CPU restatement of Mip-Splatting's 3D smoothing filter in numpy (fp32 or fp64), for the filter tests.

The filter (DESIGN.md section 1, "3D smoothing filter") is per-Gaussian data f computed from the training cameras
(``compute_filter``, the order of ``filter_3d_kernel`` in csrc/scene.cu).  It widens each activated scale to s' = sqrt(s^2 + f^2)
and scales the opacity by rho3 = sqrt(prod_k s_k^2 / s'_k^2) (``filter_forward``, the order of ``filter_3d_factor`` in fused.cu).
In tests/fused_oracle.py the filter sits between ``oracle.cull_compact_activate`` and ``oracle.project``, and in the backward
its terms sit between ``createTransformMatrix_backward`` and ``activate_backward``.  The oracle library itself has no filter.

numpy evaluates every elementwise operation below once, correctly rounded and without contraction, in the order written, so the
fp32 filter and the fp32 filtered scale and opacity are the kernels' bit for bit.
"""
import numpy as np

SQRT_02 = {np.float32: np.float32(0.4472136), np.float64: np.float64(np.sqrt(0.2))}


def compute_filter(xyz, views, projs, hws, dt=np.float32):
    """xyz [3, ...] (every slot), views / projs [V,4,4] (row-vector), hws [V,2] (height, width) -> f [...] of dtype dt."""
    dt = np.dtype(dt).type
    shape = np.shape(xyz)[1:]
    p = np.asarray(xyz).reshape(3, -1).astype(dt)
    n = p.shape[1]
    dist = np.full(n, dt(100000.0), dt)
    seen = np.zeros(n, bool)
    focal = dt(0)
    for Vm, P, (h, w) in zip(np.asarray(views).reshape(-1, 4, 4), np.asarray(projs).reshape(-1, 4, 4), np.asarray(hws).reshape(-1, 2)):
        Vm, P, H, W = Vm.astype(dt), P.astype(dt), dt(int(h)), dt(int(w))
        fx = (P[0, 0] * W) * dt(0.5)
        fy = (P[1, 1] * H) * dt(0.5)
        focal = max(focal, fx)
        col = lambda c: ((p[0] * Vm[0, c] + p[1] * Vm[1, c]) + p[2] * Vm[2, c]) + Vm[3, c]
        x, y, z = col(0), col(1), col(2)
        zc = np.maximum(z, dt(0.001))
        u = (x / zc) * fx + W * dt(0.5)
        v = (y / zc) * fy + H * dt(0.5)
        valid = (z > dt(0.2)) & (u >= dt(-0.15) * W) & (u <= dt(1.15) * W) & (v >= dt(-0.15) * H) & (v <= dt(1.15) * H)
        dist = np.where(valid, np.minimum(dist, z), dist)
        seen |= valid
    f = (dist / focal) * SQRT_02[dt]
    f = np.where(seen, f, f[seen].max() if seen.any() else dt(0)).astype(dt)
    return f.reshape(shape)


def filter_forward(s, f, opacity):
    """s [3,N] activated scale, f [N], opacity [1,N] activated -> (s' [3,N], o3 [1,N], factors)."""
    f2 = f * f
    q = s * s
    qf = q + f2
    sp = np.sqrt(qf)
    r = q / qf
    rho3 = np.sqrt((r[0] * r[1]) * r[2])
    o3 = (opacity * rho3).astype(s.dtype)
    return sp, o3, dict(s=s, f2=f2, q=q, qf=qf, sp=sp, r=r, rho3=rho3, o3=o3)
