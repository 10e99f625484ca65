"""CPU restatement of the exact gradient mode in numpy (fp32 or fp64), for the exact-gradient tests.

The mode (DESIGN.md section 1, "Exact gradient mode") adds two terms to the position gradient and to the camera gradient that
the default convention drops:

- through the ray-space Jacobian J (``lgs_ray_J`` in projection.cuh, ``jacobianRayspace`` of the oracle): dM = 2 M G with G the whole
  d cov2d (the antialiased term included), dVJ = T^T dM, dJ[k][c] = sum_a V3[a][k] dVJ[a][c], and ``J_backward`` takes dJ00,
  dJ11, dJ20, dJ21 back to the view-space position and to P00, P11, one clamp branch at a time;
- through the SH view direction: with d = p - cc, n = 1 / sqrt(|d|^2 + 1e-12) and u = d n, g_u = sum_k w_k d b_k / du with
  w_k = sum_c sh[k][c] dcol_c, and g_d = n (g_u - u (u . g_u)); d xyz += g_d and d cc = -g_d.

tests/fused_oracle.py adds both terms to the xyz gradient and to the camera gradient.  The oracle library itself has no such
mode.
"""
import numpy as np

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def fused_J(v, p00, p11, H, W):
    """(J00, J11, J20, J21) of lgs_ray_J for view-space positions v [3,N] (tx, ty, tz)."""
    tx, ty, tz = v
    fx, fy = p00 * W * 0.5, p11 * H * 0.5
    lx, ly = tz / p00 * 1.3, tz / p11 * 1.3
    tx = np.maximum(np.minimum(tx, lx), -lx)
    ty = np.maximum(np.minimum(ty, ly), -ly)
    rz = 1.0 / np.maximum(tz, 1e-2)
    rz2 = rz * rz
    return fx * rz, fy * rz, -fx * tx * rz2, -fy * ty * rz2


def _axis_backward(p, n, t, tz, rz, rz2, dJd, dJ2):
    f = p * n * 0.5
    l = tz / p * 1.3
    m = np.minimum(t, l)
    th = np.maximum(m, -l)
    df = dJd * rz - dJ2 * th * rz2
    dth = -dJ2 * f * rz2
    drz = dJd * f - 2.0 * dJ2 * f * th * rz
    lo = m < -l                                     # the lower clamp returned -l
    dm = np.where(lo, 0.0, dth)
    dl = np.where(lo, -dth, 0.0)
    hi = t > l                                      # the upper clamp returned l
    dt = np.where(hi, 0.0, dm)
    dl = dl + np.where(hi, dm, 0.0)
    return dt, dl * 1.3 / p, df * n * 0.5 - dl * l / p, drz


def J_backward(v, p00, p11, H, W, dJ00, dJ11, dJ20, dJ21):
    """Back-propagation through lgs_ray_J as written -> (dv [3,N], d p00 [N], d p11 [N]).  Each clamp passes the gradient to the
    operand it returned, the position at a tie; below the 0.01 depth floor rz is constant."""
    tx, ty, tz = v
    rz = 1.0 / np.maximum(tz, 1e-2)
    rz2 = rz * rz
    dtx, dtz_x, dp00, drz_x = _axis_backward(p00, W, tx, tz, rz, rz2, dJ00, dJ20)
    dty, dtz_y, dp11, drz_y = _axis_backward(p11, H, ty, tz, rz, rz2, dJ11, dJ21)
    dtz = dtz_x + dtz_y - np.where(tz < 1e-2, 0.0, rz2 * (drz_x + drz_y))
    return np.stack([dtx, dty, dtz]), dp00, dp11


def sh_basis(deg, u):
    """lgs_sh_basis: u [3,N] -> b [(deg+1)^2, N]."""
    x, y, z = u
    b = [np.full_like(x, SH_C0)]
    if deg > 0:
        b += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
    if deg > 2:
        b += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4 * zz - xx - yy),
              SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
              SH_C3[6] * x * (xx - 3 * yy)]
    return np.stack(b)


def sh_basis_grad(deg, u, w):
    """sum_k w[k] d b_k / du (lgs_sh_basis_grad): u [3,N], w [(deg+1)^2, N] -> [3,N]."""
    x, y, z = u
    g = np.zeros_like(u)
    if deg > 0:
        g[0] -= SH_C1 * w[3]; g[1] -= SH_C1 * w[1]; g[2] += SH_C1 * w[2]
    if deg > 1:
        C20, C22, C24 = SH_C2[0], SH_C2[2], SH_C2[4]
        g[0] += C20 * (y * w[4] - z * w[7]) + 2 * x * (C24 * w[8] - C22 * w[6])
        g[1] += C20 * (x * w[4] - z * w[5]) - 2 * y * (C22 * w[6] + C24 * w[8])
        g[2] += -C20 * (y * w[5] + x * w[7]) + 4 * C22 * z * w[6]
    if deg > 2:
        C30, C31, C32, C33, C34, C35, C36 = SH_C3
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        g[0] += (6 * C30 * xy * w[9] + C31 * yz * w[10] - 2 * C32 * xy * w[11] - 6 * C33 * xz * w[12]
                 + C34 * (4 * zz - 3 * xx - yy) * w[13] + 2 * C35 * xz * w[14] + 3 * C36 * (xx - yy) * w[15])
        g[1] += (3 * C30 * (xx - yy) * w[9] + C31 * xz * w[10] + C32 * (4 * zz - xx - 3 * yy) * w[11] - 6 * C33 * yz * w[12]
                 - 2 * C34 * xy * w[13] - 2 * C35 * yz * w[14] - 6 * C36 * xy * w[15])
        g[2] += (C31 * xy * w[10] + 8 * C32 * yz * w[11] + C33 * (6 * zz - 3 * xx - 3 * yy) * w[12] + 8 * C34 * xz * w[13]
                 + C35 * (xx - yy) * w[14])
    return g


def camera_center(Vm):
    """lgs_camera_center: cc_m = sum_k (-V[3][k]) V[m][k]."""
    return -(Vm[:3, :3] @ Vm[3, :3])


def direction_backward(deg, p, Vm, sh, dcol):
    """g_d [3,N] for positions p [3,N], the view matrix Vm [4,4], the coefficients sh [(deg+1)^2, 3, N] and the colour gradient
    dcol [3,N]."""
    d = p - camera_center(Vm)[:, None]
    n = 1.0 / np.sqrt((d * d).sum(axis=0) + 1e-12)
    u = d * n
    w = np.einsum("kcn,cn->kn", sh, dcol)
    gu = sh_basis_grad(deg, u, w)
    return n * (gu - u * (u * gu).sum(axis=0))
