"""CPU restatement of the normal mode in numpy (fp32 or fp64), for the normal tests.

The mode (DESIGN.md section 1, "Normals") renders N = sum_i w_i n_i with the colour's blend weights w_i and n_i the camera-facing
view-space normal of Gaussian i's shortest axis.  That is the oracle's own composite with the colour replaced by n / 2: |n_k| <= 1
keeps the composite below the min(c, 1) clamp, and scaling by 2 is exact.  Both use the same weights, so the backward is the sum
of the colour backward and the same backward of that normal-as-colour image; its colour gradient is dL/dn (times 1/2), which then
reaches the rotations (row a of the rotation-matrix gradient) and the camera (d view[k][j] += n_w[k] dn_c[j]).
tests/fused_oracle.py renders N and adds that backward.  The oracle library itself has no normal mode.
"""
import numpy as np

import oracle


def quat_R(qn):
    """Rotation matrix rows [9,N] of unit quaternions qn [4,N] (r, x, y, z), laid out as lgs_quat_R."""
    r, x, y, z = qn
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y),
                     2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x),
                     2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)])


def quat_R_backward(qn, dR):
    """d qn [4,N] of a gradient dR [9,N] of quat_R's rows (the derivative of quat_R)."""
    r, x, y, z = qn
    d = dR
    return np.stack([2 * z * (d[1] - d[3]) + 2 * y * (d[6] - d[2]) + 2 * x * (d[5] - d[7]),
                     2 * y * (d[3] + d[1]) + 2 * z * (d[6] + d[2]) + 2 * r * (d[5] - d[7]) - 4 * x * (d[8] + d[4]),
                     2 * x * (d[3] + d[1]) + 2 * r * (d[6] - d[2]) + 2 * z * (d[5] + d[7]) - 4 * y * (d[8] + d[0]),
                     2 * r * (d[1] - d[3]) + 2 * x * (d[6] + d[2]) + 2 * y * (d[5] + d[7]) - 4 * z * (d[4] + d[0])])


def shortest_axis(s_raw):
    """a [N] = argmin_k of the raw log-scales [3,N], the first index winning a tie."""
    a = np.where(s_raw[1] < s_raw[0], 1, 0)
    return np.where(s_raw[2] < np.where(a == 1, s_raw[1], s_raw[0]), 2, a)


def normal_frame(s_raw, q_raw, view, v, freeze=None):
    """-> dict(a, qn, rn, R, nw [3,N], nc [3,N], sg [N], n [3,N]) in the dtype of the inputs.  view: [4,4] (row-vector), v: the
    view-space positions [>=3,N].  n_c and the facing test are evaluated as the kernel does: single-rounded products and sums in
    the order ((n_w0 V[0][j] + n_w1 V[1][j]) + n_w2 V[2][j]) and ((n_c0 v0 + n_c1 v1) + n_c2 v2).  freeze: dict(a, sg) of an
    earlier frame, whose discrete decisions are then kept (finite differences)."""
    dt = q_raw.dtype
    rn = (1 / np.sqrt((q_raw * q_raw).sum(0) + dt.type(1e-12))).astype(dt)
    qn = (q_raw * rn).astype(dt)
    R = quat_R(qn).astype(dt)
    a = shortest_axis(s_raw) if freeze is None else freeze["a"]
    nw = np.stack([np.choose(a, (R[k], R[3 + k], R[6 + k])) for k in range(3)]).astype(dt)
    V = np.asarray(view, dt).reshape(4, 4)
    nc = np.stack([(nw[0] * V[0, j] + nw[1] * V[1, j]) + nw[2] * V[2, j] for j in range(3)]).astype(dt)
    dot = (nc[0] * v[0] + nc[1] * v[1]) + nc[2] * v[2]
    sg = np.where(dot > 0, dt.type(-1), dt.type(1)).astype(dt) if freeze is None else freeze["sg"].astype(dt)
    return dict(a=a, qn=qn, rn=rn, R=R, nw=nw, nc=nc, sg=sg, n=(sg * nc).astype(dt))


def normal_colour(n, dt):
    """The colour [1,3,N] whose composite is N / 2: n / 2 stays below the composite's min(c, 1) clamp, and the factor is exact."""
    return (n[None] * 0.5).astype(dt)


def normal_forward(sorted_pid, ranges, ndc, inv_cov2d, opacity, n, H, W, th, tw, specific_tiles=None):
    """N [V,3,Hp,Wp] of the records (ndc, inv_cov2d, opacity) with normals n [3,N] over the given tile lists."""
    col = normal_colour(n, ndc.dtype)
    img = oracle.rasterize_forward(sorted_pid, ranges, ndc, inv_cov2d, col, opacity, specific_tiles, H, W, th, tw)[0]
    return img * 2


def project_normal_backward(params, ids, camera, frame, dn):
    """The normal term of the project backward in fp64: (d rot [4,A,S] of the raw quaternion, d_view [4,4])."""
    C, S = params["xyz"].shape[-2:]
    q = params["rot"][:, ids, :].reshape(4, -1).astype(np.float64)
    qn = q / np.sqrt((q * q).sum(0) + 1e-12)
    rn = 1 / np.sqrt((q * q).sum(0) + 1e-12)
    V = np.asarray(camera["view"], np.float64).reshape(4, 4)
    dnc = frame["sg"].astype(np.float64) * np.asarray(dn, np.float64)
    dnw = V[:3, :3] @ dnc
    dR = np.zeros((9, dnw.shape[1]))
    for k in range(3):
        for r in range(3):
            dR[3 * r + k] = np.where(frame["a"] == r, dnw[k], 0.0)
    dqn = quat_R_backward(qn, dR)
    dq = rn * (dqn - (dqn * qn).sum(0) * qn)
    d_view = np.zeros((4, 4))
    d_view[:3, :3] = frame["nw"].astype(np.float64) @ dnc.T
    return dq.reshape(4, len(ids), S), d_view
