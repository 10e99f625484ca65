"""CPU restatement of the normal mode in numpy (fp32 or fp64), for the normal tests.

The mode (DESIGN.md section 1, "Normals") renders N = sum_i w_i n_i with the colour's blend weights w_i and n_i the camera-facing
view-space normal of Gaussian i's shortest axis.  That is the oracle's own composite with the colour replaced by n / 2: |n_k| <= 1
keeps the composite below the min(c, 1) clamp, and scaling by 2 is exact.  Both use the same weights, so the backward is the sum
of the colour backward and the same backward of that normal-as-colour image; its colour gradient is dL/dn (times 1/2), which then
reaches the rotations (row a of the rotation-matrix gradient) and the camera (d view[k][j] += n_w[k] dn_c[j]).

``render_forward_backward`` runs exact_grad_oracle's composition (and, with render_depth, depth_oracle's stages) with
``oracle.rasterize_backward`` intercepted for the duration of the call, as depth_oracle does.  The oracle library itself is not
changed, and with ``render_normal=False`` the call is depth_oracle's.
"""
import contextlib

import numpy as np

import oracle
from tests import depth_oracle as dp


def quat_R(qn):
    """Rotation matrix rows [9,N] of unit quaternions qn [4,N] (r, x, y, z), laid out as fused_quat_R."""
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


@contextlib.contextmanager
def _normal_stages(frame_fn, d_normal_fn, rec):
    backward0 = oracle.rasterize_backward

    def rasterize_backward(sorted_pid, ranges, ndc, inv, color, opacity, tiles, T, last, d_img, d_trans, scaler, H, W, th, tw, **kw):
        if "frame" in rec:               # depth_oracle's depth-as-colour pass (after the colour pass): nothing to add
            return backward0(sorted_pid, ranges, ndc, inv, color, opacity, tiles, T, last, d_img, d_trans, scaler, H, W, th, tw, **kw)
        fr = frame_fn(ndc.dtype)
        rec["frame"] = fr
        coln = normal_colour(fr["n"], ndc.dtype)
        Nimg = normal_forward(sorted_pid, ranges, ndc, inv, opacity, fr["n"], H, W, th, tw, tiles)
        rec["normal"] = Nimg
        gn = gt = None
        if d_normal_fn is not None:
            gn, gt = d_normal_fn(Nimg[..., :H, :W], T[..., :H, :W])
        s = 1.0 if scaler is None else float(np.asarray(scaler).reshape(-1)[0])
        if gt is not None:
            gt = (dp._pad(np.asarray(gt, T.dtype), T.shape) / s).astype(T.dtype)
            d_trans = gt if d_trans is None else d_trans + gt
        out = list(backward0(sorted_pid, ranges, ndc, inv, color, opacity, tiles, T, last, d_img, d_trans, scaler, H, W, th, tw, **kw))
        rec["dn"] = np.zeros(fr["n"].shape, ndc.dtype)
        if gn is not None:
            dn_img = (dp._pad(np.asarray(gn, d_img.dtype), (1, 3, *T.shape[-2:])) * 2).astype(d_img.dtype)
            nn, nc_, ncol, nop, _, _ = backward0(sorted_pid, ranges, ndc, inv, coln, opacity, tiles, T, last, dn_img, None, None,
                                                 H, W, th, tw)
            out[0], out[1], out[3] = out[0] + nn, out[1] + nc_, out[3] + nop
            rec["dn"] = ncol[0] * 0.5
        return tuple(out)

    oracle.rasterize_backward = rasterize_backward
    try:
        yield
    finally:
        oracle.rasterize_backward = backward0


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


def render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, render_normal=False, d_normal_fn=None,
                            render_depth=False, d_depth_fn=None, normal_freeze=None, **kw):
    """depth_oracle.render_forward_backward (kw as there), plus with render_normal the normal N ("normal" [V,3,H,W],
    "normal_padded"), the per-Gaussian frame ("frame": a, nw, nc, sg, n [3,N]) and, when d_normal_fn(N, T) -> (dL/dN, dL/dT or
    None) is given, the normal loss's gradients added to every parameter gradient; "dn" [3,N] is dL/dn of each visible Gaussian.
    normal_freeze: an earlier "frame" whose shortest axes and facing signs are kept."""
    if not render_normal:
        return dp.render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, render_depth=render_depth,
                                          d_depth_fn=d_depth_fn, **kw)
    _, _, ids = oracle.frustum_culling_aabb(chunk_aabb[0], chunk_aabb[1], camera["frustumplane"])
    rec_n, rec_p = {}, {}

    def frame_fn(dt):
        s_raw = params["scale"][:, ids, :].reshape(3, -1).astype(dt)
        q_raw = params["rot"][:, ids, :].reshape(4, -1).astype(dt)
        return normal_frame(s_raw, q_raw, np.asarray(camera["view"]).reshape(4, 4), rec_p["inter"]["view_pos"][0].astype(dt),
                            freeze=normal_freeze)

    project0 = oracle.project

    def project(*a, **k):
        rec_p["inter"] = project0(*a, **k)
        return rec_p["inter"]

    oracle.project = project
    try:
        with _normal_stages(frame_fn, d_normal_fn, rec_n):
            out = dp.render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, render_depth=render_depth,
                                             d_depth_fn=d_depth_fn, **kw)
    finally:
        oracle.project = project0
    H, W = img_hw
    dq, _ = project_normal_backward(params, ids, camera, rec_n["frame"], rec_n["dn"])
    gr = out["grads"]["rot"]
    out["grads"] = dict(out["grads"], rot=(gr.astype(np.float64) + dq).astype(gr.dtype))
    out.update(normal=rec_n["normal"][..., :H, :W], normal_padded=rec_n["normal"], dn=rec_n["dn"], frame=rec_n["frame"])
    return out


def camera_backward(params, out, camera, img_hw, sh_degree=None, exact_grad=False):
    """depth_oracle.camera_backward plus the normal term d view[k][j] += sum_i n_w[k] dn_c[j] (fp64) -> (d_view, d_proj)."""
    d_view, d_proj = dp.camera_backward(params, out, camera, img_hw, sh_degree=sh_degree, exact_grad=exact_grad)
    if "dn" not in out:
        return d_view, d_proj
    _, dv = project_normal_backward(params, out["visible_chunk_id"], camera, out["frame"], out["dn"])
    return np.array(d_view, np.float64) + dv, np.array(d_proj, np.float64)
