"""CPU restatement of the camera path in numpy (fp32 or fp64), for the camera tests.

- create_viewproj_forward / create_viewproj_backward restate GR/compact.cu:17-141 and :143-316 with the reference's quirks: the
  fov gradient scales d proj[1][1] by the INTEGER quotient img_w // img_h, and the quaternion gradient is the true derivative
  times |q| (the normalisation backward divides by the norm of the already normalised quaternion).  The fov gradient is the
  sum over views in view order (the reference's is a race for more than one view).
- camera_backward is the camera gradient of one view (DESIGN.md section 1): per-Gaussian contributions through the NDC mean and
  through the V3x3 factor of M = T.V3x3.J, with J and the SH direction held constant, summed over the Gaussians.  It reads the
  intermediates oracle.render_forward_backward returns, so it is the same computation the oracle's position gradient uses.
  tests/fused_oracle.py adds the modes' terms to it.
"""
import numpy as np

import oracle


def quat_view(q):
    """Normalised quaternion (r, x, y, z) -> the 3x3 block of the view matrix (row-vector convention)."""
    r, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)],
                     [2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)],
                     [2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)]], dtype=q.dtype)


def _mats(p, recp, img_h, img_w, z_near, z_far, dt):
    q = p[:4] / np.sqrt(np.sum(p[:4] * p[:4]) + dt(1e-12))
    V = np.zeros((4, 4), dt)
    V[:3, :3] = quat_view(q)
    V[3, :3] = p[4:7]
    V[3, 3] = 1
    p00 = dt(recp)
    P = np.zeros((4, 4), dt)
    P[0, 0] = p00
    P[1, 1] = p00 * dt(img_w) / dt(img_h)
    P[2, 2] = dt(z_far) / (dt(z_far) - dt(z_near))
    P[2, 3] = 1
    P[3, 2] = -dt(z_far) * dt(z_near) / (dt(z_far) - dt(z_near))
    return q, V, P


def planes_of(VP):
    """Six frustum planes [6,4] of a view-projection matrix (GR/compact.cu:90-118)."""
    c = VP
    return np.stack([c[:, 3] + c[:, 0], c[:, 3] - c[:, 0], c[:, 3] + c[:, 1], c[:, 3] - c[:, 1], c[:, 2], c[:, 3] - c[:, 2]])


def create_viewproj_forward(view_params, recp_tan_half_fov_x, img_h, img_w, z_near, z_far):
    """view_params [V,7], recp [1] -> (view, proj, viewproj [V,4,4], frustumplane [V,6,4]) in the dtype of view_params."""
    vp = np.asarray(view_params)
    dt = vp.dtype.type
    out = [np.zeros((vp.shape[0], 4, 4), dt) for _ in range(3)] + [np.zeros((vp.shape[0], 6, 4), dt)]
    for v in range(vp.shape[0]):
        _, V, P = _mats(vp[v], np.asarray(recp_tan_half_fov_x).reshape(-1)[0], img_h, img_w, z_near, z_far, dt)
        VP = V @ P
        out[0][v], out[1][v], out[2][v], out[3][v] = V, P, VP, planes_of(VP)
    return out


def create_viewproj_backward(view_grad, proj_grad, viewproj_grad, view_params, recp_tan_half_fov_x, img_h, img_w, z_near, z_far):
    """-> (grad_view_params [V,7], grad_recp [1]) with the reference's arithmetic."""
    vp = np.asarray(view_params)
    dt = vp.dtype.type
    gvp_out = np.zeros_like(vp)
    fov = dt(0)
    for v in range(vp.shape[0]):
        q, V, P = _mats(vp[v], np.asarray(recp_tan_half_fov_x).reshape(-1)[0], img_h, img_w, z_near, z_far, dt)
        G = np.asarray(viewproj_grad[v], dt)
        gV = np.asarray(view_grad[v], dt) + G @ P.T          # d(V P)/dV
        gP = np.asarray(proj_grad[v], dt) + V.T @ G          # d(V P)/dP
        r, x, y, z = q
        # d view[0:3,0:3] / d (r, x, y, z) of the normalised quaternion
        dR = np.array([
            [[0, 0, -4 * y, -4 * z], [2 * z, 2 * y, 2 * x, 2 * r], [-2 * y, 2 * z, -2 * r, 2 * x]],
            [[-2 * z, 2 * y, 2 * x, -2 * r], [0, -4 * x, 0, -4 * z], [2 * x, 2 * r, 2 * z, 2 * y]],
            [[2 * y, 2 * z, 2 * r, 2 * x], [-2 * x, -2 * r, 2 * z, 2 * y], [0, -4 * x, -4 * y, 0]]], dt)
        gq = np.einsum("ij,ijk->k", gV[:3, :3], dR)
        norm = np.sqrt(np.sum(q * q))
        dot = np.sum(q * gq) / (norm * norm)
        gvp_out[v, :4] = gq / norm - q * dot
        gvp_out[v, 4:7] = gV[3, :3]
        fov = fov + gP[0, 0]
        fov = fov + gP[1, 1] * dt(img_w // img_h)
    return gvp_out, np.array([fov], dt)


def sigma_chain(inter, view, G, dt):
    """The Sigma2 path of a d cov2d G [2,2,N] in dtype dt, every Gaussian first: M = T.V3x3.J, dM = 2 M G, dVJ = T^T dM ->
    (J [N,3,2], dVJ [N,3,2])."""
    V3 = np.asarray(view, dt).reshape(4, 4)[:3, :3]
    G = np.moveaxis(np.asarray(G, dt), -1, 0)                                      # [N,2,2]
    J = np.moveaxis(np.asarray(inter["J"][0], dt), -1, 0)[:, :, :2]                # [N,3,2]
    T = np.moveaxis(np.asarray(inter["T"], dt), -1, 0)                             # [N,3,3]
    M = np.einsum("nak,nkc->nac", T, np.einsum("ak,nkc->nac", V3, J))
    dM = 2 * np.einsum("nac,ncd->nad", M, G)
    return J, np.einsum("nak,nac->nkc", T, dM)


def camera_backward(params, out, camera, img_hw):
    """Camera gradient of one view from oracle.render_forward_backward's output -> (d_view [4,4], d_proj [4,4]).

    Also returns the per-Gaussian contributions (dict of [N,4,4] arrays, "ndc_view", "sigma_view", "ndc_proj") so that tests
    can check the parts separately."""
    inter = out["inter"]
    dt = inter["view_pos"].dtype
    ids = out["visible_chunk_id"]
    S = params["xyz"].shape[-1]
    N = inter["view_pos"].shape[2]
    pt = np.ones((N, 4), dt)
    pt[:, :3] = params["xyz"][:, ids, :].reshape(3, -1).T.astype(dt)
    P = np.asarray(camera["proj"], dt).reshape(4, 4)
    v = inter["view_pos"][0].T                                                     # [N,4]
    h = v @ P
    iw = np.where(np.abs(h[:, 3]) > 1e-12, 1.0 / np.where(h[:, 3] == 0, 1, h[:, 3]), 0.0).astype(dt)
    g = out["d_ndc"][0].T                                                          # [N,4], x and y used
    n0, n1 = h[:, 0] * iw, h[:, 1] * iw
    dh = np.stack([g[:, 0] * iw, g[:, 1] * iw, np.zeros_like(iw), -(g[:, 0] * n0 + g[:, 1] * n1) * iw], axis=1)
    dv = dh @ P.T                                                                  # dv_k = sum_j dh_j P[k][j]
    ndc_view = pt[:, :, None] * dv[:, None, :]
    ndc_proj = v[:, :, None] * dh[:, None, :]
    # Sigma2 path: G = d cov2d (inverse backward, NaN -> 0), dV3 = dVJ J^T
    G = np.nan_to_num(oracle.inv_2x2matrix_backward(inter["inv_cov2d"], out["d_cov"]), nan=0.0)[0]      # [2,2,N]
    J, dVJ = sigma_chain(inter, camera["view"], G, dt)
    sigma_view = np.zeros((N, 4, 4), dt)
    sigma_view[:, :3, :3] = np.einsum("nac,nkc->nak", dVJ, J)
    parts = dict(ndc_view=ndc_view, sigma_view=sigma_view, ndc_proj=ndc_proj)
    return (ndc_view + sigma_view).sum(axis=0), ndc_proj.sum(axis=0), parts
