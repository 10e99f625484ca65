"""CPU restatement of the antialiased mode in numpy (fp32 or fp64), for the antialiasing tests.

The mode (DESIGN.md section 1) scales each splat's opacity by rho = sqrt(det(M^T M) / det(M^T M + 0.3 I)), M = T.V3x3.J, so
that the filtered splat's integrated alpha equals the unfiltered Gaussian's.  Its forward and backward sit between the oracle's
stages: after ``oracle.project`` and before binning, and in the backward between the raster gradient and the projection /
activation backward.  ``render_forward_backward`` composes the oracle's public stages in the order of
``oracle.render_forward_backward`` with that step in between; with ``antialiased=False`` it returns the same bits as the oracle's
own composition.  The oracle library itself has no antialiased mode.

numpy evaluates every elementwise operation below once, correctly rounded and without contraction, in the order written: the
same order as ``antialias_factor`` in fused.cu, so the fp32 opacity here is the kernel's bit for bit given the same M.
"""
import numpy as np

import oracle


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


def render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, true_sigmoid_grad=False,
                            antialiased=False, lists=None, freeze=None):
    """oracle.render_forward_backward with the antialiased mode.  Returns the oracle's dict plus "o_eff", "rho" and "G_aa" (the
    antialiasing term of d cov2d, [2,2,N]; zero when off).

    lists: (ranges, sorted_pid) to use instead of binning (frozen tile lists for finite differences).
    freeze: dict that may hold "J" [1,3,3,N] and "color" [1,3,N] to use instead of the ones the camera gives (J and the SH
    directions held constant, the convention of the position and camera gradients)."""
    H, W = img_hw
    th, tw = tile_hw
    freeze = freeze or {}
    vis, nvis, ids = oracle.frustum_culling_aabb(chunk_aabb[0], chunk_aabb[1], camera["frustumplane"])
    act = oracle.cull_compact_activate(sh_degree, ids, nvis, camera["view"], params["xyz"], params["scale"], params["rot"],
                                       params["sh_0"], params["sh_rest"], params["opacity"])
    flat = [a.reshape(*a.shape[:-2], -1) for a in act]
    xyz, scale, rot, color, opacity = flat
    if "color" in freeze:
        color = freeze["color"]
    inter = oracle.project(xyz, scale, rot, camera["view"], camera["proj"], img_hw)
    if "J" in freeze:
        inter["J"] = freeze["J"]
        inter["cov2d"] = oracle.createCov2dDirectly_forward(inter["J"], camera["view"], inter["T"])
        inter["inv_cov2d"] = oracle.eigh_and_inv_2x2matrix_forward(inter["cov2d"])[2]
    N = opacity.shape[-1]
    o_rec, rho, f = opacity, np.ones(N, opacity.dtype), None
    if antialiased:
        o_rec, rho, f = antialias_forward(cov_M(inter, camera["view"]), opacity)
    if lists is None:
        ranges, sorted_pid, _, _ = oracle.binning(inter["ndc"], inter["view_pos"][:, 2], inter["inv_cov2d"], o_rec, None, img_hw,
                                                  tile_hw)
    else:
        ranges, sorted_pid = lists
    img, T, last, _, _, fragile = oracle.rasterize_forward(sorted_pid, ranges, inter["ndc"], inter["inv_cov2d"], color, o_rec, None,
                                                           H, W, th, tw)
    img_c = np.clip(img[..., :H, :W], 0, 1)
    g = d_img_fn(img_c)
    g_full = np.zeros_like(img)
    mask = (img[..., :H, :W] >= 0) & (img[..., :H, :W] <= 1)
    g_full[..., :H, :W] = g * mask
    gmax = np.abs(g_full).max()
    gmax = gmax if gmax > 0 else 1.0
    d_ndc, d_cov, d_col, d_op, _, _ = oracle.rasterize_backward(sorted_pid, ranges, inter["ndc"], inter["inv_cov2d"], color, o_rec,
                                                                None, T, last, (g_full / gmax).astype(img.dtype), None, gmax, H, W,
                                                                th, tw)
    G_aa = np.zeros((2, 2, N), img.dtype)
    d_o = d_op
    if antialiased:
        d_o, G_aa = antialias_backward(f, opacity, d_op)
    # oracle.project_backward with the antialiasing term added to d cov2d
    g_cov = np.nan_to_num(oracle.inv_2x2matrix_backward(inter["inv_cov2d"], d_cov), nan=0.0)
    if antialiased:
        g_cov = g_cov + G_aa[None]
    gT = oracle.createCov2dDirectly_backward(g_cov, inter["J"], camera["view"], inter["T"])
    gq, gs = oracle.createTransformMatrix_backward(gT, rot, scale)
    gp = oracle.mvp_transform_backward(d_ndc, np.zeros_like(inter["view_pos"]), camera["view"], camera["proj"], inter["view_pos"])
    A, S = act[0].shape[-2:]
    shp = lambda a: a.reshape(*a.shape[:-1], A, S)
    grads = oracle.activate_backward(sh_degree, ids, nvis, camera["view"], params["xyz"], params["scale"], params["rot"],
                                     params["sh_0"], params["sh_rest"], params["opacity"], shp(gp), shp(gs), shp(gq), shp(d_col),
                                     shp(d_o), true_sigmoid_grad)
    return dict(img=img_c, img_padded=img, T=T, last=last, fragile=fragile, visible_chunk_id=ids,
                grads=dict(zip(("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity"), grads)),
                inter=inter, ranges=ranges, sorted_pid=sorted_pid, color=color, opacity=o_rec, o_eff=o_rec, rho=rho,
                d_ndc=d_ndc, d_cov=d_cov, d_col=d_col, d_op=d_op, G_aa=G_aa)


def camera_backward(params, out, camera, img_hw):
    """tests/camera_oracle.camera_backward plus the antialiasing term: its G_aa reaches the view matrix through dM = 2 M G like
    the rest of d cov2d (J and the SH direction held constant) -> (d_view [4,4], d_proj [4,4])."""
    from tests import camera_oracle as co
    d_view, d_proj, _ = co.camera_backward(params, out, camera, img_hw)
    inter = out["inter"]
    dt = inter["view_pos"].dtype
    Vm = np.asarray(camera["view"], dt).reshape(4, 4)
    Gc = np.moveaxis(out["G_aa"], -1, 0)                                           # [N,2,2]
    J = np.moveaxis(inter["J"][0], -1, 0)[:, :, :2]                                # [N,3,2]
    T = np.moveaxis(inter["T"], -1, 0)                                             # [N,3,3]
    VJ = np.einsum("ak,nkc->nac", Vm[:3, :3], J)
    M = np.einsum("nak,nkc->nac", T, VJ)
    dM = 2 * np.einsum("nac,ncd->nad", M, Gc)
    dVJ = np.einsum("nak,nac->nkc", T, dM)
    d_view = d_view.copy()
    d_view[:3, :3] += np.einsum("nac,nkc->ak", dVJ, J)
    return d_view, d_proj
