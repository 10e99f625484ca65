"""CPU restatement of Mip-Splatting's 3D smoothing filter in numpy (fp32 or fp64), for the filter tests.

The filter (DESIGN.md section 1, "3D smoothing filter") is per-Gaussian data f computed from the training cameras
(``compute_filter``, the order of ``filter_3d_kernel`` in csrc/scene.cu).  It widens each activated scale to s' = sqrt(s^2 + f^2)
and scales the opacity by rho3 = sqrt(prod_k s_k^2 / s'_k^2) (``filter_forward``, the order of ``filter_3d_factor`` in fused.cu).
``render_forward_backward`` composes the oracle's public stages in the order of ``oracle.render_forward_backward``: the filter
sits between ``oracle.cull_compact_activate`` and ``oracle.project``, the antialiased step of tests/aa_oracle.py (when asked)
after ``oracle.project``, and in the backward the filter's terms sit between ``createTransformMatrix_backward`` and
``activate_backward``.  With ``filter_3d=None`` it returns the same bits as aa_oracle's composition, and so, with the
antialiased mode off, the oracle's own.  The oracle library itself has no filter.

numpy evaluates every elementwise operation below once, correctly rounded and without contraction, in the order written, so the
fp32 filter and the fp32 filtered scale and opacity are the kernels' bit for bit.
"""
import numpy as np

import oracle
from tests import aa_oracle as aa

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


def render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, true_sigmoid_grad=False,
                            antialiased=False, filter_3d=None, lists=None, freeze=None):
    """aa_oracle.render_forward_backward with the 3D filter filter_3d ([1,C,S] or None).  Returns its dict plus "rho3" [N] and
    "scale_f" (the filtered activated scale [3,N]); lists and freeze as there."""
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
    N = opacity.shape[-1]
    scale_f, o3, ff = scale, opacity, None
    if filter_3d is not None:
        C, S = params["xyz"].shape[-2:]
        fc = np.asarray(filter_3d).reshape(C, S)[ids].reshape(-1).astype(scale.dtype)
        scale_f, o3, ff = filter_forward(scale, fc, opacity)
    inter = oracle.project(xyz, scale_f, rot, camera["view"], camera["proj"], img_hw)
    if "J" in freeze:
        inter["J"] = freeze["J"]
        inter["cov2d"] = oracle.createCov2dDirectly_forward(inter["J"], camera["view"], inter["T"])
        inter["inv_cov2d"] = oracle.eigh_and_inv_2x2matrix_forward(inter["cov2d"])[2]
    o_rec, rho, fa = o3, np.ones(N, opacity.dtype), None
    if antialiased:
        o_rec, rho, fa = aa.antialias_forward(aa.cov_M(inter, camera["view"]), o3)
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
    d_o = d_op                                       # d o3 from here on
    if antialiased:
        d_o, G_aa = aa.antialias_backward(fa, o3, d_op)
    g_cov = np.nan_to_num(oracle.inv_2x2matrix_backward(inter["inv_cov2d"], d_cov), nan=0.0)
    if antialiased:
        g_cov = g_cov + G_aa[None]
    gT = oracle.createCov2dDirectly_backward(g_cov, inter["J"], camera["view"], inter["T"])
    gq, gs = oracle.createTransformMatrix_backward(gT, rot, scale_f)
    d_sig, extra = d_o, None
    if ff is not None:
        gs = gs * (ff["s"] / ff["sp"])               # d s from d s'
        d_sig = d_o * ff["rho3"]
        extra = (d_o * o3) * (ff["f2"] / ff["qf"])   # d s_raw of o3 = sigma rho3(s), f held constant
    gp = oracle.mvp_transform_backward(d_ndc, np.zeros_like(inter["view_pos"]), camera["view"], camera["proj"], inter["view_pos"])
    A, S = act[0].shape[-2:]
    shp = lambda a: a.reshape(*a.shape[:-1], A, S)
    grads = list(oracle.activate_backward(sh_degree, ids, nvis, camera["view"], params["xyz"], params["scale"], params["rot"],
                                          params["sh_0"], params["sh_rest"], params["opacity"], shp(gp), shp(gs), shp(gq), shp(d_col),
                                          shp(d_sig), true_sigmoid_grad))
    if extra is not None:
        grads[1] = (grads[1] + shp(extra)).astype(grads[1].dtype)
    return dict(img=img_c, img_padded=img, T=T, last=last, fragile=fragile, visible_chunk_id=ids,
                grads=dict(zip(("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity"), grads)),
                inter=inter, ranges=ranges, sorted_pid=sorted_pid, color=color, opacity=o_rec, o_eff=o_rec, rho=rho,
                rho3=np.ones(N, opacity.dtype) if ff is None else ff["rho3"], scale_f=scale_f,
                d_ndc=d_ndc, d_cov=d_cov, d_col=d_col, d_op=d_op, G_aa=G_aa)

