"""CPU restatement of the fused path with all its modes, in numpy (fp32 or fp64), for the mode tests.

``render_forward_backward`` runs the oracle's public stages in the order of ``oracle.render_forward_backward`` and puts each
mode's step between them (DESIGN.md section 1): the 3D filter (tests/filter3d_oracle.py) between activation and projection, the
antialiased opacity (tests/aa_oracle.py) after the projection, the depth and normal images (tests/depth_oracle.py,
tests/normal_oracle.py) as extra composites with the colour's blend weights, and the exact terms (tests/exact_grad_oracle.py)
after the activation backward.  With every mode off it computes what the oracle's own composition computes.
``camera_backward`` is the camera gradient of one view of that composition.  The oracle library itself has no modes.
"""
import numpy as np

import oracle
from tests import aa_oracle as aa
from tests import camera_oracle as co
from tests import depth_oracle as dp
from tests import exact_grad_oracle as ex
from tests import filter3d_oracle as f3
from tests import normal_oracle as nm


def _pad(g, shape):
    full = np.zeros(shape, g.dtype)
    full[..., :g.shape[-2], :g.shape[-1]] = g
    return full


def render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, *, true_sigmoid_grad=False,
                            antialiased=False, filter_3d=None, exact_grad=False, render_depth=False, d_depth_fn=None,
                            render_normal=False, d_normal_fn=None, lists=None, freeze=None, normal_freeze=None):
    """Forward and backward of one view with the modes asked for -> the oracle's dict plus the modes' outputs.

    filter_3d: the 3D filter [1,C,S] or None.  d_depth_fn(D, T) and d_normal_fn(N, T) -> (dL/dD or dL/dN, dL/dT or None): the
    gradients of a depth or normal loss; without one the image is rendered and no gradient added.
    lists: (ranges, sorted_pid) to use instead of binning (frozen tile lists for finite differences).
    freeze: dict that may hold "J" [1,3,3,N] and "color" [1,3,N] to use instead of the ones the camera gives (J and the SH
    directions held constant, the convention of the position and camera gradients).
    normal_freeze: an earlier "frame" whose shortest axes and facing signs are kept.

    Beyond the oracle's keys: "o_eff" (= "opacity", the opacity the raster sees), "rho" and "rho3" (the antialiasing and filter
    factors, ones when off), "scale_f" (the filtered activated scale), "G_aa" (the antialiasing term of d cov2d [2,2,N], zero when
    off), "exact_terms" (see _exact_terms), "depth" [V,1,H,W], "depth_padded", "dz" [N] (dL/dz), "normal" [V,3,H,W],
    "normal_padded", "dn" [3,N] (dL/dn) and "frame" (normal_oracle.normal_frame); None for a mode that is off."""
    H, W = img_hw
    th, tw = tile_hw
    freeze = freeze or {}
    view, proj = camera["view"], camera["proj"]
    # cull, activate
    _, nvis, ids = oracle.frustum_culling_aabb(chunk_aabb[0], chunk_aabb[1], camera["frustumplane"])
    act = oracle.cull_compact_activate(sh_degree, ids, nvis, view, params["xyz"], params["scale"], params["rot"], params["sh_0"],
                                       params["sh_rest"], params["opacity"])
    xyz, scale, rot, color, opacity = [a.reshape(*a.shape[:-2], -1) for a in act]
    if "color" in freeze:
        color = freeze["color"]
    N = opacity.shape[-1]
    # 3D filter
    scale_f, o3, ff = scale, opacity, None
    if filter_3d is not None:
        C, S = params["xyz"].shape[-2:]
        fc = np.asarray(filter_3d).reshape(C, S)[ids].reshape(-1).astype(scale.dtype)
        scale_f, o3, ff = f3.filter_forward(scale, fc, opacity)
    # project
    inter = oracle.project(xyz, scale_f, rot, view, proj, img_hw)
    if "J" in freeze:
        inter["J"] = freeze["J"]
        inter["cov2d"] = oracle.createCov2dDirectly_forward(inter["J"], view, inter["T"])
        inter["inv_cov2d"] = oracle.eigh_and_inv_2x2matrix_forward(inter["cov2d"])[2]
    ndc, inv = inter["ndc"], inter["inv_cov2d"]
    dt = ndc.dtype
    # antialias
    o_rec, rho, fa = o3, np.ones(N, opacity.dtype), None
    if antialiased:
        o_rec, rho, fa = aa.antialias_forward(aa.cov_M(inter, view), o3)
    # bin
    if lists is None:
        ranges, sorted_pid, _, _ = oracle.binning(ndc, inter["view_pos"][:, 2], inv, o_rec, None, img_hw, tile_hw)
    else:
        ranges, sorted_pid = lists
    # raster forward: the colour, and the depth and normal composites with the same blend weights
    img, T, last, _, _, fragile = oracle.rasterize_forward(sorted_pid, ranges, ndc, inv, color, o_rec, None, H, W, th, tw)
    img_c = np.clip(img[..., :H, :W], 0, 1)
    g_full = np.zeros_like(img)
    g_full[..., :H, :W] = d_img_fn(img_c) * ((img[..., :H, :W] >= 0) & (img[..., :H, :W] <= 1))
    gmax = np.abs(g_full).max()
    gmax = gmax if gmax > 0 else 1.0
    d_img = (g_full / gmax).astype(img.dtype)
    D = gz = gt_depth = colz = None
    if render_depth:
        z = inter["view_pos"][0, 2]
        colz, zs = dp.depth_colour(z, dt)
        D = dp.depth_forward(sorted_pid, ranges, ndc, inv, o_rec, z, H, W, th, tw)
        if d_depth_fn is not None:
            gz, gt_depth = d_depth_fn(D[..., :H, :W], T[..., :H, :W])
    Nimg = gn = gt_normal = frame = coln = None
    if render_normal:
        s_raw = params["scale"][:, ids, :].reshape(3, -1).astype(dt)
        q_raw = params["rot"][:, ids, :].reshape(4, -1).astype(dt)
        frame = nm.normal_frame(s_raw, q_raw, np.asarray(view).reshape(4, 4), inter["view_pos"][0].astype(dt), freeze=normal_freeze)
        coln = nm.normal_colour(frame["n"], dt)
        Nimg = nm.normal_forward(sorted_pid, ranges, ndc, inv, o_rec, frame["n"], H, W, th, tw)
        if d_normal_fn is not None:
            gn, gt_normal = d_normal_fn(Nimg[..., :H, :W], T[..., :H, :W])
    # raster backward.  The colour pass takes the transmittance gradient, divided by the scaler like its other inputs, summed as
    # gt_depth + gt_normal; the record gradients of the normal and then the depth pass are added to the colour pass's in that
    # order: (colour + normal) + depth.
    d_trans = None
    for gt in (gt_depth, gt_normal):
        if gt is not None:
            gt = (_pad(np.asarray(gt, T.dtype), T.shape) / float(gmax)).astype(T.dtype)
            d_trans = gt if d_trans is None else d_trans + gt
    d_ndc, d_cov, d_col, d_op, _, _ = oracle.rasterize_backward(sorted_pid, ranges, ndc, inv, color, o_rec, None, T, last, d_img,
                                                                d_trans, gmax, H, W, th, tw)
    dn = None if frame is None else np.zeros(frame["n"].shape, dt)
    if gn is not None:
        dn_img = (_pad(np.asarray(gn, d_img.dtype), (1, 3, *T.shape[-2:])) * 2).astype(d_img.dtype)
        nn, nc, ncol, nop, _, _ = oracle.rasterize_backward(sorted_pid, ranges, ndc, inv, coln, o_rec, None, T, last, dn_img, None,
                                                            None, H, W, th, tw)
        d_ndc, d_cov, d_op = d_ndc + nn, d_cov + nc, d_op + nop
        dn = ncol[0] * 0.5
    dz = None if D is None else np.zeros(z.shape, dt)
    if gz is not None:
        dz_img = np.zeros_like(d_img)
        dz_img[:, :1] = _pad(np.asarray(gz, d_img.dtype), T.shape) * zs
        zn, zc, zcol, zop, _, _ = oracle.rasterize_backward(sorted_pid, ranges, ndc, inv, colz, o_rec, None, T, last, dz_img, None,
                                                            None, H, W, th, tw)
        d_ndc, d_cov, d_op = d_ndc + zn, d_cov + zc, d_op + zop
        dz = zcol[0, 0] / zs
    # antialias backward
    G_aa = np.zeros((2, 2, N), img.dtype)
    d_o = d_op                                       # d o3 from here on
    if antialiased:
        d_o, G_aa = aa.antialias_backward(fa, o3, d_op)
    # project backward, with the antialiasing term added to d cov2d and the filter's terms after createTransformMatrix_backward
    g_cov = np.nan_to_num(oracle.inv_2x2matrix_backward(inv, d_cov), nan=0.0)
    if antialiased:
        g_cov = g_cov + G_aa[None]
    gT = oracle.createCov2dDirectly_backward(g_cov, inter["J"], view, inter["T"])
    gq, gs = oracle.createTransformMatrix_backward(gT, rot, scale_f)
    d_sig, extra = d_o, None
    if ff is not None:
        gs = gs * (ff["s"] / ff["sp"])               # d s from d s'
        d_sig = d_o * ff["rho3"]
        extra = (d_o * o3) * (ff["f2"] / ff["qf"])   # d s_raw of o3 = sigma rho3(s), f held constant
    gp = oracle.mvp_transform_backward(d_ndc, np.zeros_like(inter["view_pos"]), view, proj, inter["view_pos"])
    # activate backward
    A, S = act[0].shape[-2:]
    shp = lambda a: a.reshape(*a.shape[:-1], A, S)
    grads = list(oracle.activate_backward(sh_degree, ids, nvis, view, params["xyz"], params["scale"], params["rot"], params["sh_0"],
                                          params["sh_rest"], params["opacity"], shp(gp), shp(gs), shp(gq), shp(d_col), shp(d_sig),
                                          true_sigmoid_grad))
    if extra is not None:
        grads[1] = (grads[1] + shp(extra)).astype(grads[1].dtype)
    out = dict(img=img_c, img_padded=img, T=T, last=last, fragile=fragile, visible_chunk_id=ids,
               grads=dict(zip(("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity"), grads)),
               inter=inter, ranges=ranges, sorted_pid=sorted_pid, color=color, opacity=o_rec, o_eff=o_rec, rho=rho,
               rho3=np.ones(N, opacity.dtype) if ff is None else ff["rho3"], scale_f=scale_f,
               d_ndc=d_ndc, d_cov=d_cov, d_col=d_col, d_op=d_op, G_aa=G_aa, exact_terms=None,
               depth=None if D is None else D[..., :H, :W], depth_padded=D, dz=dz,
               normal=None if Nimg is None else Nimg[..., :H, :W], normal_padded=Nimg, dn=dn, frame=frame)
    # the exact, depth and normal terms, each added in fp64 and rounded to the gradient's dtype, in that order
    Vm = np.asarray(view, np.float64).reshape(4, 4)
    gx = grads[0]
    if exact_grad:
        dvJ, _, _, gd, _ = out["exact_terms"] = _exact_terms(params, out, camera, img_hw, sh_degree)
        gx = (gx.astype(np.float64) + (Vm[:3, :3] @ dvJ + gd).reshape(gx.shape)).astype(gx.dtype)
    if dz is not None:
        gx = (gx.astype(np.float64) + (Vm[:3, 2][:, None] * dz).reshape(gx.shape)).astype(gx.dtype)
    out["grads"]["xyz"] = gx
    if dn is not None:
        dq, _ = nm.project_normal_backward(params, ids, camera, frame, dn)
        out["grads"]["rot"] = (grads[2].astype(np.float64) + dq).astype(grads[2].dtype)
    return out


def _exact_terms(params, out, camera, img_hw, sh_degree):
    """Per-Gaussian terms of the exact mode: (dv_J [3,N] view space, d p00 [N], d p11 [N], g_d [3,N], p [3,N]) in fp64."""
    inter = out["inter"]
    Vm = np.asarray(camera["view"], np.float64).reshape(4, 4)
    P = np.asarray(camera["proj"], np.float64).reshape(4, 4)
    ids = out["visible_chunk_id"]
    p = params["xyz"][:, ids, :].reshape(3, -1).astype(np.float64)
    N = p.shape[1]
    # J term: G the whole d cov2d (the antialiased term included), dJ = V3^T dVJ
    G = np.nan_to_num(oracle.inv_2x2matrix_backward(inter["inv_cov2d"], out["d_cov"]), nan=0.0)[0] + out["G_aa"]
    _, dVJ = co.sigma_chain(inter, camera["view"], G, np.float64)
    dJ = np.einsum("ak,nac->nkc", Vm[:3, :3], dVJ)                                 # [N,3,2]
    v = inter["view_pos"][0, :3].astype(np.float64)
    dvJ, dp00, dp11 = ex.J_backward(v, P[0, 0], P[1, 1], *img_hw, dJ[:, 0, 0], dJ[:, 1, 1], dJ[:, 2, 0], dJ[:, 2, 1])
    # SH direction term
    gd = np.zeros((3, N))
    if sh_degree > 0:
        K = (sh_degree + 1) ** 2
        sh = np.concatenate([params["sh_0"][:, :, ids, :], params["sh_rest"][:K - 1, :, ids, :]]).reshape(K, 3, N)
        gd = ex.direction_backward(sh_degree, p, Vm, sh.astype(np.float64), out["d_col"][0].astype(np.float64))
    return dvJ, dp00, dp11, gd, p


def camera_backward(params, out, camera, img_hw, sh_degree=None, exact_grad=False):
    """Camera gradient of one view from render_forward_backward's dict -> (d_view [4,4], d_proj [4,4]).

    camera_oracle.camera_backward (J and the SH direction held constant), plus the antialiasing term in the records' dtype, plus
    in fp64 the exact terms (with exact_grad; they need sh_degree or the dict's "exact_terms"), the depth term and the normal term,
    in that order.  The result is fp64 when any of the last three is there."""
    d_view, d_proj, _ = co.camera_backward(params, out, camera, img_hw)
    inter = out["inter"]
    # G_aa reaches the view matrix through dM = 2 M G like the rest of d cov2d
    J, dVJ = co.sigma_chain(inter, camera["view"], out["G_aa"], inter["view_pos"].dtype)
    d_view[:3, :3] += np.einsum("nac,nkc->ak", dVJ, J)
    if not (exact_grad or out["dz"] is not None or out["dn"] is not None):
        return d_view, d_proj
    d_view, d_proj = d_view.astype(np.float64), d_proj.astype(np.float64)
    ids = out["visible_chunk_id"]
    if exact_grad:
        dvJ, dp00, dp11, gd, p = out["exact_terms"] or _exact_terms(params, out, camera, img_hw, sh_degree)
        Vm = np.asarray(camera["view"], np.float64).reshape(4, 4)
        d_view[:3, :3] += p @ dvJ.T                     # d V[k][j] += p~_k dv_j
        d_view[3, :3] += dvJ.sum(axis=1)
        g = gd.sum(axis=1)
        d_view[3, :3] += Vm[:3, :3].T @ g               # d V[3][k] += sum_m g_d[m] V[m][k]
        d_view[:3, :3] += np.outer(g, Vm[3, :3])        # d V[m][k] += g_d[m] V[3][k]
        d_proj[0, 0] += dp00.sum()
        d_proj[1, 1] += dp11.sum()
    if out["dz"] is not None:                           # d view[k][2] += sum_i p~_ik dz_i
        p = params["xyz"][:, ids, :].reshape(3, -1).astype(np.float64)
        dz = np.asarray(out["dz"], np.float64)
        d_view[:3, 2] += p @ dz
        d_view[3, 2] += dz.sum()
    if out["dn"] is not None:                           # d view[k][j] += sum_i n_w[k] dn_c[j]
        d_view += nm.project_normal_backward(params, ids, camera, out["frame"], out["dn"])[1]
    return d_view, d_proj
