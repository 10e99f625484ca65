"""CPU restatement of the depth mode in numpy (fp32 or fp64), for the depth tests.

The mode (DESIGN.md section 1, "Depth") renders D = sum_i w_i z_i with the colour's blend weights w_i and the view-space z_i.
That is the oracle's own composite with the colour replaced by z: ``depth_forward`` draws the colour (z / zs, 0, 0) with zs a
power of two above every z, so the composite stays below the min(c, 1) clamp and scaling back by zs is exact.  Both channels
use the same weights, so the backward is the sum of the oracle's colour backward and the same backward of that depth-as-colour
image; its colour gradient is sum_pixels w g_z = dL/dz (times zs), which joins the view-space z gradient of the position and the
camera.

``render_forward_backward`` runs exact_grad_oracle's composition (and through it filter3d_oracle's and aa_oracle's) with two of
the oracle's public stages intercepted for the duration of the call: ``oracle.project`` to keep z, and
``oracle.rasterize_backward`` to render D and add the depth-as-colour backward.  The oracle library itself is not changed, and
with ``render_depth=False`` the composition runs untouched.
"""
import contextlib

import numpy as np

import oracle
from tests import exact_grad_oracle as ex


def _zscale(z):
    m = float(np.abs(z).max()) if z.size else 1.0
    return 2.0 ** (int(np.ceil(np.log2(max(m, 1e-30)))) + 1)


def _depth_colour(z, dt):
    zs = _zscale(z)
    col = np.zeros((1, 3, z.shape[-1]), dt)
    col[0, 0] = (z / zs).astype(dt)
    return col, zs


def depth_forward(sorted_pid, ranges, ndc, inv_cov2d, opacity, z, H, W, th, tw, specific_tiles=None):
    """D [V,1,Hp,Wp] of the records (ndc, inv_cov2d, opacity) with view-space z [N] over the given tile lists."""
    col, zs = _depth_colour(z, ndc.dtype)
    img = oracle.rasterize_forward(sorted_pid, ranges, ndc, inv_cov2d, col, opacity, specific_tiles, H, W, th, tw)[0]
    return img[:, :1] * zs


def _pad(g, shape):
    full = np.zeros(shape, g.dtype)
    full[..., :g.shape[-2], :g.shape[-1]] = g
    return full


@contextlib.contextmanager
def _depth_stages(d_depth_fn, rec):
    project0, backward0 = oracle.project, oracle.rasterize_backward

    def project(*a, **k):
        rec["inter"] = project0(*a, **k)
        return rec["inter"]

    def rasterize_backward(sorted_pid, ranges, ndc, inv, color, opacity, tiles, T, last, d_img, d_trans, scaler, H, W, th, tw,
                           **kw):
        z = rec["inter"]["view_pos"][0, 2]
        colz, zs = _depth_colour(z, ndc.dtype)
        D = oracle.rasterize_forward(sorted_pid, ranges, ndc, inv, colz, opacity, tiles, H, W, th, tw)[0][:, :1] * zs
        rec["depth"] = D
        gz = gt = None
        if d_depth_fn is not None:
            gz, gt = d_depth_fn(D[..., :H, :W], T[..., :H, :W])
        s = 1.0 if scaler is None else float(np.asarray(scaler).reshape(-1)[0])
        if gt is not None:              # the colour pass takes the transmittance gradient (its inputs are divided by the scaler)
            gt = (_pad(np.asarray(gt, T.dtype), T.shape) / s).astype(T.dtype)
            d_trans = gt if d_trans is None else d_trans + gt
        out = list(backward0(sorted_pid, ranges, ndc, inv, color, opacity, tiles, T, last, d_img, d_trans, scaler, H, W, th, tw, **kw))
        rec["dz"] = np.zeros(z.shape, ndc.dtype)
        if gz is not None:
            dz_img = np.zeros_like(d_img)
            dz_img[:, :1] = _pad(np.asarray(gz, d_img.dtype), T.shape) * zs
            zn, zc, zcol, zop, _, _ = backward0(sorted_pid, ranges, ndc, inv, colz, opacity, tiles, T, last, dz_img, None, None,
                                                H, W, th, tw)
            out[0], out[1], out[3] = out[0] + zn, out[1] + zc, out[3] + zop
            rec["dz"] = zcol[0, 0] / zs
        return tuple(out)

    oracle.project, oracle.rasterize_backward = project, rasterize_backward
    try:
        yield
    finally:
        oracle.project, oracle.rasterize_backward = project0, backward0


def render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, render_depth=False, d_depth_fn=None,
                            **kw):
    """exact_grad_oracle.render_forward_backward (kw: true_sigmoid_grad, antialiased, filter_3d, exact_grad, lists, freeze), plus
    with render_depth the depth D ("depth" [V,1,H,W], "depth_padded") and, when d_depth_fn(D, T) -> (dL/dD, dL/dT or None) is
    given, the depth loss's gradients added to every parameter gradient; "dz" [N] is dL/dz of each visible Gaussian."""
    if not render_depth:
        return ex.render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, **kw)
    rec = {}
    with _depth_stages(d_depth_fn, rec):
        out = ex.render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn, **kw)
    H, W = img_hw
    dz = rec["dz"]
    Vm = np.asarray(camera["view"], np.float64).reshape(4, 4)
    gx = out["grads"]["xyz"]
    out["grads"] = dict(out["grads"], xyz=(gx.astype(np.float64) + (Vm[:3, 2][:, None] * dz).reshape(gx.shape)).astype(gx.dtype))
    out.update(depth=rec["depth"][..., :H, :W], depth_padded=rec["depth"], dz=dz)
    return out


def camera_backward(params, out, camera, img_hw, sh_degree=None, exact_grad=False):
    """exact_grad_oracle.camera_backward plus the depth term d view[k][2] += sum_i p~_ik dz_i (fp64) -> (d_view, d_proj)."""
    d_view, d_proj = ex.camera_backward(params, out, camera, img_hw, sh_degree=sh_degree, exact_grad=exact_grad)
    if "dz" not in out:
        return d_view, d_proj
    ids = out["visible_chunk_id"]
    p = params["xyz"][:, ids, :].reshape(3, -1).astype(np.float64)
    dz = np.asarray(out["dz"], np.float64)
    d_view = np.array(d_view, np.float64)
    d_view[:3, 2] += p @ dz
    d_view[3, 2] += dz.sum()
    return d_view, np.array(d_proj, np.float64)
