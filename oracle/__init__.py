"""CPU oracle for the LiteGS render hot path -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this package.  The product (``litegs_b200``) never does: it fails loudly when its CUDA
library is missing instead of falling back to anything here.

The arithmetic lives in ``oracle_core.h`` (plain C, compiled for fp32 and fp64); this module is the
numpy/ctypes veneer.  Function names and argument order mirror the reference's ``litegs_fused`` pybind
module (``GR/ext_cuda.cpp:9-35``) so that parity tests read like calls into the reference.

Parity pinning: the reference ships no CPU path and no golden vectors for this path (SURVEY.md 8c).
The oracle is pinned against the reference's own CUDA kernels (``oracle/build_ref.py`` builds them
into ``oracle/_ref``; ``tests/golden/make_golden.py`` runs them on an H100 and writes fixtures).
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    """Compile liborc.so with the committed Makefile (gcc, OpenMP when available)."""
    so = os.path.join(_HERE, "liborc.so")
    srcs = [os.path.join(_HERE, f) for f in ("oracle.c", "oracle_core.h", "Makefile")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s", "liborc.so"])
    return so


def lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.orc_num_threads.restype = ctypes.c_int
    return _LIB


def num_threads() -> int:
    return int(lib().orc_num_threads())


def set_num_threads(n: int) -> None:
    lib().orc_set_num_threads(int(n))


def _suf(dt) -> str:
    dt = np.dtype(dt)
    if dt == np.float32:
        return "_f32"
    if dt == np.float64:
        return "_f64"
    raise TypeError(f"oracle supports float32/float64, got {dt}")


def _c(a, dt=None):
    a = np.ascontiguousarray(a, dtype=dt)
    return a


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _real(dt):
    return ctypes.c_float if np.dtype(dt) == np.float32 else ctypes.c_double


def _call(name, dt, *args):
    fn = getattr(lib(), name + _suf(dt))
    fn.restype = None
    conv = []
    for a in args:
        if isinstance(a, np.ndarray):
            conv.append(_p(a))
        elif a is None:
            conv.append(None)
        elif isinstance(a, float):
            conv.append(_real(dt)(a))
        elif isinstance(a, (int, np.integer, bool)):
            conv.append(ctypes.c_int(int(a)))
        else:
            conv.append(a)
    fn(*conv)


def _valid(valid_length, n):
    if valid_length is None:
        return int(n)
    return int(min(int(np.asarray(valid_length).reshape(-1)[0]), n))


# ---------------------------------------------------------------------------------------------
# litegs_fused-shaped entry points
# ---------------------------------------------------------------------------------------------

def frustum_culling_aabb(aabb_origin, aabb_ext, frustumplane):
    """GR/compact.cu:503-551 -> (visibility bool[M], visible_num int32[1], visible_chunk_id int64[count])."""
    dt = aabb_origin.dtype
    o, e, f = _c(aabb_origin), _c(aabb_ext, dt), _c(frustumplane, dt)
    M, V = o.shape[1], f.shape[0]
    vis = np.zeros(M, np.uint8)
    ids = np.zeros(M, np.int64)
    cnt = np.zeros(1, np.int32)
    _call("orc_frustum_culling_aabb", dt, o, e, f, M, V, vis, ids, cnt)
    return vis.astype(bool), cnt, ids[: int(cnt[0])].copy()


def cull_compact_activate(sh_degree, visible_chunk_id, visible_chunks_num, view_matrix,
                          position, scale, rotation, sh_base, sh_rest, opacity):
    """GR/compact.cu:983-1085.  Returns activated [4|3|4,A,S], color [V,3,A,S], opacity [1,A,S]."""
    dt = position.dtype
    ids = _c(visible_chunk_id, np.int64)
    nvis = _valid(visible_chunks_num, ids.shape[0])
    view = _c(view_matrix, dt)
    V = view.shape[0]
    C, S = position.shape[-2:]
    A = ids.shape[0]
    apos = np.zeros((4, A, S), dt); ascale = np.zeros((3, A, S), dt); arot = np.zeros((4, A, S), dt)
    color = np.zeros((V, 3, A, S), dt); aop = np.zeros((1, A, S), dt)
    _call("orc_cull_compact_activate", dt, sh_degree, ids, nvis, view, V, _c(position), _c(scale, dt),
          _c(rotation, dt), _c(sh_base, dt), _c(sh_rest, dt), _c(opacity, dt), C, S, A,
          apos, ascale, arot, color, aop)
    return apos, ascale, arot, color, aop


def activate_backward(sh_degree, visible_chunk_id, visible_chunks_num, view_matrix,
                      position, scale, rotation, sh_base, sh_rest, opacity,
                      g_pos, g_scale, g_rot, g_color, g_opacity, true_sigmoid_grad=False):
    """GR/compact.cu:1087-1212 -> compacted grads (pos[3], scale[3], rot[4], sh0[1,3], sh_rest[R,3], opacity[1])."""
    dt = position.dtype
    ids = _c(visible_chunk_id, np.int64)
    nvis = _valid(visible_chunks_num, ids.shape[0])
    view = _c(view_matrix, dt)
    V = view.shape[0]
    C, S = position.shape[-2:]
    A = ids.shape[0]
    R = sh_rest.shape[0]
    o_pos = np.zeros((3, A, S), dt); o_scale = np.zeros((3, A, S), dt); o_rot = np.zeros((4, A, S), dt)
    o_sh0 = np.zeros((1, 3, A, S), dt); o_shr = np.zeros((R, 3, A, S), dt); o_op = np.zeros((1, A, S), dt)
    _call("orc_activate_backward", dt, sh_degree, ids, nvis, view, V, _c(position), _c(scale, dt), _c(rotation, dt),
          _c(opacity, dt), C, S, A, R, int(bool(true_sigmoid_grad)),
          _c(g_pos, dt), _c(g_scale, dt), _c(g_rot, dt), _c(g_color, dt), _c(g_opacity, dt),
          o_pos, o_scale, o_rot, o_sh0, o_shr, o_op)
    return o_pos, o_scale, o_rot, o_sh0, o_shr, o_op


def mvp_transform_forward(world_position, view_matrix, proj_matrix, valid_length=None):
    """GR/transform.cu:440-470 -> (view_pos [V,4,N], ndc_pos [V,4,N])."""
    dt = world_position.dtype
    p = _c(world_position); N = p.shape[1]; V = view_matrix.shape[0]
    vp = np.zeros((V, 4, N), dt); ndc = np.zeros((V, 4, N), dt)
    _call("orc_mvp_forward", dt, p, _c(view_matrix, dt), _c(proj_matrix, dt), V, N, _valid(valid_length, N), vp, ndc)
    return vp, ndc


def mvp_transform_backward(grad_ndc, grad_view, view_matrix, proj_matrix, view_pos, valid_length=None):
    """GR/transform.cu:562-598 -> d position [4,N]."""
    dt = view_pos.dtype
    V, _, N = view_pos.shape
    out = np.zeros((4, N), dt)
    _call("orc_mvp_backward", dt, _c(grad_ndc, dt), _c(grad_view, dt), _c(view_matrix, dt), _c(proj_matrix, dt),
          _c(view_pos), V, N, _valid(valid_length, N), out)
    return out


def createTransformMatrix_forward(quaternion, scale, valid_length=None):
    """GR/transform.cu:129-149 -> [3,3,N]."""
    dt = quaternion.dtype; N = quaternion.shape[1]
    T = np.zeros((3, 3, N), dt)
    _call("orc_transform_forward", dt, _c(quaternion), _c(scale, dt), N, _valid(valid_length, N), T)
    return T


def createTransformMatrix_backward(grad_T, quaternion, scale, valid_length=None):
    """GR/transform.cu:231-256 -> (d quaternion [4,N], d scale [3,N])."""
    dt = quaternion.dtype; N = quaternion.shape[1]
    gq = np.zeros((4, N), dt); gs = np.zeros((3, N), dt)
    _call("orc_transform_backward", dt, _c(grad_T, dt), _c(quaternion), _c(scale, dt), N, _valid(valid_length, N), gq, gs)
    return gq, gs


def jacobianRayspace(view_pos, proj_matrix, output_h, output_w, valid_length=None):
    """GR/transform.cu:54-90 -> [V,3,3,N]."""
    dt = view_pos.dtype; V, _, N = view_pos.shape
    J = np.zeros((V, 3, 3, N), dt)
    _call("orc_jacobian_rayspace", dt, _c(view_pos), _c(proj_matrix, dt), V, N, _valid(valid_length, N),
          int(output_h), int(output_w), J)
    return J


def createCov2dDirectly_forward(J, view_matrix, transform_matrix, valid_length=None):
    """GR/transform.cu:783-821 -> [V,2,2,N]."""
    dt = J.dtype; V = J.shape[0]; N = J.shape[3]
    cov = np.zeros((V, 2, 2, N), dt)
    _call("orc_cov2d_forward", dt, _c(J), _c(view_matrix, dt), _c(transform_matrix, dt), V, N, _valid(valid_length, N), cov)
    return cov


def createCov2dDirectly_backward(grad_cov, J, view_matrix, transform_matrix, valid_length=None):
    """GR/transform.cu:892-927 -> d transform [3,3,N]."""
    dt = J.dtype; V = J.shape[0]; N = J.shape[3]
    gT = np.zeros((3, 3, N), dt)
    _call("orc_cov2d_backward", dt, _c(grad_cov, dt), _c(J), _c(view_matrix, dt), _c(transform_matrix, dt), V, N,
          _valid(valid_length, N), gT)
    return gT


def eigh_and_inv_2x2matrix_forward(cov2d, valid_length=None):
    """GR/transform.cu:1456-1487 -> (val [V,2,N], vec [V,2,2,N], inv [V,2,2,N])."""
    dt = cov2d.dtype; V = cov2d.shape[0]; N = cov2d.shape[3]
    val = np.zeros((V, 2, N), dt); vec = np.zeros((V, 2, 2, N), dt); inv = np.zeros((V, 2, 2, N), dt)
    _call("orc_eigh_inv_forward", dt, _c(cov2d), V, N, _valid(valid_length, N), val, vec, inv)
    return val, vec, inv


def inv_2x2matrix_backward(inv_matrix, grad_inv, valid_length=None):
    """GR/transform.cu:1489-1518 -> d matrix [V,2,2,N]."""
    dt = inv_matrix.dtype; V = inv_matrix.shape[0]; N = inv_matrix.shape[3]
    out = np.zeros((V, 2, 2, N), dt)
    _call("orc_inv2x2_backward", dt, _c(inv_matrix), _c(grad_inv, dt), V, N, _valid(valid_length, N), out)
    return out


def sh2rgb_forward(degree, sh_base, sh_rest, dirs):
    """GR/transform.cu:1039-1086 -> rgb [V,3,N]."""
    dt = sh_base.dtype; V = dirs.shape[0]; N = dirs.shape[2]
    rgb = np.zeros((V, 3, N), dt)
    _call("orc_sh2rgb_forward", dt, degree, _c(sh_base), _c(sh_rest, dt), _c(dirs, dt), V, N, rgb)
    return rgb


def sh2rgb_backward(degree, rgb_grad, sh_rest_dim, dirs, sh_base=None, sh_rest=None):
    """GR/transform.cu:1298-1361 -> (d sh_base [1,3,N], d sh_rest [R,3,N], d dir = 0)."""
    dt = rgb_grad.dtype; V = dirs.shape[0]; N = dirs.shape[2]
    g0 = np.zeros((1, 3, N), dt); gr = np.zeros((sh_rest_dim, 3, N), dt)
    _call("orc_sh2rgb_backward", dt, degree, _c(rgb_grad), int(sh_rest_dim), _c(dirs, dt), V, N, g0, gr)
    return g0, gr, np.zeros_like(dirs)


def get_allocate_size(ndc, view_space_z, inv_cov2d, opacity, height, width, tile_h, tile_w, valid_length=None,
                      exact_tile_bound=True):
    """GR/binning.cu:398-440 -> (left_up i32[V,2,N], right_down i32[V,2,N], allocate_size i32[V,N]).

    exact_tile_bound=False: the reference's last tile row / column, floor((bbox_max + T - 1) / T), which drops a tile the
    ellipse reaches by less than a pixel (DESIGN.md section 7, D14); True: floor((bbox_max + T) / T)."""
    dt = ndc.dtype; V = ndc.shape[0]; N = ndc.shape[2]
    lu = np.zeros((V, 2, N), np.int32); rd = np.zeros((V, 2, N), np.int32); al = np.zeros((V, N), np.int32)
    _call("orc_get_allocate_size", dt, _c(ndc), _c(view_space_z, dt), _c(inv_cov2d, dt), _c(opacity, dt),
          V, N, _valid(valid_length, N), int(height), int(width), int(tile_h), int(tile_w), int(bool(exact_tile_bound)), lu, rd, al)
    return lu, rd, al


def create_table(ndc, inv_cov2d, opacity, offset, depth_sorted_pointid, allocate, height, width, tile_h, tile_w,
                 exact_tile_bound=True):
    """GR/binning.cu:123-226 with the table size given explicitly -> (sorted_tileId, sorted_pointId) i32[V,allocate].
    exact_tile_bound: as in get_allocate_size; the offsets must come from counts made with the same rule."""
    dt = ndc.dtype; V = ndc.shape[0]; N = ndc.shape[2]
    cap = int(allocate)
    keys = np.zeros((V, cap), np.int32); vals = np.zeros((V, cap), np.int32)
    _call("orc_create_table", dt, _c(ndc), _c(inv_cov2d, dt), _c(opacity, dt), _c(offset, np.int32),
          _c(depth_sorted_pointid, np.int64), V, N, cap, int(height), int(width), int(tile_h), int(tile_w),
          int(bool(exact_tile_bound)), keys, vals)
    return keys, vals


def tileRange(table_tileId, max_tileId, fix_last=True):
    """GR/binning.cu:267-287 -> i32[V,max_tileId+2]; fix_last=False reproduces SURVEY Q3 bit for bit."""
    k = _c(table_tileId, np.int32); V, L = k.shape
    out = np.zeros((V, int(max_tileId) + 2), np.int32)
    _call("orc_tile_range", np.float32, k, V, L, int(max_tileId), int(bool(fix_last)), out)
    return out


def padded_hw(img_h, img_w, tile_h, tile_w):
    gy = (img_h + tile_h - 1) // tile_h; gx = (img_w + tile_w - 1) // tile_w
    return gy * tile_h, gx * tile_w


def rasterize_forward(sorted_points, start_index, ndc, cov2d_inv, color, opacity, specific_tiles,
                      img_h, img_w, tile_h, tile_w, enable_statistic=False, enable_trans=False,
                      enable_depth=False, fragile_eps=1e-5):
    """GR/raster.cu:386-492 in fp32/fp64 (no half quantisation).

    Returns (img, T, last_contributor, fragment_count, fragment_weight_sum, fragile_mask)."""
    dt = ndc.dtype; V = ndc.shape[0]; N = ndc.shape[2]
    sp = _c(sorted_points, np.int32); cap = sp.shape[1]
    Hp, Wp = padded_hw(img_h, img_w, tile_h, tile_w)
    img = np.zeros((V, 3, Hp, Wp), dt); T = np.ones((V, 1, Hp, Wp), dt); last = np.zeros((V, 1, Hp, Wp), np.int16)
    fc = np.zeros((V, 1, N), np.int32); fw = np.zeros((V, 1, N), dt)
    frag = np.zeros((V, Hp, Wp), np.uint8)
    tiles = None if specific_tiles is None else _c(specific_tiles, np.int32)
    _call("orc_raster_forward", dt, sp, _c(start_index, np.int32), _c(ndc), _c(cov2d_inv, dt), _c(color, dt),
          _c(opacity, dt), tiles, 0 if tiles is None else tiles.shape[1], V, N, cap,
          int(img_h), int(img_w), int(tile_h), int(tile_w), img, T, last,
          fc if enable_statistic else None, fw if enable_statistic else None, frag, float(fragile_eps))
    return img, T, last, fc, fw, frag.astype(bool)


def rasterize_backward(sorted_points, start_index, ndc, cov2d_inv, color, opacity, specific_tiles,
                       final_T, last_contributor, d_img, d_trans, grad_inv_scaler,
                       img_h, img_w, tile_h, tile_w, enable_statistic=False, err_mode="reference"):
    """GR/raster.cu:917-1037 -> (d_ndc [V,4,N], d_cov2d_inv [V,2,2,N], d_color [V,3,N], d_opacity [1,N], err_sum, err_sq).

    err_mode: "reference" = the lane-running recurrence of GR/raster.cu:779-784 (orc_raster_err_square_ref),
    "pixel" = sum over pixels of (G dalpha)^2."""
    dt = ndc.dtype; V = ndc.shape[0]; N = ndc.shape[2]
    sp = _c(sorted_points, np.int32); cap = sp.shape[1]
    d_ndc = np.zeros((V, 4, N), dt); d_cov = np.zeros((V, 2, 2, N), dt); d_col = np.zeros((V, 3, N), dt)
    d_op = np.zeros((1, N), dt); err = np.zeros((V, 1, N), dt)
    tiles = None if specific_tiles is None else _c(specific_tiles, np.int32)
    scaler = 1.0 if grad_inv_scaler is None else float(np.asarray(grad_inv_scaler).reshape(-1)[0])
    _call("orc_raster_backward", dt, sp, _c(start_index, np.int32), _c(ndc), _c(cov2d_inv, dt), _c(color, dt),
          _c(opacity, dt), tiles, 0 if tiles is None else tiles.shape[1], _c(final_T, dt),
          _c(last_contributor, np.int16), _c(d_img, dt), None if d_trans is None else _c(d_trans, dt), scaler,
          V, N, cap, int(img_h), int(img_w), int(tile_h), int(tile_w), d_ndc, d_cov, d_col, d_op,
          err if enable_statistic else None)
    if enable_statistic and err_mode == "reference":
        _call("orc_raster_err_square_ref", dt, sp, _c(start_index, np.int32), _c(ndc), _c(cov2d_inv, dt), _c(color, dt),
              _c(opacity, dt), tiles, 0 if tiles is None else tiles.shape[1], _c(final_T, dt),
              _c(last_contributor, np.int16), _c(d_img, dt), None if d_trans is None else _c(d_trans, dt),
              V, N, cap, int(img_h), int(img_w), int(tile_h), int(tile_w), err)
    return d_ndc, d_cov, d_col, d_op, np.zeros((V, 1, N), dt), err


def adamUpdate(param, grad, exp_avg, exp_avg_sq, visible_index, valid_length, lr, b1, b2, eps):
    """GR/compact.cu:377-417, chunk ([R,C,S]) form; in place on param/exp_avg/exp_avg_sq."""
    dt = param.dtype
    R, C, S = param.shape
    ids = _c(visible_index, np.int64); A = grad.shape[1]
    nvis = _valid(valid_length, ids.shape[0])
    assert param.flags.c_contiguous and exp_avg.flags.c_contiguous and exp_avg_sq.flags.c_contiguous
    _call("orc_adam_chunk", dt, param, _c(grad, dt), exp_avg, exp_avg_sq, ids, nvis, R, C, S, A,
          float(lr), float(b1), float(b2), float(eps))


# ---------------------------------------------------------------------------------------------
# composed pipeline (the Python glue of litegs/render/__init__.py:50-94 + wrapper.py:718-763)
# ---------------------------------------------------------------------------------------------

def binning(ndc, view_depth, inv_cov2d, opacity, valid_length, img_hw, tile_hw, fix_last=True):
    """wrapper.py:718-763: count -> stable depth sort -> inclusive scan -> emit -> tile sort -> ranges.
    fix_last=False reproduces the reference's tables: the last populated tile's range left open (SURVEY Q3) and the
    reference's tile rectangle (exact_tile_bound=False, DESIGN.md section 7, D14), as litegs_fused.CONFIG["fix_last_tile"]."""
    exact_tile_bound = bool(fix_last)
    H, W = img_hw; th, tw = tile_hw
    gy = (H + th - 1) // th; gx = (W + tw - 1) // tw
    _, _, alloc = get_allocate_size(ndc, view_depth, inv_cov2d, opacity, H, W, th, tw, valid_length, exact_tile_bound)
    order = np.argsort(view_depth, axis=-1, kind="stable").astype(np.int64)
    sorted_alloc = np.take_along_axis(alloc, order, axis=-1)
    prefix = np.cumsum(sorted_alloc, axis=-1, dtype=np.int64).astype(np.int32)
    total = max(int(prefix[:, -1].max()), 1)
    keys, vals = create_table(ndc, inv_cov2d, opacity, prefix, order, total, H, W, th, tw, exact_tile_bound)
    ranges = tileRange(keys, gx * gy, fix_last=fix_last)
    return ranges, vals, (alloc != 0), keys


def project(xyz, scale, rot, view_matrix, proj_matrix, img_hw, valid_length=None):
    """render/__init__.py:57-62: MVP, S.R, J, cov2d, inverse."""
    vp, ndc = mvp_transform_forward(xyz, view_matrix, proj_matrix, valid_length)
    T = createTransformMatrix_forward(rot, scale, valid_length)
    J = jacobianRayspace(vp, proj_matrix, img_hw[0], img_hw[1], valid_length)
    cov = createCov2dDirectly_forward(J, view_matrix, T, valid_length)
    _, _, inv = eigh_and_inv_2x2matrix_forward(cov, valid_length)
    return dict(view_pos=vp, ndc=ndc, T=T, J=J, cov2d=cov, inv_cov2d=inv)


def project_backward(inter, d_ndc, d_inv_cov, scale, rot, view_matrix, proj_matrix, valid_length=None):
    """Backward chain of wrapper.py:588-592,404-407,190-193,278-285 -> (d xyz [4,N], d scale [3,N], d rot [4,N])."""
    g_cov = inv_2x2matrix_backward(inter["inv_cov2d"], d_inv_cov, valid_length)
    g_cov = np.nan_to_num(g_cov, nan=0.0)
    gT = createCov2dDirectly_backward(g_cov, inter["J"], view_matrix, inter["T"], valid_length)
    gq, gs = createTransformMatrix_backward(gT, rot, scale, valid_length)
    gp = mvp_transform_backward(d_ndc, np.zeros_like(inter["view_pos"]), view_matrix, proj_matrix,
                                inter["view_pos"], valid_length)
    return gp, gs, gq


def render_forward_backward(params, chunk_aabb, camera, img_hw, tile_hw, sh_degree, d_img_fn,
                            true_sigmoid_grad=False, fix_last=True):
    """End-to-end oracle for one view: render_preprocess + render + backward to the six parameter grads.

    params: dict xyz[3,C,S] scale rot sh_0[1,3,C,S] sh_rest[R,3,C,S] opacity[1,C,S];
    chunk_aabb: (origin[3,C], extend[3,C]); camera: dict view[1,4,4] proj[1,4,4] frustumplane[1,6,4];
    d_img_fn(img_cropped) -> dL/dimg (same shape).  Returns dict with image, grads and intermediates."""
    H, W = img_hw; th, tw = tile_hw
    vis, nvis, ids = frustum_culling_aabb(chunk_aabb[0], chunk_aabb[1], camera["frustumplane"])
    act = cull_compact_activate(sh_degree, ids, nvis, camera["view"], params["xyz"], params["scale"], params["rot"],
                                params["sh_0"], params["sh_rest"], params["opacity"])
    flat = [a.reshape(*a.shape[:-2], -1) for a in act]
    xyz, scale, rot, color, opacity = flat
    inter = project(xyz, scale, rot, camera["view"], camera["proj"], img_hw)
    ranges, sorted_pid, visible, _ = binning(inter["ndc"], inter["view_pos"][:, 2], inter["inv_cov2d"], opacity,
                                             None, img_hw, tile_hw, fix_last)
    img, T, last, _, _, fragile = rasterize_forward(sorted_pid, ranges, inter["ndc"], inter["inv_cov2d"], color,
                                                    opacity, None, H, W, th, tw)
    img_c = np.clip(img[..., :H, :W], 0, 1)
    g = d_img_fn(img_c)
    g_full = np.zeros_like(img)
    # clamp(0,1) backward: gradient passes where 0 <= img <= 1 (render/__init__.py:87)
    mask = (img[..., :H, :W] >= 0) & (img[..., :H, :W] <= 1)
    g_full[..., :H, :W] = g * mask
    gmax = np.abs(g_full).max()
    gmax = gmax if gmax > 0 else 1.0
    d_ndc, d_cov, d_col, d_op, _, _ = rasterize_backward(sorted_pid, ranges, inter["ndc"], inter["inv_cov2d"], color,
                                                         opacity, None, T, last, (g_full / gmax).astype(img.dtype), None,
                                                         gmax, H, W, th, tw)
    gp, gs, gq = project_backward(inter, d_ndc, d_cov, scale, rot, camera["view"], camera["proj"])
    A, S = act[0].shape[-2:]
    shp = lambda a: a.reshape(*a.shape[:-1], A, S)
    grads = activate_backward(sh_degree, ids, nvis, camera["view"], params["xyz"], params["scale"], params["rot"],
                              params["sh_0"], params["sh_rest"], params["opacity"],
                              shp(gp), shp(gs), shp(gq), shp(d_col), shp(d_op), true_sigmoid_grad)
    return dict(img=img_c, img_padded=img, T=T, last=last, fragile=fragile, visible_chunk_id=ids,
                grads=dict(zip(("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity"), grads)),
                inter=inter, ranges=ranges, sorted_pid=sorted_pid, color=color, opacity=opacity,
                d_ndc=d_ndc, d_cov=d_cov, d_col=d_col, d_op=d_op)


# ---------------------------------------------------------------------------------------------
# fused_ssim-shaped entry points (fused_ssim/ext.cpp:4-9)
# ---------------------------------------------------------------------------------------------

def _ssim_forward(l1_mode, ssim_weight, C1, C2, img1, img2, train):
    dt = img1.dtype
    a, b = _c(img1), _c(img2, dt)
    B, CH, H, W = a.shape
    out = np.zeros_like(a)
    d = [np.zeros_like(a) for _ in range(3)] if train else [None, None, None]
    _call("orc_ssim_forward", dt, a, b, B, CH, H, W, float(C1), float(C2), int(l1_mode), float(ssim_weight), out, *d)
    e = np.zeros((0,), dt)
    return (out, d[0], d[1], d[2]) if train else (out, e, e, e)


def _ssim_backward(l1_mode, ssim_weight, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    dt = img1.dtype
    a = _c(img1)
    B, CH, H, W = a.shape
    out = np.zeros_like(a)
    _call("orc_ssim_backward", dt, a, _c(img2, dt), _c(dL_dmap, dt), _c(dm_dmu1, dt), _c(dm_dsigma1_sq, dt), _c(dm_dsigma12, dt),
          B, CH, H, W, int(l1_mode), float(ssim_weight), out)
    return out


def fusedssim(C1, C2, img1, img2, train=True):
    """ssim.cu:444-479 -> (ssim_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)."""
    return _ssim_forward(0, 0.0, C1, C2, img1, img2, train)


def fusedssim_backward(C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    """ssim.cu:487-524 -> dL/dimg1."""
    return _ssim_backward(0, 0.0, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)


def fusedl1ssim_loss(ssim_weight, C1, C2, img1, img2, train=True):
    """ssim.cu:855-900 -> (loss_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)."""
    return _ssim_forward(1, ssim_weight, C1, C2, img1, img2, train)


def fusedl1ssim_loss_backward(ssim_weight, C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    """ssim.cu:904-942 -> dL/dimg1."""
    return _ssim_backward(1, ssim_weight, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)
