"""Host-side mirror of the reference's ``litegs_fused`` pybind module, above the C ABI.

Same names, same positional arguments, same return lists as ``GR/ext_cuda.cpp:9-35`` (headers
``GR/raster.h``, ``GR/binning.h``, ``GR/compact.h``, ``GR/transform.h``), so the reference's
``litegs/utils/wrapper.py`` and ``litegs/render/__init__.py`` run on it unchanged once it is registered
as ``sys.modules['litegs_fused']`` (see ``litegs_fused.py`` at the repo root and INTEGRATION.md).

PyTorch is used here for what the reference's C++ host code uses ATen for: output allocation from the
caching allocator, the current stream, device guards.  All arithmetic happens in liblitegs_b200.so.
The reference's host code is C++; this mirror is Python + ctypes because the image has no way to ship
a second toolchain-specific binding, and every entry point is a single C call.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Optional

import torch

from . import _lib

_F32, _I32, _I64 = torch.float32, torch.int32, torch.int64

# Deviations that can be switched back to bit-compatibility with the reference (SURVEY Q3, Q15)
CONFIG = {
    # close the last populated tile's range (reference leaves it empty, Q3) and keep the tile a splat reaches by less than a
    # pixel (the reference drops it, DESIGN.md section 7, D14); False = the reference's tile tables bit for bit
    "fix_last_tile": True,
    "true_sigmoid_grad": False,     # False = reference's d_o * sigma(x) on the cluster path
    "tile_order": os.environ.get("LGS_TILE_ORDER", "1") != "0",   # fused pipeline: backward tiles launched heaviest-first (lgs_tile_order)
}


def _ptr(t: Optional[torch.Tensor]):
    """Raw device address for a c_void_p argument (ctypes converts the int; None is NULL)."""
    return None if t is None else t.data_ptr()


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class _OnDevice:
    """`with _on(dev):` -- torch.cuda.device(dev) only when dev is not already current (the context manager costs ~10 us,
    and the common case is one process per GPU)."""
    __slots__ = ("ctx",)

    def __init__(self, dev):
        self.ctx = None if torch.cuda.current_device() == (dev.index if dev.index is not None else torch.cuda.current_device()) \
            else torch.cuda.device(dev)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *a):
        if self.ctx is not None:
            return self.ctx.__exit__(*a)
        return False


_on = _OnDevice


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (litegs_b200 has no CPU path)")
    if t.dtype != _F32:
        raise RuntimeError(f"{name}: expected float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _asc(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dtype != dtype:
        raise RuntimeError(f"{name}: expected {dtype}, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _vl(valid_length: Optional[torch.Tensor]):
    if valid_length is None:
        return None
    return _asc(valid_length, _I32, "valid_length")


def _tiles(img_h, img_w, th, tw):
    gy = (int(img_h) + th - 1) // th
    gx = (int(img_w) + tw - 1) // tw
    return gx, gy


# ---------------------------------------------------------------------------------------------------
# chunk culling / activation
# ---------------------------------------------------------------------------------------------------

def frustum_culling_aabb(aabb_origin, aabb_ext, frustumplane, feedback_buffer_arg=None, data_idx_arg=None):
    """GR/compact.cu:503-551 -> [visibility bool[M], visible_chunks_num i32[1], visible_chunk_id i64[pred]].

    Sizing policy as the reference: 1.2x the count this frame had last epoch (pinned CPU feedback
    buffer, refreshed with an async D2H copy), else one blocking read-back."""
    o = _f32c(aabb_origin, "aabb_origin"); e = _f32c(aabb_ext, "aabb_ext"); f = _f32c(frustumplane, "frustumplane")
    M, V = o.shape[1], f.shape[0]
    dev = o.device
    with torch.cuda.device(dev):
        vis = torch.empty(M, dtype=torch.bool, device=dev)
        num = torch.zeros(1, dtype=_I32, device=dev)
        ids = torch.arange(M, dtype=_I64, device=dev)
        _lib.call("lgs_frustum_culling_aabb", _ptr(o), _ptr(e), _ptr(f), M, V, _ptr(vis), _ptr(num), _ptr(ids), _stream(dev))
        pred = 0
        if feedback_buffer_arg is not None and data_idx_arg is not None:
            for i in range(data_idx_arg.shape[0]):
                idx = int(data_idx_arg[i])
                pred = max(pred, int(feedback_buffer_arg[idx]))
                feedback_buffer_arg[idx:idx + 1].copy_(num, non_blocking=True)
        pred = int(1.2 * pred)
        if pred <= 0:
            pred = int(num.item())
        pred = min(pred, M)
    return [vis, num, ids[:pred]]


def cull_compact_activate(sh_degree, visible_chunk_id, visible_chunks_num, view_matrix,
                          position, scale, rotation, sh_base, sh_rest, opacity):
    """GR/compact.cu:983-1085."""
    ids = _asc(visible_chunk_id, _I64, "visible_chunk_id"); num = _asc(visible_chunks_num, _I32, "visible_chunks_num")
    view = _f32c(view_matrix, "view_matrix")
    pos = _f32c(position, "position"); sc = _f32c(scale, "scale"); rot = _f32c(rotation, "rotation")
    s0 = _f32c(sh_base, "sh_base"); sr = _f32c(sh_rest, "sh_rest"); op = _f32c(opacity, "opacity")
    K = (int(sh_degree) + 1) ** 2
    if sr.shape[0] < K - 1:
        raise RuntimeError(f"sh_rest has {sr.shape[0]} rows, sh_degree {sh_degree} needs {K - 1}")
    C, S = pos.shape[-2:]
    A, V = ids.shape[0], view.shape[0]
    dev = pos.device
    with torch.cuda.device(dev):
        apos = torch.empty((4, A, S), dtype=_F32, device=dev)
        asc = torch.empty((3, A, S), dtype=_F32, device=dev)
        arot = torch.empty((4, A, S), dtype=_F32, device=dev)
        color = torch.empty((V, 3, A, S), dtype=_F32, device=dev)
        aop = torch.empty((1, A, S), dtype=_F32, device=dev)
        _lib.call("lgs_cull_compact_activate", int(sh_degree), _ptr(ids), _ptr(num), _ptr(view), V, _ptr(pos), _ptr(sc),
                  _ptr(rot), _ptr(s0), _ptr(sr), _ptr(op), C, S, A, _ptr(apos), _ptr(asc), _ptr(arot), _ptr(color),
                  _ptr(aop), _stream(dev))
    return [apos, asc, arot, color, aop]


def activate_backward(sh_degree, visible_chunk_id, visible_chunks_num, view_matrix,
                      position, scale, rotation, sh_base, sh_rest, opacity,
                      activated_position_grad, activated_scale_grad, activated_rotation_grad, color_grad,
                      activated_opacity_grad):
    """GR/compact.cu:1087-1212 -> six compacted gradients [..,A,S]."""
    ids = _asc(visible_chunk_id, _I64, "visible_chunk_id"); num = _asc(visible_chunks_num, _I32, "visible_chunks_num")
    view = _f32c(view_matrix, "view_matrix")
    pos = _f32c(position, "position"); sc = _f32c(scale, "scale"); rot = _f32c(rotation, "rotation")
    op = _f32c(opacity, "opacity")
    gp = _f32c(activated_position_grad, "activated_position_grad"); gs = _f32c(activated_scale_grad, "activated_scale_grad")
    gr = _f32c(activated_rotation_grad, "activated_rotation_grad"); gc = _f32c(color_grad, "color_grad")
    go = _f32c(activated_opacity_grad, "activated_opacity_grad")
    C, S = pos.shape[-2:]
    A, V, R = ids.shape[0], view.shape[0], sh_rest.shape[0]
    dev = pos.device
    with torch.cuda.device(dev):
        o_pos = torch.empty((3, A, S), dtype=_F32, device=dev)
        o_sc = torch.empty((3, A, S), dtype=_F32, device=dev)
        o_rot = torch.empty((4, A, S), dtype=_F32, device=dev)
        o_s0 = torch.empty((1, 3, A, S), dtype=_F32, device=dev)
        o_sr = torch.empty((R, 3, A, S), dtype=_F32, device=dev)
        o_op = torch.empty((1, A, S), dtype=_F32, device=dev)
        _lib.call("lgs_activate_backward", int(sh_degree), _ptr(ids), _ptr(num), _ptr(view), V, _ptr(pos), _ptr(sc), _ptr(rot),
                  _ptr(op), C, S, A, R, int(CONFIG["true_sigmoid_grad"]), _ptr(gp), _ptr(gs), _ptr(gr), _ptr(gc), _ptr(go),
                  _ptr(o_pos), _ptr(o_sc), _ptr(o_rot), _ptr(o_s0), _ptr(o_sr), _ptr(o_op), _stream(dev))
    return [o_pos, o_sc, o_rot, o_s0, o_sr, o_op]


# ---------------------------------------------------------------------------------------------------
# per-Gaussian projection operators
# ---------------------------------------------------------------------------------------------------

def mvp_transform_forward(world_position, view_matrix, proj_matrix, valid_length=None):
    """GR/transform.cu:440-470 -> [view_position f32[V,4,N], ndc_position f32[V,4,N]]."""
    p = _f32c(world_position, "world_position"); vm = _f32c(view_matrix, "view_matrix"); pm = _f32c(proj_matrix, "proj_matrix")
    V, N = vm.shape[0], p.shape[1]
    dev = p.device
    with torch.cuda.device(dev):
        vp = torch.empty((V, 4, N), dtype=_F32, device=dev)
        ndc = torch.empty((V, 4, N), dtype=_F32, device=dev)
        _lib.call("lgs_mvp_transform_forward", _ptr(p), _ptr(vm), _ptr(pm), _ptr(_vl(valid_length)), V, N, _ptr(vp), _ptr(ndc), _stream(dev))
    return [vp, ndc]


def mvp_transform_backward(grad_ndc_pos, grad_view_pos, view_matrix, proj_matrix, view_pos, valid_length=None):
    """GR/transform.cu:562-598 -> d world_position f32[4,N]."""
    gn = _f32c(grad_ndc_pos, "grad_ndc_pos"); gv = _f32c(grad_view_pos, "grad_view_pos")
    vm = _f32c(view_matrix, "view_matrix"); pm = _f32c(proj_matrix, "proj_matrix"); vp = _f32c(view_pos, "view_pos")
    V, N = gn.shape[0], gn.shape[2]
    dev = gn.device
    with torch.cuda.device(dev):
        out = torch.empty((4, N), dtype=_F32, device=dev)
        _lib.call("lgs_mvp_transform_backward", _ptr(gn), _ptr(gv), _ptr(vm), _ptr(pm), _ptr(vp), _ptr(_vl(valid_length)), V, N,
                  _ptr(out), _stream(dev))
    return out


def createTransformMatrix_forward(quaternion, scale, valid_length=None):
    """GR/transform.cu:129-149 -> f32[3,3,N]."""
    q = _f32c(quaternion, "quaternion"); s = _f32c(scale, "scale")
    N = q.shape[1]
    dev = q.device
    with torch.cuda.device(dev):
        T = torch.empty((3, 3, N), dtype=_F32, device=dev)
        _lib.call("lgs_create_transform_matrix_forward", _ptr(q), _ptr(s), _ptr(_vl(valid_length)), N, _ptr(T), _stream(dev))
    return T


def createTransformMatrix_backward(transform_matrix_grad, quaternion, scale, valid_length=None):
    """GR/transform.cu:231-256 -> [d quaternion f32[4,N], d scale f32[3,N]]."""
    g = _f32c(transform_matrix_grad, "transform_matrix_grad"); q = _f32c(quaternion, "quaternion"); s = _f32c(scale, "scale")
    N = q.shape[1]
    dev = q.device
    with torch.cuda.device(dev):
        gq = torch.empty((4, N), dtype=_F32, device=dev)
        gs = torch.empty((3, N), dtype=_F32, device=dev)
        _lib.call("lgs_create_transform_matrix_backward", _ptr(g), _ptr(q), _ptr(s), _ptr(_vl(valid_length)), N, _ptr(gq), _ptr(gs),
                  _stream(dev))
    return [gq, gs]


def jacobianRayspace(translated_position, proj_matrix, output_h, output_w, valid_length=None):
    """GR/transform.cu:54-90 -> f32[V,3,3,N]."""
    vp = _f32c(translated_position, "translated_position"); pm = _f32c(proj_matrix, "proj_matrix")
    V, N = vp.shape[0], vp.shape[2]
    dev = vp.device
    with torch.cuda.device(dev):
        J = torch.empty((V, 3, 3, N), dtype=_F32, device=dev)
        _lib.call("lgs_jacobian_rayspace", _ptr(vp), _ptr(pm), _ptr(_vl(valid_length)), V, N, int(output_h), int(output_w), _ptr(J),
                  _stream(dev))
    return J


def createCov2dDirectly_forward(J, view_matrix, transform_matrix, valid_length=None):
    """GR/transform.cu:783-821 -> f32[V,2,2,N]."""
    j = _f32c(J, "J"); vm = _f32c(view_matrix, "view_matrix"); T = _f32c(transform_matrix, "transform_matrix")
    V, N = vm.shape[0], T.shape[2]
    dev = T.device
    with torch.cuda.device(dev):
        cov = torch.empty((V, 2, 2, N), dtype=_F32, device=dev)
        _lib.call("lgs_create_cov2d_forward", _ptr(j), _ptr(vm), _ptr(T), _ptr(_vl(valid_length)), V, N, _ptr(cov), _stream(dev))
    return cov


def createCov2dDirectly_backward(cov2d_grad, J, view_matrix, transform_matrix, valid_length=None):
    """GR/transform.cu:892-927 -> d transform_matrix f32[3,3,N]."""
    g = _f32c(cov2d_grad, "cov2d_grad"); j = _f32c(J, "J"); vm = _f32c(view_matrix, "view_matrix")
    T = _f32c(transform_matrix, "transform_matrix")
    V, N = vm.shape[0], T.shape[2]
    dev = T.device
    with torch.cuda.device(dev):
        gT = torch.empty((3, 3, N), dtype=_F32, device=dev)
        _lib.call("lgs_create_cov2d_backward", _ptr(g), _ptr(j), _ptr(vm), _ptr(T), _ptr(_vl(valid_length)), V, N, _ptr(gT), _stream(dev))
    return gT


def eigh_and_inv_2x2matrix_forward(input, valid_length=None):
    """GR/transform.cu:1456-1487 -> [val f32[V,2,N], vec f32[V,2,2,N], inv f32[V,2,2,N]]."""
    m = _f32c(input, "input")
    V, N = m.shape[0], m.shape[3]
    dev = m.device
    with torch.cuda.device(dev):
        val = torch.empty((V, 2, N), dtype=_F32, device=dev)
        vec = torch.empty((V, 2, 2, N), dtype=_F32, device=dev)
        inv = torch.empty((V, 2, 2, N), dtype=_F32, device=dev)
        _lib.call("lgs_eigh_and_inv_2x2_forward", _ptr(m), _ptr(_vl(valid_length)), V, N, _ptr(val), _ptr(vec), _ptr(inv), _stream(dev))
    return [val, vec, inv]


def inv_2x2matrix_backward(inv_matrix, dL_dInvMatrix, valid_length=None):
    """GR/transform.cu:1489-1518 -> d matrix f32[V,2,2,N]."""
    a = _f32c(inv_matrix, "inv_matrix"); g = _f32c(dL_dInvMatrix, "dL_dInvMatrix")
    V, N = a.shape[0], a.shape[3]
    dev = a.device
    with torch.cuda.device(dev):
        out = torch.empty_like(g)
        _lib.call("lgs_inv_2x2_backward", _ptr(a), _ptr(g), _ptr(_vl(valid_length)), V, N, _ptr(out), _stream(dev))
    return out


def sh2rgb_forward(degree, sh_base, sh_rest, dir):
    """GR/transform.cu:1039-1086 -> rgb f32[V,3,N]."""
    s0 = _f32c(sh_base, "sh_base"); sr = _f32c(sh_rest, "sh_rest"); d = _f32c(dir, "dir")
    V, N = d.shape[0], d.shape[2]
    dev = d.device
    with torch.cuda.device(dev):
        rgb = torch.empty((V, 3, N), dtype=_F32, device=dev)
        _lib.call("lgs_sh2rgb_forward", int(degree), _ptr(s0), _ptr(sr), _ptr(d), V, N, _ptr(rgb), _stream(dev))
    return rgb


def sh2rgb_backward(degree, rgb_grad, sh_rest_dim, dir, SH_base, SH_rest):
    """GR/transform.cu:1298-1361 -> [d sh_base f32[1,3,N], d sh_rest f32[R,3,N], d dir (zeros)]."""
    g = _f32c(rgb_grad, "rgb_grad"); d = _f32c(dir, "dir")
    V, N = g.shape[0], g.shape[2]
    dev = g.device
    with torch.cuda.device(dev):
        g0 = torch.empty((1, 3, N), dtype=_F32, device=dev)
        gr = torch.empty((int(sh_rest_dim), 3, N), dtype=_F32, device=dev)
        gd = torch.empty_like(d)
        _lib.call("lgs_sh2rgb_backward", int(degree), _ptr(g), int(sh_rest_dim), _ptr(d), V, N, _ptr(g0), _ptr(gr), _ptr(gd), _stream(dev))
    return [g0, gr, gd]


# ---------------------------------------------------------------------------------------------------
# binning
# ---------------------------------------------------------------------------------------------------

def get_allocate_size(ndc, view_space_z, inv_cov2d, opacity, height, width, tilesize_h, tilesize_w, valid_length=None):
    """GR/binning.cu:398-440 -> [left_up i32[V,2,N], right_down i32[V,2,N], allocate_size i32[V,N]]."""
    n = _f32c(ndc, "ndc"); z = _f32c(view_space_z, "view_space_z"); c = _f32c(inv_cov2d, "inv_cov2d"); o = _f32c(opacity, "opacity")
    V, N = n.shape[0], n.shape[2]
    dev = n.device
    with torch.cuda.device(dev):
        _lib.call("lgs_set_exact_tile_bound", int(bool(CONFIG["fix_last_tile"])))
        lu = torch.empty((V, 2, N), dtype=_I32, device=dev)
        rd = torch.empty((V, 2, N), dtype=_I32, device=dev)
        al = torch.empty((V, N), dtype=_I32, device=dev)
        _lib.call("lgs_get_allocate_size", _ptr(n), _ptr(z), _ptr(c), _ptr(o), _ptr(_vl(valid_length)), V, N, int(height), int(width),
                  int(tilesize_h), int(tilesize_w), _ptr(lu), _ptr(rd), _ptr(al), _stream(dev))
    return [lu, rd, al]


def create_table(ndc, inv_cov2d, opacity, offset, depth_sorted_pointid, feedback_buffer_cpu, idx_tensor_cpu,
                 height, width, tile_size_h, tile_size_w):
    """GR/binning.cu:123-226 -> [sorted_tileId i32[V,alloc], sorted_pointId i32[V,alloc]].

    Table size: 1.5x what this frame needed last epoch (pinned feedback buffer) or, the first time, one
    blocking read of the scan total -- the reference's policy.  Pairs beyond the table are dropped."""
    n = _f32c(ndc, "ndc"); c = _f32c(inv_cov2d, "inv_cov2d"); o = _f32c(opacity, "opacity")
    off = _asc(offset, _I32, "offset"); sid = _asc(depth_sorted_pointid, _I64, "depth_sorted_pointid")
    V, N = n.shape[0], n.shape[2]
    dev = n.device
    with torch.cuda.device(dev):
        pred = 0
        if feedback_buffer_cpu is not None and idx_tensor_cpu is not None:
            for i in range(V):
                idx = int(idx_tensor_cpu[i])
                pred = max(pred, int(feedback_buffer_cpu[idx]))
                feedback_buffer_cpu[idx:idx + 1].copy_(off[i, N - 1:N], non_blocking=True)
        pred = int(1.5 * pred)
        if pred <= 0:
            pred = int(off[:, N - 1].max().item()) if N > 0 else 0
        if pred <= 0:
            raise RuntimeError("error pred_allocate_size")
        nbytes = ctypes.c_size_t(0)
        _lib.call("lgs_create_table_workspace_bytes", V, pred, ctypes.byref(nbytes))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        keys = torch.empty((V, pred), dtype=_I32, device=dev)
        vals = torch.empty((V, pred), dtype=_I32, device=dev)
        _lib.call("lgs_set_exact_tile_bound", int(bool(CONFIG["fix_last_tile"])))
        _lib.call("lgs_create_table", _ptr(n), _ptr(c), _ptr(o), _ptr(off), _ptr(sid), V, N, pred, int(height), int(width),
                  int(tile_size_h), int(tile_size_w), _ptr(keys), _ptr(vals), _ptr(ws), ctypes.c_size_t(nbytes.value), _stream(dev))
    return [keys, vals]


def tileRange(table_tileId, max_tileId):
    """GR/binning.cu:267-287 -> i32[V,max_tileId+2] (-1 = no splats)."""
    k = _asc(table_tileId, _I32, "table_tileId")
    V, L = k.shape
    dev = k.device
    with torch.cuda.device(dev):
        out = torch.empty((V, int(max_tileId) + 2), dtype=_I32, device=dev)
        _lib.call("lgs_tile_range", _ptr(k), V, L, int(max_tileId), int(CONFIG["fix_last_tile"]), _ptr(out), _stream(dev))
    return out


# ---------------------------------------------------------------------------------------------------
# rasterisation
# ---------------------------------------------------------------------------------------------------

def _raster_forward_impl(sorted_points, start_index, packed, specific_tiles, img_h, img_w, th, tw,
                         enable_statistic, enable_trans, enable_depth):
    sp = _asc(sorted_points, _I32, "sorted_points"); si = _asc(start_index, _I32, "start_index")
    V, N = packed.shape[0], packed.shape[1]
    cap = sp.shape[1]
    gx, gy = _tiles(img_h, img_w, th, tw)
    Hp, Wp = gy * th, gx * tw
    if si.shape[1] != gx * gy + 2:
        raise RuntimeError(f"start_index has {si.shape[1]} entries, expected tiles+2 = {gx * gy + 2}")
    dev = packed.device
    tiles = None if specific_tiles is None else _asc(specific_tiles, _I32, "specific_tiles")
    n_sel = 0 if tiles is None else tiles.shape[1]
    img = torch.empty((V, 3, Hp, Wp), dtype=_F32, device=dev)
    T = torch.empty((V, 1, Hp, Wp), dtype=_F32, device=dev)
    if tiles is not None:   # tiles that are not rendered must read as empty
        img.zero_(); T.fill_(1.0)
    last = torch.zeros((V, 1, Hp, Wp), dtype=torch.int16, device=dev) if tiles is not None else \
        torch.empty((V, 1, Hp, Wp), dtype=torch.int16, device=dev)
    depth = torch.zeros((V, 1, Hp, Wp), dtype=_F32, device=dev) if enable_depth else torch.empty((0, 0, 0, 0), dtype=_F32, device=dev)
    fc = torch.zeros((V, 1, N), dtype=_I32, device=dev)
    fw = torch.zeros((V, 1, N), dtype=_F32, device=dev)
    _lib.call("lgs_rasterize_forward_packed", _ptr(sp), _ptr(si), _ptr(packed), _ptr(tiles), n_sel, V, N, cap, int(img_h), int(img_w),
              int(th), int(tw), int(bool(enable_statistic)), 0, _ptr(img), _ptr(T), _ptr(last), _ptr(fc), _ptr(fw), None, None, None, None,
              _stream(dev))
    return img, T, depth, last, fc, fw


def rasterize_forward(sorted_points, start_index, ndc, cov2d_inv, color, opacity, specific_tiles,
                      img_h, img_w, tilesize_h, tilesize_w, enable_statistic, enable_trans, enable_depth):
    """GR/raster.cu:386-492 -> [img, transmittance, depth, last_contributor, packed_params, fragment_count, fragment_weight_sum].

    packed_params is f32[V,N,12] (fp32 record) instead of the reference's f32[V,N,8] half-packed one;
    it is opaque to the callers (only handed back to rasterize_backward)."""
    n = _f32c(ndc, "ndc"); c = _f32c(cov2d_inv, "cov2d_inv"); col = _f32c(color, "color"); o = _f32c(opacity, "opacity")
    V, N = n.shape[0], n.shape[2]
    dev = n.device
    th, tw = int(tilesize_h), int(tilesize_w)
    with torch.cuda.device(dev):
        packed = torch.empty((V, N, 12), dtype=_F32, device=dev)
        _lib.call("lgs_pack_params", _ptr(n), _ptr(c), _ptr(col), _ptr(o), V, N, int(img_h), int(img_w), _ptr(packed), _stream(dev))
        img, T, depth, last, fc, fw = _raster_forward_impl(sorted_points, start_index, packed, specific_tiles, img_h, img_w, th, tw,
                                                           enable_statistic, enable_trans, enable_depth)
    return [img, T, depth, last, packed, fc, fw]


def rasterize_forward_packed(sorted_points, start_index, packed_params, specific_tiles, img_h, img_w, tile_h, tile_w,
                             enable_statistic, enable_trans, enable_depth):
    """GR/raster.cu:495-586 -> [img, transmittance, depth, last_contributor, fragment_count, fragment_weight_sum]."""
    packed = _f32c(packed_params, "packed_params")
    if packed.shape[-1] != 12:
        raise RuntimeError("packed_params must be the f32[V,N,12] record produced by rasterize_forward")
    with torch.cuda.device(packed.device):
        img, T, depth, last, fc, fw = _raster_forward_impl(sorted_points, start_index, packed, specific_tiles, img_h, img_w,
                                                           int(tile_h), int(tile_w), enable_statistic, enable_trans, enable_depth)
    return [img, T, depth, last, fc, fw]


def rasterize_backward(sorted_points, start_index, packed_params, specific_tiles, final_transmitance, last_contributor,
                       d_img, d_trans_img_arg, d_depth_img_arg, grad_inv_sacler_arg,
                       img_h, img_w, tilesize_h, tilesize_w, enable_statistic):
    """GR/raster.cu:917-1037 -> [d_ndc, d_cov2d_inv, d_color, d_opacity, err_sum, err_square_sum]."""
    sp = _asc(sorted_points, _I32, "sorted_points"); si = _asc(start_index, _I32, "start_index")
    packed = _f32c(packed_params, "packed_params")
    T = _f32c(final_transmitance, "final_transmitance"); last = _asc(last_contributor, torch.int16, "last_contributor")
    g = _f32c(d_img, "d_img")
    gt = None if d_trans_img_arg is None else _f32c(d_trans_img_arg, "d_trans_img")
    sc = None if grad_inv_sacler_arg is None else _f32c(grad_inv_sacler_arg.reshape(1), "grad_inv_scaler")
    tiles = None if specific_tiles is None else _asc(specific_tiles, _I32, "specific_tiles")
    V, N = packed.shape[0], packed.shape[1]
    cap = sp.shape[1]
    dev = packed.device
    with torch.cuda.device(dev):
        pg = torch.empty((V, N, 12), dtype=_F32, device=dev)
        d_ndc = torch.empty((V, 4, N), dtype=_F32, device=dev)
        d_cov = torch.empty((V, 2, 2, N), dtype=_F32, device=dev)
        d_col = torch.empty((V, 3, N), dtype=_F32, device=dev)
        d_op = torch.empty((1, N), dtype=_F32, device=dev)
        e1 = torch.empty((V, 1, N), dtype=_F32, device=dev)
        e2 = torch.empty((V, 1, N), dtype=_F32, device=dev)
        _lib.call("lgs_rasterize_backward", _ptr(sp), _ptr(si), _ptr(packed), _ptr(tiles), 0 if tiles is None else tiles.shape[1],
                  _ptr(T), _ptr(last), _ptr(g), _ptr(gt), None, _ptr(sc), V, N, cap, int(img_h), int(img_w), int(tilesize_h),
                  int(tilesize_w), int(bool(enable_statistic)), _ptr(pg), _ptr(d_ndc), _ptr(d_cov), _ptr(d_col), _ptr(d_op),
                  _ptr(e1), _ptr(e2), None, None, None, None, _stream(dev))
    return [d_ndc, d_cov, d_col, d_op, e1, e2]


# ---------------------------------------------------------------------------------------------------
# optimiser / statistics
# ---------------------------------------------------------------------------------------------------

def adamUpdate(param, param_grad, exp_avg, exp_avg_sq, visible_index, valid_length, lr, b1, b2, eps):
    """GR/compact.cu:377-417: in-place sparse Adam without bias correction (chunk [R,C,S] or primitive [R,N] form)."""
    for name, t in (("param", param), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        if not (t.is_cuda and t.dtype == _F32 and t.is_contiguous()):
            raise RuntimeError(f"adamUpdate: {name} must be a contiguous float32 CUDA tensor (updated in place)")
    g = _f32c(param_grad, "param_grad"); vi = _asc(visible_index, _I64, "visible_index")
    dev = param.device
    with torch.cuda.device(dev):
        if param.dim() == 3:
            R, C, S = param.shape
            A = vi.shape[0]
            _lib.call("lgs_adam_update_chunk", _ptr(param), _ptr(g), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(vi), _ptr(_vl(valid_length)),
                      R, C, S, A, float(lr), float(b1), float(b2), float(eps), _stream(dev))
        elif param.dim() == 2:
            R, N = param.shape
            _lib.call("lgs_adam_update_primitive", _ptr(param), _ptr(g), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(vi), R, N,
                      float(lr), float(b1), float(b2), float(eps), _stream(dev))
        else:
            raise RuntimeError("adamUpdate: param must be [R,chunks,chunk_size] or [R,N]")


def gpu_driven_pipeline_sparse_op(A, B, visible_chunk_ids, visible_count, op_name):
    """GR/compact.cu:1257-1336: A[:, ids[j], :] (op)= B[:, j, :] for j < *visible_count, in place."""
    for name, t in (("A", A), ("B", B), ("visible_chunk_ids", visible_chunk_ids), ("visible_count", visible_count)):
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor")
    ops = {"add": 0, "sum": 0, "min": 1, "max": 2}
    if op_name not in ops:
        raise RuntimeError(f"Unsupported op: {op_name}. Expected: add, min, max")
    codes = {_F32: 0, _I32: 1, torch.float64: 2, _I64: 3, torch.int16: 4, torch.int8: 5, torch.uint8: 6}     # AT_DISPATCH_ALL_TYPES
    if A.dtype != B.dtype or A.dtype not in codes:
        raise RuntimeError(f"gpu_driven_pipeline_sparse_op: dtype {A.dtype}/{B.dtype} unsupported (expected one of {list(codes)})")
    if not A.is_contiguous():
        raise RuntimeError("gpu_driven_pipeline_sparse_op: A must be contiguous (updated in place)")
    Bc = B if B.is_contiguous() else B.contiguous()
    ids = _asc(visible_chunk_ids, _I64, "visible_chunk_ids"); cnt = _asc(visible_count, _I32, "visible_count")
    E, C, S = A.shape
    if S > 1024:
        raise RuntimeError("chunk_size exceeds max threads per block")
    dev = A.device
    with torch.cuda.device(dev):
        _lib.call("lgs_sparse_chunk_op", _ptr(A), _ptr(Bc), _ptr(ids), _ptr(cnt), codes[A.dtype], ops[op_name], E, C,
                  Bc.shape[1], S, _stream(dev))


# ---------------------------------------------------------------------------------------------------
# learnable cameras
# ---------------------------------------------------------------------------------------------------

def create_viewproj_forward(view_params, recp_tan_half_fov_x, img_h, img_w, z_near, z_far):
    """GR/compact.cu:123-141: view_params f32[V,7] (qw qx qy qz tx ty tz), recp_tan_half_fov_x f32[1] ->
    [view f32[V,4,4], proj f32[V,4,4], viewproj f32[V,4,4], frustumplane f32[V,6,4]] (row-vector convention)."""
    vp = _f32c(view_params, "view_params"); rf = _f32c(recp_tan_half_fov_x.reshape(-1), "recp_tan_half_fov_x")
    if vp.dim() != 2 or vp.shape[1] != 7:
        raise RuntimeError(f"view_params must be [V,7], got {tuple(vp.shape)}")
    V = vp.shape[0]
    dev = vp.device
    with torch.cuda.device(dev):
        view = torch.empty((V, 4, 4), dtype=_F32, device=dev)
        proj = torch.empty((V, 4, 4), dtype=_F32, device=dev)
        viewproj = torch.empty((V, 4, 4), dtype=_F32, device=dev)
        planes = torch.empty((V, 6, 4), dtype=_F32, device=dev)
        _lib.call("lgs_create_viewproj_forward", _ptr(vp), _ptr(rf), V, int(img_h), int(img_w), float(z_near), float(z_far),
                  _ptr(view), _ptr(proj), _ptr(viewproj), _ptr(planes), _stream(dev))
    return [view, proj, viewproj, planes]


def create_viewproj_backward(view_matrix_grad, proj_matrix_grad, viewproj_matrix_grad, view_params, recp_tan_half_fov_x,
                             img_h, img_w, z_near, z_far):
    """GR/compact.cu:289-316 -> [grad_view_params f32[V,7], grad_recp_tan_half_fov_x f32[1]].

    The reference's arithmetic, quirks included (DESIGN.md section 7): the quaternion gradient is the true one times |q|, and the
    fov gradient scales d proj[1][1] by the integer quotient img_w // img_h.  The fov gradient is summed over the views in a
    fixed order (the reference's is a race for more than one view)."""
    vp = _f32c(view_params, "view_params"); rf = _f32c(recp_tan_half_fov_x.reshape(-1), "recp_tan_half_fov_x")
    V = vp.shape[0]
    gv = _f32c(view_matrix_grad, "view_matrix_grad"); gp = _f32c(proj_matrix_grad, "proj_matrix_grad")
    gvp = _f32c(viewproj_matrix_grad, "viewproj_matrix_grad")
    for name, g in (("view_matrix_grad", gv), ("proj_matrix_grad", gp), ("viewproj_matrix_grad", gvp)):
        if g.numel() != V * 16:
            raise RuntimeError(f"{name} must be [V,4,4] with V = {V}, got {tuple(g.shape)}")
    dev = vp.device
    with torch.cuda.device(dev):
        g_params = torch.empty((V, 7), dtype=_F32, device=dev)
        g_recp = torch.zeros_like(rf)         # only [0] is a parameter of the camera (GR/compact.cu:54); the rest stays zero
        _lib.call("lgs_create_viewproj_backward", _ptr(gv), _ptr(gp), _ptr(gvp), _ptr(vp), _ptr(rf), V, int(img_h), int(img_w),
                  float(z_near), float(z_far), _ptr(g_params), _ptr(g_recp), _stream(dev))
    return [g_params, g_recp.reshape(recp_tan_half_fov_x.shape)]


# ---------------------------------------------------------------------------------------------------
# entry points outside the hot path (SURVEY 8b: optional / dead in the reference)
# ---------------------------------------------------------------------------------------------------

def _out_of_scope(name, why):
    def fn(*args, **kwargs):
        raise NotImplementedError(f"litegs_fused.{name} is outside the render hot path rebuilt by litegs_b200: {why}")
    fn.__name__ = name
    return fn


world2ndc_forward = _out_of_scope("world2ndc_forward", "only reachable through the unused World2NdcFunc (wrapper.py:287)")
world2ndc_backword = _out_of_scope("world2ndc_backword", "only reachable through the unused World2NdcFunc (wrapper.py:287)")

# the 26 names of GR/ext_cuda.cpp:9-35
EXPORTS = [
    "create_viewproj_forward", "create_viewproj_backward", "create_table", "tileRange", "get_allocate_size",
    "rasterize_forward", "rasterize_forward_packed", "rasterize_backward", "jacobianRayspace",
    "createTransformMatrix_forward", "createTransformMatrix_backward", "world2ndc_forward", "world2ndc_backword",
    "mvp_transform_forward", "mvp_transform_backward", "createCov2dDirectly_forward", "createCov2dDirectly_backward",
    "sh2rgb_forward", "sh2rgb_backward", "eigh_and_inv_2x2matrix_forward", "inv_2x2matrix_backward",
    "cull_compact_activate", "activate_backward", "adamUpdate", "frustum_culling_aabb", "gpu_driven_pipeline_sparse_op",
]
