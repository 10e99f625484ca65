"""Fused per-view render pipeline ("Level B", SURVEY.md section 7) above the C ABI.

One view = render_preprocess + render of the reference (litegs/render/__init__.py:11-94) collapsed to

    cull_chunks -> project_forward -> view_params -> [one 32-byte D2H: sizes + depth-key bits] -> depth radix sort (N keys) ->
    gathered scan -> emit_pairs -> tile radix sort (tile bits only) -> tile_range -> raster_forward

and the backward to  raster_backward -> project_backward  (two kernels + one memset).  Everything runs on
the current CUDA stream; the only host synchronisation is the read-back of lgs_view_params' parameter block (visible chunks,
pair count, depth-key bits) that sizes the buffers, exactly one per view (the reference pays two: GR/compact.cu:527-549 and
GR/binning.cu:137-163, hidden behind last epoch's feedback values when available).  ViewWorkspace enqueues the same chain
without the read-back, on capacities.
"""
from __future__ import annotations

import collections
import ctypes
import os
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from .fused import CONFIG, _on, _ptr, _stream

_F32, _I32, _I64, _U8 = torch.float32, torch.int32, torch.int64, torch.uint8
_KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")

_ws_bytes_cache: dict = {}


def _query_bytes(fn: str, *args) -> int:
    key = (fn,) + args
    v = _ws_bytes_cache.get(key)
    if v is None:
        n = ctypes.c_size_t(0)
        _lib.call(fn, *args, ctypes.byref(n))
        v = _ws_bytes_cache[key] = int(n.value)
    return v


def _round_up(n: int, m: int) -> int:
    return ((n + m - 1) // m) * m


def _u16_keys(ntile: int) -> bool:
    """16-bit tile keys whenever (tile + 1) fits them (up to 4K at 8x16)."""
    return (ntile + 1) < 65536


def _binning_ws_bytes(n_splats: int, n_pairs: int, u16: bool) -> int:
    """Workspace of _bin: the depth sort and the scan of n_splats slots, the tile sort of n_pairs pairs (one buffer, used in turn)."""
    return max(_query_bytes("lgs_sort_pairs_u32_workspace_bytes", _round_up(n_splats, 1 << 16)),
               _query_bytes("lgs_scan_gathered_workspace_bytes", _round_up(n_splats, 1 << 16)),
               _query_bytes(f"lgs_sort_pairs_{'u16' if u16 else 'u32'}_workspace_bytes", _round_up(n_pairs, 1 << 18)))


@dataclass
class ViewState:
    """Everything the backward of one view needs (the reference keeps the same set alive through
    ctx.save_for_backward in wrapper.py:469,815)."""
    sh_degree: int
    hw: tuple
    tile: tuple
    n_chunks_visible: int
    n_pairs: int
    depth_bits: int                  # bits of the depth-key range of the splats that own pairs (1 without pairs)
    chunk_ids: torch.Tensor          # i64[M], first n_chunks_visible valid, ascending
    counters: torch.Tensor           # i32[4] = (visible chunks, pairs, ~min depth key, max depth key) on device
    view: torch.Tensor
    proj: torch.Tensor
    packed: torch.Tensor             # f32[1, Nv, 12]
    tile_count: torch.Tensor         # i32[Nv]
    sorted_pid: torch.Tensor         # i32[1, D]
    ranges: torch.Tensor             # i32[1, tiles+2]
    T: torch.Tensor                  # f32[1,1,Hp,Wp]
    last: torch.Tensor               # i16[1,1,Hp,Wp] (unsigned 16-bit counts)
    tile_order: Optional[torch.Tensor] = None   # i32[1,tiles]: tile ids, heaviest backward work first
    antialiased: bool = False        # antialiased mode (DESIGN.md section 1): the backward must use the forward's setting
    filter_3d: Optional[torch.Tensor] = None    # 3D smoothing filter f32[1,C,S] the forward used (DESIGN.md section 1), or None
    depth: Optional[torch.Tensor] = None        # f32[1,1,Hp,Wp] per-pixel depth D (render_depth, DESIGN.md section 1), or None
    normal: Optional[torch.Tensor] = None       # f32[1,3,Hp,Wp] per-pixel normal N (render_normal, DESIGN.md section 1), or None
    normal_rec: Optional[torch.Tensor] = None   # f32[Nv,4] each record's camera-facing view-space normal (render_normal), or None


class _Pinned:
    """Per-device pinned int32[8] used for the read-back of lgs_view_params' parameter block."""
    _bufs: dict = {}

    @classmethod
    def get(cls, dev) -> torch.Tensor:
        b = cls._bufs.get(dev)
        if b is None:
            b = cls._bufs[dev] = torch.zeros(8, dtype=_I32).pin_memory()
        return b


def _padded(g: torch.Tensor, shape) -> torch.Tensor:
    """A per-pixel gradient f32[1,c,H,W] or [1,c,Hp,Wp] as a contiguous f32[1,c,Hp,Wp] (zeros in the padding), c = shape[1]."""
    if not (g.is_cuda and g.dtype == _F32 and g.dim() == 4 and tuple(g.shape[:2]) == tuple(shape[:2])):
        raise RuntimeError(f"per-pixel gradients must be float32 CUDA tensors of shape [1,{shape[1]},H,W]")
    if tuple(g.shape) != tuple(shape):
        g = torch.nn.functional.pad(g, (0, shape[-1] - g.shape[-1], 0, shape[-2] - g.shape[-2]))
    return g if g.is_contiguous() else g.contiguous()


def check_filter_3d(filter_3d: Optional[torch.Tensor], xyz: torch.Tensor) -> Optional[torch.Tensor]:
    """filter_3d must be None or a contiguous float32 tensor on xyz's device, clustered like the opacity ([1,C,S])."""
    if filter_3d is None:
        return None
    C, S = xyz.shape[-2:]
    if not (filter_3d.device == xyz.device and filter_3d.dtype == _F32 and filter_3d.is_contiguous()
            and tuple(filter_3d.shape[-2:]) == (C, S) and filter_3d.numel() == C * S):
        raise RuntimeError(f"filter_3d must be a contiguous float32 tensor of shape [1,{C},{S}] on {xyz.device}")
    return filter_3d.detach()


# The five fused stages, each issued from here alone for both view paths (the synchronising functions below and ViewWorkspace).
# An absent buffer is None, and NULL selects the kernels without that mode.  hw = (H, W), tile = (th, tw).

def _project_forward(st, params, sh_degree, chunk_ids, counters, view, proj, hw, tile, packed, dkey, iota, tcount, filter_3d,
                     antialiased, normal_rec):
    C, S = params["xyz"].shape[-2:]
    cnt = counters.data_ptr()
    _lib.call("lgs_project_forward", int(sh_degree), _ptr(chunk_ids), ctypes.c_void_p(cnt), _ptr(view), _ptr(proj),
              *[_ptr(params[k]) for k in _KEYS], C, S, C, *hw, *tile, _ptr(packed), _ptr(dkey), _ptr(iota), _ptr(tcount),
              ctypes.c_void_p(cnt + 4), _ptr(filter_3d), int(bool(antialiased)), _ptr(normal_rec), st)


def _bin(st, vparams, hw, tile, depth_bits, exact, packed, dkey, iota, tcount, dkey_s, order, keys, vals, keys_s, sorted_pid, ranges,
         ws):
    """Depth sort, gathered scan, pair emission, tile sort and tile ranges of one view: enqueue only (nothing allocated, nothing
    read back), so that it can be captured in a CUDA graph.  The live splat and pair counts and the depth-key bias come from
    lgs_view_params' block vparams on the device; the buffers' lengths are the launch sizes (order: splat slots, keys: pairs),
    ranges i32[1, tiles+2].  depth_bits: bits of the depth sort.  exact: keys holds exactly the view's pairs (the synchronising
    path), else a capacity (ViewWorkspace)."""
    vp = vparams.data_ptr()
    n_dev, d_dev, bias_dev = ctypes.c_void_p(vp), ctypes.c_void_p(vp + 4), ctypes.c_void_p(vp + 8)
    N, D, ntile = order.shape[0], keys.shape[0], ranges.shape[1] - 2
    u16 = _u16_keys(ntile)
    wsz = ctypes.c_size_t(ws.numel())
    # depth order of the live slots: stable LSD radix sort on the float bits of view z, rebased to the smallest key of a splat
    # that owns pairs and limited to depth_bits (z in [1.3, 4.7) spans 31 bits of float pattern but 24 bits of range: 3 passes
    # instead of 4); where a splat without pairs lands in the order is irrelevant, it emits nothing
    _lib.call("lgs_sort_pairs_u32_dev", _ptr(dkey), _ptr(dkey_s), _ptr(iota), _ptr(order), N, n_dev, bias_dev, depth_bits, _ptr(ws), wsz,
              st)
    offsets = dkey_s           # the sorted keys are dead: their storage receives the scan
    _lib.call("lgs_scan_gathered_dev", _ptr(tcount), _ptr(order), N, n_dev, _ptr(offsets), _ptr(ws), wsz, st)
    _lib.call("lgs_emit_pairs_dev", _ptr(packed), _ptr(offsets), _ptr(order), N, n_dev, D, *hw, *tile, 16 if u16 else 32, _ptr(keys),
              _ptr(vals), d_dev, st)
    bits = ntile.bit_length()  # floor(log2(tiles)) + 1, GR/binning.cu:199-202
    if exact:
        # the host-count tile sort: on more than 14 tile bits and 8 M pairs (4K) it takes cub's onesweep, which needs the count on
        # the host (csrc/sort.cu: sort_impl_for) and beats the own passes there (C4 on an H100 SXM at 700 W: 231.7 against
        # 195.3 views/s, DESIGN.md section 5.0)
        _lib.call(f"lgs_sort_pairs_{'u16' if u16 else 'u32'}", _ptr(keys), _ptr(keys_s), _ptr(vals), _ptr(sorted_pid), D, 0, bits,
                  _ptr(ws), wsz, st)
    else:
        _lib.call("lgs_sort_pairs_u16_dev" if u16 else "lgs_sort_pairs_u32k_dev", _ptr(keys), _ptr(keys_s), _ptr(vals), _ptr(sorted_pid),
                  D, d_dev, 0, bits, _ptr(ws), wsz, st)
    _lib.call("lgs_tile_range_u16_dev" if u16 else "lgs_tile_range_dev", _ptr(keys_s), D, d_dev, ntile, 1, _ptr(ranges), st)


def _raster_forward(st, hw, tile, sorted_pid, ranges, packed, tiles, stats, clamp_zero, img, T, last, work, depth, normal_rec, normal):
    fc, fw = stats if stats is not None else (None, None)
    _lib.call("lgs_rasterize_forward_packed", _ptr(sorted_pid), _ptr(ranges), _ptr(packed), _ptr(tiles),
              0 if tiles is None else tiles.shape[1], 1, packed.shape[1], sorted_pid.shape[1], *hw, *tile, int(stats is not None),
              int(bool(clamp_zero)), _ptr(img), _ptr(T), _ptr(last), _ptr(fc), _ptr(fw), _ptr(work), _ptr(depth), _ptr(normal_rec),
              _ptr(normal), st)


def _raster_backward(st, hw, tile, sorted_pid, ranges, packed, tiles, T, last, d_img, d_trans, clamped_img, enable_statistic, pg,
                     d_depth, normal_rec, d_normal, grad_normal):
    _lib.call("lgs_rasterize_backward", _ptr(sorted_pid), _ptr(ranges), _ptr(packed), _ptr(tiles), 0 if tiles is None else tiles.shape[1],
              _ptr(T), _ptr(last), _ptr(d_img), _ptr(d_trans), _ptr(clamped_img), None, 1, packed.shape[1], sorted_pid.shape[1], *hw,
              *tile, int(bool(enable_statistic)), _ptr(pg), None, None, None, None, None, None, _ptr(d_depth), _ptr(normal_rec),
              _ptr(d_normal), _ptr(grad_normal), st)


def _project_backward(st, params, sh_degree, chunk_ids, counters, view, proj, hw, A, pg, zero_outputs, outs, touched, cam_partials,
                      d_cam, filter_3d, antialiased, exact_grad, depth, grad_normal):
    """outs: the six gradient outputs in _KEYS order; depth: whether pg carries the depth slot."""
    C, S = params["xyz"].shape[-2:]
    _lib.call("lgs_project_backward", int(sh_degree), _ptr(chunk_ids), ctypes.c_void_p(counters.data_ptr()), _ptr(view), _ptr(proj),
              _ptr(params["xyz"]), _ptr(params["scale"]), _ptr(params["rot"]), _ptr(params["opacity"]), C, S, A,
              params["sh_rest"].shape[0], *hw, int(CONFIG["true_sigmoid_grad"]), _ptr(pg), None, zero_outputs, *[_ptr(t) for t in outs],
              _ptr(touched), _ptr(cam_partials), _ptr(d_cam), _ptr(filter_3d), int(bool(antialiased)), _ptr(params["sh_0"]),
              _ptr(params["sh_rest"]), int(bool(exact_grad)), int(bool(depth)), _ptr(grad_normal), st)


def render_view_forward(params: dict, cluster_origin: torch.Tensor, cluster_extend: torch.Tensor, frustumplane: torch.Tensor,
                        view_matrix: torch.Tensor, proj_matrix: torch.Tensor, sh_degree: int, hw: tuple, tile: tuple,
                        enable_statistic: bool = False, specific_tiles: Optional[torch.Tensor] = None, clamp_zero: bool = False,
                        antialiased: bool = False, filter_3d: Optional[torch.Tensor] = None, render_depth: bool = False,
                        render_normal: bool = False):
    """Forward of one view.  params: xyz[3,C,S] scale[3,C,S] rot[4,C,S] sh_0[1,3,C,S] sh_rest[R,3,C,S]
    opacity[1,C,S] (raw, clustered; float32 CUDA, contiguous).  Returns (img f32[1,3,Hp,Wp] padded to whole
    tiles, ViewState, (fragment_count, fragment_weight) or None).

    antialiased: scale each splat's opacity by the compensation of the 2D low-pass filter (DESIGN.md section 1), so that its
    integrated alpha does not depend on the resolution.  The state remembers it for the backward.

    filter_3d: Mip-Splatting's 3D smoothing filter f32[1,C,S] (scene.filter_3d_device), or None.  Each Gaussian is drawn with
    the scale sqrt(s^2 + f^2) and its opacity scaled by the matching volume ratio (DESIGN.md section 1); the state keeps the
    tensor for the backward, which must see the same values.

    render_depth: also render the per-pixel depth D = sum_i w_i z_i (w_i the colour's blend weights, z_i the view-space z; not
    clamped; DESIGN.md section 1, "Depth") into state.depth f32[1,1,Hp,Wp].  The expected depth is D / (1 - T).

    render_normal: also render the per-pixel normal N = sum_i w_i n_i (n_i the camera-facing view-space normal of Gaussian i's
    shortest axis; neither clamped nor normalised; DESIGN.md section 1, "Normals") into state.normal f32[1,3,Hp,Wp], and keep
    the per-record normals in state.normal_rec for the backward.  The expected normal is N / (1 - T), the unit normal N / |N|."""
    xyz = params["xyz"]
    dev = xyz.device
    filter_3d = check_filter_3d(filter_3d, xyz)
    C, S = xyz.shape[-2:]
    H, W = int(hw[0]), int(hw[1])
    th, tw = int(tile[0]), int(tile[1])
    if view_matrix.shape[0] != 1:
        raise RuntimeError("the fused pipeline renders one view per call (loop over views on the host)")
    for k in _KEYS:
        t = params[k]
        if not (t.is_cuda and t.dtype == _F32 and t.is_contiguous()):
            raise RuntimeError(f"params['{k}'] must be a contiguous float32 CUDA tensor")
    gx, gy = (W + tw - 1) // tw, (H + th - 1) // th
    ntile = gx * gy
    Hp, Wp = gy * th, gx * tw
    M = C
    with _on(dev):
        st = _stream(dev)
        counters = torch.empty(4, dtype=_I32, device=dev)
        vis = torch.empty(M, dtype=_U8, device=dev)
        ids = torch.empty(M, dtype=_I64, device=dev)
        _lib.call("lgs_frustum_culling_aabb", _ptr(cluster_origin), _ptr(cluster_extend), _ptr(frustumplane), M, 1, _ptr(vis),
                  ctypes.c_void_p(counters.data_ptr()), _ptr(ids), st)
        Nmax = M * S
        packed = torch.empty((1, Nmax, 12), dtype=_F32, device=dev)
        dkey = torch.empty(Nmax, dtype=_I32, device=dev)
        iota = torch.empty(Nmax, dtype=_I32, device=dev)
        tcount = torch.empty(Nmax, dtype=_I32, device=dev)
        normal_rec = torch.empty((Nmax, 4), dtype=_F32, device=dev) if render_normal else None
        _project_forward(st, params, sh_degree, ids, counters, view_matrix, proj_matrix, (H, W), (th, tw), packed, dkey, iota, tcount,
                         filter_3d, antialiased, normal_rec)
        # no pair capacity and all 32 bits planned: the block only carries the sizes, nothing is flagged
        vparams = torch.empty(8, dtype=_I32, device=dev)
        _lib.call("lgs_view_params", ctypes.c_void_p(counters.data_ptr()), S, 0x7FFFFFFF, 32, _ptr(vparams), None, st)
        pinned = _Pinned.get(dev)
        pinned.copy_(vparams, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        nvis, D, depth_bits = int(pinned[6]), int(pinned[5]), int(pinned[3])
        Nv = nvis * S

        ranges = torch.empty((1, ntile + 2), dtype=_I32, device=dev)
        if D > 0:
            u16 = _u16_keys(ntile)
            kdt = torch.int16 if u16 else _I32
            e = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
            sorted_pid = e((1, D), _I32)
            _bin(st, vparams, (H, W), (th, tw), depth_bits, True, packed, dkey, iota, tcount, e(Nv, _I32), e(Nv, _I32), e(D, kdt),
                 e(D, _I32), e((1, D), kdt), sorted_pid, ranges, e(_binning_ws_bytes(Nv, D, u16), _U8))
        else:
            sorted_pid = torch.zeros((1, 1), dtype=_I32, device=dev)
            _lib.call("lgs_tile_range", None, 1, 0, ntile, 1, _ptr(ranges), st)

        img = torch.empty((1, 3, Hp, Wp), dtype=_F32, device=dev)
        T = torch.empty((1, 1, Hp, Wp), dtype=_F32, device=dev)
        last = torch.empty((1, 1, Hp, Wp), dtype=torch.int16, device=dev)
        depth = torch.empty((1, 1, Hp, Wp), dtype=_F32, device=dev) if render_depth else None
        normal = torch.empty((1, 3, Hp, Wp), dtype=_F32, device=dev) if render_normal else None
        if specific_tiles is not None:
            img.zero_(); T.fill_(1.0); last.zero_()
            if depth is not None:
                depth.zero_()
            if normal is not None:
                normal.zero_()
        stats = None
        if enable_statistic:           # (fragment_count, fragment_weight)
            stats = (torch.zeros((1, 1, Nmax), dtype=_I32, device=dev), torch.zeros((1, 1, Nmax), dtype=_F32, device=dev))
        # per-tile trip count of the backward (deepest list position any pixel consumed) -> heaviest-first tile order
        order = None
        work = torch.empty((1, ntile), dtype=_I32, device=dev) if (CONFIG["tile_order"] and specific_tiles is None and D > 0) else None
        _raster_forward(st, (H, W), (th, tw), sorted_pid, ranges, packed, specific_tiles, stats, clamp_zero, img, T, last, work, depth,
                        normal_rec, normal)
        if work is not None:
            order = torch.empty((1, ntile), dtype=_I32, device=dev)
            _lib.call("lgs_tile_order", _ptr(work), 1, ntile, _ptr(order), st)
    state = ViewState(sh_degree=int(sh_degree), hw=(H, W), tile=(th, tw), n_chunks_visible=nvis, n_pairs=D, depth_bits=depth_bits,
                      chunk_ids=ids, counters=counters, view=view_matrix, proj=proj_matrix, packed=packed, tile_count=tcount,
                      sorted_pid=sorted_pid, ranges=ranges, T=T, last=last, tile_order=order, antialiased=bool(antialiased),
                      filter_3d=filter_3d, depth=depth, normal=normal, normal_rec=normal_rec)
    return img, state, stats


def render_view_backward(params: dict, state: ViewState, d_img: torch.Tensor, d_trans: Optional[torch.Tensor] = None,
                         enable_statistic: bool = False, specific_tiles: Optional[torch.Tensor] = None,
                         accumulate_into: Optional[dict] = None, clamped_img: Optional[torch.Tensor] = None,
                         camera_grad: Optional[torch.Tensor] = None, exact_grad: bool = False,
                         d_depth: Optional[torch.Tensor] = None, d_normal: Optional[torch.Tensor] = None):
    """Backward of one view: d_img f32[1,3,Hp,Wp] (padded) -> compacted parameter gradients
    (xyz[3,A,S], scale[3,A,S], rot[4,A,S], sh_0[1,3,A,S], sh_rest[R,3,A,S], opacity[1,A,S]) with
    A = state.n_chunks_visible, plus packed_grad (whose slot 9 carries the statistics term).

    accumulate_into: dict of DENSE contiguous gradient tensors shaped like the parameters; when given, this
    view's gradients are added into them by the kernel itself and no compacted tensors are produced
    (returns (None, packed_grad)).  An optional "_touched" entry (f32[C]) receives 1 at every visible chunk.

    camera_grad: optional contiguous f32[2,4,4] CUDA tensor that receives (d view_matrix, d proj_matrix) of this view, with
    J and the SH view direction held constant (DESIGN.md section 1).  It is assigned, not accumulated.

    exact_grad: exact gradient mode (DESIGN.md section 1): the xyz gradient and camera_grad also carry the terms through the
    ray-space Jacobian J and through the SH view direction.  The other gradients and the forward do not depend on it.

    d_depth: dL/dD f32[1,1,H,W] or [1,1,Hp,Wp] of the depth the forward rendered (render_depth=True), or None.  It reaches every
    parameter through the blend weights and the positions and camera through the view-space z.

    d_normal: dL/dN f32[1,3,H,W] or [1,3,Hp,Wp] of the normal the forward rendered (render_normal=True), or None.  It reaches
    every parameter through the blend weights, and the rotations and the camera through the normals (the shortest axis and the
    facing sign held constant)."""
    dev = params["xyz"].device
    S = params["xyz"].shape[-1]
    A = state.n_chunks_visible
    R = params["sh_rest"].shape[0]
    Nmax = state.packed.shape[1]
    if not (d_img.is_cuda and d_img.dtype == _F32):
        raise RuntimeError("d_img must be a float32 CUDA tensor")
    d_img = d_img if d_img.is_contiguous() else d_img.contiguous()
    if d_trans is not None:
        d_trans = d_trans if d_trans.is_contiguous() else d_trans.contiguous()
    if d_depth is not None:
        if state.depth is None:
            raise RuntimeError("d_depth is given, but the forward of this view did not render depth (render_depth=False)")
        d_depth = _padded(d_depth, state.T.shape)
    if d_normal is not None:
        if state.normal is None:
            raise RuntimeError("d_normal is given, but the forward of this view did not render normals (render_normal=False)")
        d_normal = _padded(d_normal, state.normal.shape)
    if camera_grad is not None and not (camera_grad.is_cuda and camera_grad.dtype == _F32 and camera_grad.is_contiguous()
                                        and tuple(camera_grad.shape) == (2, 4, 4)):
        raise RuntimeError("camera_grad must be a contiguous float32 CUDA tensor of shape [2,4,4]")
    with _on(dev):
        st = _stream(dev)
        pg = torch.empty((1, Nmax, 12), dtype=_F32, device=dev)
        if specific_tiles is None:
            specific_tiles = state.tile_order          # every tile, longest lists first (None = index order)
        nrm = d_normal is not None
        gn = torch.empty((Nmax, 4), dtype=_F32, device=dev) if nrm else None     # dL/dn per record (zeroed by the raster backward)
        _raster_backward(st, state.hw, state.tile, state.sorted_pid, state.ranges, state.packed, specific_tiles, state.T, state.last,
                         d_img, d_trans, clamped_img, enable_statistic, pg, d_depth, state.normal_rec if nrm else None, d_normal, gn)
        if accumulate_into is not None:
            for k in _KEYS:
                t = accumulate_into[k]
                if not (t.is_cuda and t.dtype == _F32 and t.is_contiguous() and tuple(t.shape) == tuple(params[k].shape)):
                    raise RuntimeError(f"accumulate_into['{k}'] must be a contiguous float32 CUDA tensor shaped like the parameter")
            # "_touched": chunk marks for the fused optimizer step
            grads, outs, touched = None, [accumulate_into[k] for k in _KEYS], accumulate_into.get("_touched")
        else:
            g_pos = torch.empty((3, A, S), dtype=_F32, device=dev)
            g_sc = torch.empty((3, A, S), dtype=_F32, device=dev)
            g_rot = torch.empty((4, A, S), dtype=_F32, device=dev)
            g_s0 = torch.empty((1, 3, A, S), dtype=_F32, device=dev)
            K = (state.sh_degree + 1) ** 2
            g_sr = torch.zeros((R, 3, A, S), dtype=_F32, device=dev) if R > K - 1 else torch.empty((R, 3, A, S), dtype=_F32, device=dev)
            g_op = torch.empty((1, A, S), dtype=_F32, device=dev)
            grads = outs = [g_pos, g_sc, g_rot, g_s0, g_sr, g_op]
            touched = None
        if A > 0:
            cam_partials = None if camera_grad is None else torch.empty((A, 32), dtype=_F32, device=dev)
            _project_backward(st, params, state.sh_degree, state.chunk_ids, state.counters, state.view, state.proj, state.hw, A, pg,
                              0 if grads is not None else 2, outs, touched, cam_partials, camera_grad, state.filter_3d, state.antialiased,
                              exact_grad, d_depth is not None, gn)
        elif camera_grad is not None:
            camera_grad.zero_()
    return grads, pg


# ---------------------------------------------------------------------------------------------------
# GPU-driven path: preallocated workspace, no host synchronisation, optionally replayed as CUDA graphs
# ---------------------------------------------------------------------------------------------------

GRAPHS_ENABLED = os.environ.get("LGS_GRAPHS", "1") != "0"      # replay the per-view forward / backward as CUDA graphs
SYNC_FREE = os.environ.get("LGS_SYNC_FREE", "1") != "0"        # render_views: GPU-driven sizing on preallocated workspaces


class ViewWorkspace:
    """Every buffer one view needs, allocated once for fixed capacities, plus (optionally) the view's forward and backward
    captured as CUDA graphs.

    The forward is enqueued without reading anything back: the sorts, the scan, the pair emission and the tile ranges take the
    live counts from device memory (``lgs_*_dev`` entry points), the number of (tile, splat) pairs is bounded by
    ``pair_capacity`` and the depth sort by ``planned_depth_bits``.  ``lgs_view_params`` raises a device-side flag when either
    prediction was too small; :meth:`check` (called by the owner when it synchronises anyway, e.g. at the end of a step) reads it
    and raises :class:`CapacityExceeded` so that the caller can grow the workspace and redo the step.  This is the reference's
    "size from the previous epoch, write feedback for the next" protocol (GR/compact.cu:527-549, GR/binning.cu:137-163,
    data.py:238) moved onto the device.

    A workspace serves ONE view at a time: its state (lists, transmittance, counts) is consumed by the backward of the same view
    before the next forward on it; ``render_views`` keeps one workspace per stream slot."""

    def __init__(self, params: dict, hw: tuple, tile: tuple, pair_capacity: int, planned_depth_bits: int = 24, use_graphs: bool = True):
        xyz = params["xyz"]
        dev = xyz.device
        C, S = xyz.shape[-2:]
        H, W = int(hw[0]), int(hw[1])
        th, tw = int(tile[0]), int(tile[1])
        gx, gy = (W + tw - 1) // tw, (H + th - 1) // th
        self.dev, self.C, self.S, self.hw, self.tile = dev, C, S, (H, W), (th, tw)
        self.ntile, self.Hp, self.Wp = gx * gy, gy * th, gx * tw
        self.Nmax = C * S
        self.cap = int(max(1024, pair_capacity))
        self.planned_bits = int(planned_depth_bits)
        self.use_graphs = bool(use_graphs)
        self.u16 = _u16_keys(self.ntile)
        kdt = torch.int16 if self.u16 else _I32
        N, D = self.Nmax, self.cap
        e = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
        self.counters = torch.zeros(4, dtype=_I32, device=dev)
        self.vparams = torch.zeros(8, dtype=_I32, device=dev)
        self.vis, self.chunk_ids = e(C, _U8), e(C, _I64)
        self.packed, self.dkey, self.iota, self.tcount = e((1, N, 12), _F32), e(N, _I32), e(N, _I32), e(N, _I32)
        self.dkey_s, self.order = e(N, _I32), e(N, _I32)
        self.keys, self.vals, self.keys_s, self.sorted_pid = e(D, kdt), e(D, _I32), e((1, D), kdt), e((1, D), _I32)
        self.ranges = e((1, self.ntile + 2), _I32)
        self.img, self.T = e((1, 3, self.Hp, self.Wp), _F32), e((1, 1, self.Hp, self.Wp), _F32)
        self.last = e((1, 1, self.Hp, self.Wp), torch.int16)
        self.work, self.tile_order = e((1, self.ntile), _I32), e((1, self.ntile), _I32)
        self.pg = e((1, N, 12), _F32)
        self.d_img = e((1, 3, self.Hp, self.Wp), _F32)
        self.depth = self.d_depth = self.d_trans = None     # f32[1,1,Hp,Wp] each, allocated on first use (depth mode, d_trans)
        self.rendered_depth = False                          # whether the last forward on this workspace rendered depth
        self.normal = self.d_normal = None                   # f32[1,3,Hp,Wp] each, allocated on first use (normal mode)
        self.normal_rec = self.grad_normal = None            # f32[N,4] each, allocated on first use (normal mode)
        self.rendered_normal = False                         # whether the last forward on this workspace rendered normals
        self.cam_view, self.cam_proj, self.cam_planes = e((1, 4, 4), _F32), e((1, 4, 4), _F32), e((1, 6, 4), _F32)
        self.cam_partials, self.d_cam = e((C, 32), _F32), e((2, 4, 4), _F32)     # camera gradient: per-chunk rows, their sum
        self.ws = e(_binning_ws_bytes(N, D, self.u16), _U8)
        self.sticky = torch.zeros(4, dtype=_I32, device=dev)      # |flags, max pairs, max depth bits, views since the last post
        self._posted = collections.deque()    # (event, pinned i32[4]) of every post_flags() not yet read by check(), oldest first
        self._free_host = []                  # pinned i32[4] buffers whose result has been read
        self._graphs = {}               # ("fwd"|"bwd", pointer signature) -> torch.cuda.CUDAGraph
        self._eager_runs = {}           # same key -> eager runs so far (the first run of a signature is never captured)
        self.views_done = 0

    # -- enqueue ---------------------------------------------------------------------------------------------------
    def _plane(self, name, shape=None):
        """The f32 buffer `name` (default shape [1,1,Hp,Wp]), allocated the first time it is asked for (its pointer then stays
        fixed)."""
        if getattr(self, name) is None:
            setattr(self, name, torch.zeros(shape or (1, 1, self.Hp, self.Wp), dtype=_F32, device=self.dev))
        return getattr(self, name)

    def _run(self, kind, sig, fn):
        """Eager the first time a pointer signature is seen, captured into a CUDA graph the second time, replayed afterwards."""
        key = (kind, sig)
        graphs = self.use_graphs and GRAPHS_ENABLED          # GRAPHS_ENABLED: module-wide switch (stage timing, A/B)
        g = self._graphs.get(key) if graphs else None
        if g is not None:
            g.replay()
            return
        seen = self._eager_runs.get(key, 0)
        cur = torch.cuda.current_stream(self.dev)
        # graphs cannot be captured on the legacy default stream
        if not graphs or seen < 1 or cur.cuda_stream == 0:
            self._eager_runs[key] = seen + 1
            fn()
            return
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=cur, capture_error_mode="thread_local"):
            fn()
        self._graphs[key] = g
        g.replay()

    def forward(self, params, cluster_origin, cluster_extend, cam, sh_degree, clamp_zero=True, antialiased=False, filter_3d=None,
                render_depth=False, render_normal=False):
        """cam: dict(view, proj, frustumplane) of device tensors.  Returns the padded image (a view of the workspace).
        render_depth: also render the per-pixel depth D into ``self.depth`` (f32[1,1,Hp,Wp], DESIGN.md section 1); the transmittance
        is ``self.T``.
        render_normal: also render the per-pixel normal N into ``self.normal`` (f32[1,3,Hp,Wp], DESIGN.md section 1, "Normals").
        antialiased: antialiased mode (DESIGN.md section 1); the backward of this view must be given the same value.
        filter_3d: 3D smoothing filter f32[1,C,S] or None; the backward of this view must be given the same tensor.  Its data
        pointer is part of the graph signature: a replayed graph reads whatever the tensor holds, so recomputing it in place
        (scene.filter_3d_device(..., out=)) needs no new capture."""
        filter_3d = check_filter_3d(filter_3d, params["xyz"])
        render_depth, render_normal, order = bool(render_depth), bool(render_normal), bool(CONFIG["tile_order"])
        if render_depth:
            self._plane("depth")
        if render_normal:
            self._plane("normal", (1, 3, self.Hp, self.Wp))
            self._plane("normal_rec", (self.Nmax, 4))
        self.cam_view.copy_(cam["view"], non_blocking=True)
        self.cam_proj.copy_(cam["proj"], non_blocking=True)
        self.cam_planes.copy_(cam["frustumplane"], non_blocking=True)

        def kernels():
            st = _stream(self.dev)
            cnt = ctypes.c_void_p(self.counters.data_ptr())
            _lib.call("lgs_frustum_culling_aabb", _ptr(cluster_origin), _ptr(cluster_extend), _ptr(self.cam_planes), self.C, 1,
                      _ptr(self.vis), cnt, _ptr(self.chunk_ids), st)
            _project_forward(st, params, sh_degree, self.chunk_ids, self.counters, self.cam_view, self.cam_proj, self.hw, self.tile,
                             self.packed, self.dkey, self.iota, self.tcount, filter_3d, antialiased,
                             self.normal_rec if render_normal else None)
            _lib.call("lgs_view_params", cnt, self.S, self.cap, self.planned_bits, _ptr(self.vparams), _ptr(self.sticky), st)
            _bin(st, self.vparams, self.hw, self.tile, self.planned_bits, False, self.packed, self.dkey, self.iota, self.tcount,
                 self.dkey_s, self.order, self.keys, self.vals, self.keys_s, self.sorted_pid, self.ranges, self.ws)
            _raster_forward(st, self.hw, self.tile, self.sorted_pid, self.ranges, self.packed, None, None, clamp_zero, self.img, self.T,
                            self.last, self.work if order else None, self.depth if render_depth else None,
                            self.normal_rec if render_normal else None, self.normal if render_normal else None)
            if order:
                _lib.call("lgs_tile_order", _ptr(self.work), 1, self.ntile, _ptr(self.tile_order), st)

        sig = (tuple(params[k].data_ptr() for k in _KEYS), cluster_origin.data_ptr(), cluster_extend.data_ptr(), int(sh_degree),
               bool(clamp_zero), order, 0 if filter_3d is None else filter_3d.data_ptr(), bool(antialiased))
        if render_depth:
            sig += ("depth",)
        if render_normal:
            sig += ("normal",)
        self._run("fwd", sig, kernels)
        self.rendered_depth = render_depth
        self.rendered_normal = render_normal
        self.views_done += 1
        return self.img

    def backward(self, params, d_img, sh_degree, accumulate_into, use_clamp=True, camera_grad=None, antialiased=False, filter_3d=None,
                 exact_grad=False, d_depth=None, d_trans=None, d_normal=None):
        """d_img f32[1,3,H,W] or [1,3,Hp,Wp]: gradient of the loss w.r.t. the (clamped) image.  camera_grad (optional f32[2,4,4]
        CUDA tensor) receives (d view_matrix, d proj_matrix) of this view, copied on the stream after the backward.
        antialiased, filter_3d: the values the forward of this view was given.  exact_grad: exact gradient mode (DESIGN.md
        section 1); a backward-only choice, so it is part of the backward graph's signature and of nothing else.
        d_depth, d_trans: f32[1,1,H,W] or [1,1,Hp,Wp] gradients of the depth (the forward must have rendered it) and of the
        transmittance, or None; whether each is given is part of the backward graph's signature.
        d_normal: f32[1,3,H,W] or [1,3,Hp,Wp] gradient of the normal (the forward must have rendered it), or None; whether it is
        given is part of the backward graph's signature."""
        filter_3d = check_filter_3d(filter_3d, params["xyz"])
        if camera_grad is not None and not (camera_grad.is_cuda and camera_grad.dtype == _F32 and tuple(camera_grad.shape) == (2, 4, 4)):
            raise RuntimeError("camera_grad must be a float32 CUDA tensor of shape [2,4,4]")
        if d_depth is not None and not self.rendered_depth:
            raise RuntimeError("d_depth is given, but the last forward on this workspace did not render depth (render_depth=False)")
        if d_normal is not None and not self.rendered_normal:
            raise RuntimeError("d_normal is given, but the last forward on this workspace did not render normals (render_normal=False)")
        cam, dep, trans, nrm = camera_grad is not None, d_depth is not None, d_trans is not None, d_normal is not None
        tiled = bool(CONFIG["tile_order"])
        if nrm:
            self._plane("grad_normal", (self.Nmax, 4))
        H, W = self.hw
        for name, g, c in (("d_img", d_img, 3), ("d_depth", d_depth, 1), ("d_trans", d_trans, 1), ("d_normal", d_normal, 3)):
            if g is None:
                continue
            plane = self._plane(name, (1, c, self.Hp, self.Wp))
            if g.shape[-2:] == (self.Hp, self.Wp):
                plane.copy_(g, non_blocking=True)
            else:
                if self.Hp != H or self.Wp != W:
                    plane.zero_()
                plane[..., :H, :W].copy_(g, non_blocking=True)

        def kernels():
            st = _stream(self.dev)
            _raster_backward(st, self.hw, self.tile, self.sorted_pid, self.ranges, self.packed, self.tile_order if tiled else None, self.T,
                             self.last, self.d_img, self.d_trans if trans else None, self.img if use_clamp else None, False, self.pg,
                             self.d_depth if dep else None, self.normal_rec if nrm else None, self.d_normal if nrm else None,
                             self.grad_normal if nrm else None)
            # A = all chunks: project_backward returns at once for chunks past the (device) visible count
            _project_backward(st, params, sh_degree, self.chunk_ids, self.counters, self.cam_view, self.cam_proj, self.hw, self.C, self.pg,
                              2, [accumulate_into[k] for k in _KEYS], accumulate_into.get("_touched"), self.cam_partials if cam else None,
                              self.d_cam if cam else None, filter_3d, antialiased, exact_grad, dep, self.grad_normal if nrm else None)

        sig = (tuple(params[k].data_ptr() for k in _KEYS), tuple(accumulate_into[k].data_ptr() for k in _KEYS),
               0 if accumulate_into.get("_touched") is None else accumulate_into["_touched"].data_ptr(), int(sh_degree), bool(use_clamp),
               tiled, bool(antialiased), 0 if filter_3d is None else filter_3d.data_ptr(), bool(exact_grad), cam)
        if dep or trans:
            sig += (("depth", dep, trans),)
        if nrm:
            sig += ("normal",)
        self._run("bwd", sig, kernels)
        if cam:
            camera_grad.copy_(self.d_cam, non_blocking=True)

    # -- feedback --------------------------------------------------------------------------------------------------
    def post_flags(self):
        """Enqueue (on the current stream) the copy of the sticky overflow word to a pinned buffer of its own and reset the word on
        the device.  The result stays queued until check() reads it: a post whose copy has not landed when the next one is made
        is never dropped or overwritten."""
        host = self._free_host.pop() if self._free_host else torch.zeros(4, dtype=_I32).pin_memory()
        host.copy_(self.sticky, non_blocking=True)
        self.sticky.zero_()
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        self._posted.append((ev, host))

    def check(self, wait: bool = False):
        """Fold the results of every post_flags() not yet read, oldest first, that have landed (with wait, all of them: waits
        for their copies).  None if there is none; otherwise a dict over the folded posts (max pairs and depth bits of a view, the
        number of views), or CapacityExceeded if a view of any of them overflowed a prediction (its lists were truncated).
        Posts that have not landed stay queued for a later check."""
        flags, pairs, bits, views, read = 0, 0, 0, 0, 0
        while self._posted:
            ev, host = self._posted[0]
            if not ev.query():
                if not wait:
                    break
                ev.synchronize()
            self._posted.popleft()
            f, p, b, v = (int(x) for x in host)
            self._free_host.append(host)
            flags, pairs, bits, views, read = flags | f, max(pairs, p), max(bits, b), views + v, read + 1
        if not read:
            return None
        if flags:
            raise CapacityExceeded(pairs=pairs, pair_capacity=self.cap, depth_bits=bits, planned_depth_bits=self.planned_bits)
        return {"max_pairs": pairs, "max_depth_bits": bits, "views": views}


class CapacityExceeded(RuntimeError):
    def __init__(self, pairs, pair_capacity, depth_bits, planned_depth_bits):
        super().__init__(f"view workspace too small: {pairs} (tile, splat) pairs for a capacity of {pair_capacity}, depth keys span {depth_bits} "
                         f"bits with {planned_depth_bits} planned; grow the workspace and redo the step")
        self.pairs, self.pair_capacity, self.depth_bits, self.planned_depth_bits = pairs, pair_capacity, depth_bits, planned_depth_bits


def probe_view_sizes(params, cluster_origin, cluster_extend, cams, sh_degree, hw, tile, antialiased=False, filter_3d=None):
    """One synchronising forward per camera (the cold path) -> (max pairs, max depth-key bits): the first-epoch sizing step of
    the reference's feedback protocol, used to dimension a ViewWorkspace.  antialiased, filter_3d: size for that mode and filter
    (both change the pair count)."""
    max_pairs, max_bits = 0, 1
    p = {k: params[k].detach() for k in ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")}
    with torch.no_grad():
        for cam in cams:
            _, st, _ = render_view_forward(p, cluster_origin, cluster_extend, cam["frustumplane"], cam["view"], cam["proj"], sh_degree, hw, tile,
                                           antialiased=antialiased, filter_3d=filter_3d)
            max_pairs, max_bits = max(max_pairs, st.n_pairs), max(max_bits, st.depth_bits)
    return max_pairs, max_bits
