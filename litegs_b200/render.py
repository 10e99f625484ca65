"""The render operator: ``render_preprocess`` + ``render`` with the signatures of the reference's
``litegs/render/__init__.py:11-94`` (Level A: op by op through ``litegs_b200.wrapper``), and
``render_view`` -- the same computation as ONE differentiable call on the fused pipeline (Level B).

Both levels produce the same image and the same six parameter gradients (tests/test_gpu_pipeline.py);
Level B is what ``bench.py`` measures.
"""
from __future__ import annotations

import copy
import math
import os
from collections import namedtuple
from typing import Optional

import torch
import torch.cuda.nvtx as nvtx

from . import pipeline, wrapper
from .compacted import CompactedTensor
from .statistics import StatisticsHelperInst


def uncluster(*tensors):
    """[..., chunks, chunk_size] -> [..., chunks*chunk_size] views (reference scene/cluster.py:24-28)."""
    return tuple(t.reshape(*t.shape[:-2], t.shape[-2] * t.shape[-1]) for t in tensors)


_Modes = namedtuple("_Modes", "antialiased exact_grad render_depth render_normal")


def _modes(pp) -> _Modes:
    """The fused path's opt-in modes (DESIGN.md section 1), read with getattr so that the reference's own PipelineParams, which
    has none of them, still works (absent = off)."""
    return _Modes(*(bool(getattr(pp, f, False)) for f in _Modes._fields))


# ---------------------------------------------------------------------------------------------------
# Level A: the reference's two-call surface
# ---------------------------------------------------------------------------------------------------

def render_preprocess(cluster_origin, cluster_extend, frustumplane, view_matrix,
                      xyz, scale, rot, sh_0, sh_rest, opacity,
                      feedback_buffer, idx_tensor, pp, actived_sh_degree: int):
    """Chunk frustum culling -> compaction -> activation (+ SH->RGB).

    Returns (visible_chunkid, visible_chunks_num, culled_xyz [4,N], culled_scale [3,N], culled_rot [4,N],
    color [V,3,N], culled_opacity [1,N]) exactly as render/__init__.py:11-48."""
    visible_chunkid = None
    visible_chunks_num = None
    if pp.cluster_size:
        if cluster_origin is None or cluster_extend is None:
            raise RuntimeError("cluster_origin / cluster_extend are required when cluster_size > 0 "
                               "(compute them with litegs_b200.scene.cluster_aabb or the caller's scene code)")
        _, visible_chunks_num, visible_chunkid = wrapper.litegs_fused.frustum_culling_aabb(cluster_origin, cluster_extend, frustumplane,
                                                                                 feedback_buffer, idx_tensor)
        if StatisticsHelperInst.bStart and StatisticsHelperInst.on_compact_mask is not None:
            StatisticsHelperInst.on_compact_mask(visible_chunkid, visible_chunks_num)
        culled = wrapper.CullCompactActivateWithSparseGrad.apply(pp.sparse_grad, actived_sh_degree, visible_chunkid,
                                                                 visible_chunks_num, view_matrix, xyz, scale, rot, sh_0, sh_rest, opacity)
        culled_xyz, culled_scale, culled_rot, color, culled_opacity = uncluster(*culled)
    else:
        nvtx.range_push("Activate")
        ones = torch.ones((1, xyz.shape[-1]), dtype=xyz.dtype, device=xyz.device)
        culled_xyz = torch.cat((xyz, ones), dim=0)
        culled_scale = scale.exp()
        culled_rot = torch.nn.functional.normalize(rot, dim=0)
        culled_opacity = opacity.sigmoid()
        with torch.no_grad():
            R = view_matrix[..., :3, :3]
            t = view_matrix[..., 3:4, :3]
            camera_center = (-t @ R.transpose(-1, -2)).squeeze(1)
            dirs = torch.nn.functional.normalize(culled_xyz[:3] - camera_center.unsqueeze(-1), dim=-2)
        color = wrapper.SphericalHarmonicToRGB.call_fused(actived_sh_degree, sh_0, sh_rest, dirs)
        nvtx.range_pop()
    return visible_chunkid, visible_chunks_num, culled_xyz, culled_scale, culled_rot, color, culled_opacity


def render(view_matrix, proj_matrix, xyz, scale, rot, color, opacity,
           valid_length, feedback_binning_allocate_size, idx_tensor,
           actived_sh_degree: int, output_shape, pp):
    """Projection -> binning -> rasterisation; returns (img, transmittance, depth, normal, primitive_visible)
    as render/__init__.py:50-94.  The antialiased, exact gradient, depth and normal modes exist on the fused path only (render_view,
    render_views)."""
    why = {"antialiased": "has no antialiased mode and would draw every splat without its opacity compensation",
           "exact_grad": "has no exact gradient mode and would return position gradients with J and the SH direction held constant",
           "render_depth": "has no depth mode (its depth slot keeps the reference's enable_depth contract)",
           "render_normal": "has no normal mode (its normal slot stays None)"}
    for flag, on in _modes(pp)._asdict().items():
        if on:
            raise RuntimeError(f"pp.{flag} is set, but the op-by-op render() {why[flag]}; render through render_view or render_views instead")
    nvtx.range_push("Proj")
    view_pos, ndc_pos = wrapper.MVPTransform.apply(xyz, view_matrix, proj_matrix, valid_length)
    transform_matrix = wrapper.CreateTransformMatrix.call_fused(scale, rot, valid_length)
    J = wrapper.CreateRaySpaceTransformMatrix.call_fused(view_pos, proj_matrix, output_shape, valid_length)
    cov2d = wrapper.CreateCov2dDirectly.call_fused(J, view_matrix, transform_matrix, valid_length)
    _, _, inv_cov2d = wrapper.EighAndInverse2x2Matrix.call_fused(cov2d, valid_length)
    view_depth = view_pos[:, 2, :]
    nvtx.range_pop()

    tile_start_index, sorted_pointId, primitive_visible = wrapper.Binning.call_fused(
        ndc_pos, view_depth, inv_cov2d, opacity, valid_length, feedback_binning_allocate_size, idx_tensor,
        output_shape, pp.tile_size)

    tiles = None
    cached = StatisticsHelperInst.cached_sorted_tile_list.get(StatisticsHelperInst.cur_sample)
    if cached is not None:
        tiles = cached.unsqueeze(0)
    H, W = int(output_shape[0]), int(output_shape[1])
    img, transmitance, depth, normal, last = wrapper.GaussiansRasterFunc.apply(
        sorted_pointId, tile_start_index, ndc_pos, inv_cov2d, color, opacity, tiles, H, W,
        pp.tile_size[0], pp.tile_size[1], pp.enable_transmitance, pp.enable_depth)
    if StatisticsHelperInst.bStart and StatisticsHelperInst.on_blend_count is not None:
        StatisticsHelperInst.on_blend_count(last, pp.tile_size[0], pp.tile_size[1])

    img = img[..., :H, :W].clamp(0, 1).contiguous()
    if transmitance is not None:
        transmitance = transmitance[..., :H, :W].contiguous()
    if depth is not None:
        depth = depth[..., :H, :W].contiguous()
    return img, transmitance, depth, normal, primitive_visible


# ---------------------------------------------------------------------------------------------------
# Level B: one differentiable call per view
# ---------------------------------------------------------------------------------------------------

@torch.no_grad()
def _feed_statistics(state, stats, packed_grad, tile):
    """What Level A feeds the StatisticsHelper op by op (render/__init__.py:24-25,84-85; wrapper.py:501-506,733-737), from the
    fused pipeline's state: compact mask + device-side visible count, visible splats, fragment weight / count, fragment error
    (d_opacity = sum s0 / o and the err_square term of the gradient record), per-tile blend counts."""
    SH = StatisticsHelperInst
    if SH.on_compact_mask is not None:
        SH.on_compact_mask(state.chunk_ids, state.counters[:1])
    if SH.on_visible is not None:
        SH.on_visible((state.tile_count > 0).reshape(1, -1))
    fc, fw = stats
    if SH.on_fragment_weight is not None:
        SH.on_fragment_weight(fw, fc)
    if SH.on_fragment_err is not None and packed_grad is not None:
        o = state.packed[..., 5]
        d_op = torch.where(o > 0, packed_grad[..., 8] / o.clamp_min(1e-30), torch.zeros_like(o))
        SH.on_fragment_err(d_op.unsqueeze(0), packed_grad[..., 9].unsqueeze(0), fc)
    if SH.on_blend_count is not None:
        SH.on_blend_count(state.last, tile[0], tile[1])


class _RenderViewFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, scale, rot, sh_0, sh_rest, opacity, cluster_origin, cluster_extend, frustumplane,
                view_matrix, proj_matrix, sh_degree, hw, tile, sparse_grad, enable_transmitance, accumulate_into, filter_3d, modes):
        params = dict(xyz=xyz, scale=scale, rot=rot, sh_0=sh_0, sh_rest=sh_rest, opacity=opacity)
        stat = bool(StatisticsHelperInst.bStart)
        ctx.set_materialize_grads(False)       # an unused transmittance output must not cost a zero-filled gradient image
        # the kernel writes clamp(c,0,1) directly (render/__init__.py:87 does it as a separate pass) ...
        img, state, stats = pipeline.render_view_forward(params, cluster_origin, cluster_extend, frustumplane, view_matrix,
                                                         proj_matrix, sh_degree, hw, tile, enable_statistic=stat, clamp_zero=True,
                                                         antialiased=modes.antialiased, filter_3d=filter_3d,
                                                         render_depth=modes.render_depth, render_normal=modes.render_normal)
        ctx.state = state
        ctx.stats = stats
        ctx.stat = stat
        ctx.sparse = bool(sparse_grad)
        ctx.trans = bool(enable_transmitance)
        ctx.accumulate_into = accumulate_into
        ctx.exact_grad = modes.exact_grad           # backward only: the forward does not depend on it
        ctx.save_for_backward(xyz, scale, rot, sh_0, sh_rest, opacity, img)
        ctx.mark_non_differentiable(state.last)
        return img, state.T, state.last, state.depth, state.normal   # depth, normal: None unless render_depth, render_normal

    @staticmethod
    def backward(ctx, g_img, g_T, _g_last, g_depth, g_normal):
        xyz, scale, rot, sh_0, sh_rest, opacity, img_out = ctx.saved_tensors
        params = dict(xyz=xyz, scale=scale, rot=rot, sh_0=sh_0, sh_rest=sh_rest, opacity=opacity)
        state = ctx.state
        if g_img is None:
            g_img = torch.zeros((1, 3, *state.T.shape[-2:]), dtype=torch.float32, device=xyz.device)
        # ... and the backward kernel applies that clamp's gradient mask from the saved image
        # camera gradient only when the view or projection matrix asks for one: otherwise the kernel without it runs
        cam = None
        if ctx.needs_input_grad[9] or ctx.needs_input_grad[10]:
            cam = torch.empty((2, 4, 4), dtype=torch.float32, device=xyz.device)
        grads, pg = pipeline.render_view_backward(params, state, g_img, g_T if (ctx.trans and g_T is not None) else None,
                                                  enable_statistic=ctx.stat,
                                                  accumulate_into=ctx.accumulate_into, clamped_img=img_out, camera_grad=cam,
                                                  exact_grad=ctx.exact_grad, d_depth=g_depth, d_normal=g_normal)
        if ctx.stat:
            _feed_statistics(state, ctx.stats, pg, state.tile)
        out = [None] * len(ctx.needs_input_grad)           # one slot per input of forward
        if cam is not None:
            out[9] = cam[0].reshape(state.view.shape) if ctx.needs_input_grad[9] else None
            out[10] = cam[1].reshape(state.proj.shape) if ctx.needs_input_grad[10] else None
        if grads is not None:      # None: the gradients went straight into the caller's dense buffers
            C, S = xyz.shape[-2:]
            ids = state.chunk_ids[: state.n_chunks_visible]
            for k, g in enumerate(grads):
                ct = CompactedTensor((*g.shape[:-2], C, S), ids, g)
                out[k] = ct if ctx.sparse else ct.to_dense()
        ctx.state = None
        return tuple(out)


def render_view(cluster_origin, cluster_extend, frustumplane, view_matrix, proj_matrix,
                xyz, scale, rot, sh_0, sh_rest, opacity, actived_sh_degree: int, output_shape, pp, accumulate_into=None, filter_3d=None):
    """render_preprocess + render of one view on the fused pipeline.

    Same inputs as the two reference calls (raw clustered parameters, chunk AABBs, camera); returns the five values of the
    reference's render() with the contributor counts in the last slot: (img [1,3,H,W] clamped to [0,1], transmittance or
    None, depth=None, normal=None, last_contributor [1,1,Hp,Wp]).  Gradients reach the six parameter tensors as CompactedTensor (pp.sparse_grad) or dense
    tensors -- or, with ``accumulate_into`` (dict of dense gradient tensors, e.g. ``GradAccumulator.grads()``), are
    ADDED into those buffers by the backward kernel itself and ``param.grad`` stays untouched (multi-view batches,
    data-parallel training).  ``pp.antialiased`` (absent = False) selects the antialiased mode (DESIGN.md section 1).
    ``pp.exact_grad`` (absent = False) selects the exact gradient mode (DESIGN.md section 1): the xyz and camera gradients also
    carry the terms through the ray-space Jacobian J and the SH view direction.
    ``pp.render_depth`` (absent = False) also renders the per-pixel depth D = sum_i w_i z_i (DESIGN.md section 1, "Depth") and
    returns it, differentiable, in the depth slot as [1,1,H,W]; the expected depth is D / (1 - transmittance).  ``pp.enable_depth``
    keeps the reference's meaning.
    ``pp.render_normal`` (absent = False) also renders the per-pixel normal N = sum_i w_i n_i, n_i the camera-facing view-space
    normal of Gaussian i's shortest axis (DESIGN.md section 1, "Normals"), and returns it, differentiable, in the normal slot as
    [1,3,H,W]; the expected normal is N / (1 - transmittance), the unit normal N / |N|.
    ``filter_3d`` (f32[1,C,S] or None): Mip-Splatting's 3D smoothing filter (scene.filter_3d_device, DESIGN.md section 1); it is
    an input without a gradient."""
    if not pp.cluster_size:
        raise RuntimeError("render_view needs the clustered layout (cluster_size > 0); use render_preprocess + render otherwise")
    H, W = int(output_shape[0]), int(output_shape[1])
    th, tw = int(pp.tile_size[0]), int(pp.tile_size[1])
    img, T, last, depth, normal = _RenderViewFn.apply(xyz, scale, rot, sh_0, sh_rest, opacity, cluster_origin, cluster_extend,
                                                      frustumplane, view_matrix, proj_matrix, int(actived_sh_degree), (H, W), (th, tw),
                                                      pp.sparse_grad, pp.enable_transmitance, accumulate_into, filter_3d, _modes(pp))
    img = img[..., :H, :W]          # already clamped to [0,1] by the kernel
    trans = T[..., :H, :W] if pp.enable_transmitance else None
    return (img, trans, None if depth is None else depth[..., :H, :W], None if normal is None else normal[..., :H, :W], last)


# ---------------------------------------------------------------------------------------------------
# multi-view micro-batch: views pipelined over CUDA streams, gradients summed in dense buffers
# ---------------------------------------------------------------------------------------------------

_side_streams: dict = {}
# render_views drives the pipeline's forward/backward directly and uses autograd only for the caller's loss (default);
# LGS_VIEWS_AUTOGRAD=1 routes every view through the render_view autograd Function instead (A/B switch)
_DIRECT_VIEWS = os.environ.get("LGS_VIEWS_AUTOGRAD", "0") != "1"


def _streams(dev, n):
    key = (dev, n)
    if key not in _side_streams:
        _side_streams[key] = [torch.cuda.Stream(device=dev) for _ in range(n)]
    return _side_streams[key]


def render_views(n_views: int, camera_fn, loss_fn, cluster_origin, cluster_extend,
                 xyz, scale, rot, sh_0, sh_rest, opacity, actived_sh_degree: int, output_shape, pp,
                 accumulate_into: dict, n_streams: int = 4, loss_and_grad_fn=None, camera_grads=None, filter_3d=None):
    """Forward + backward of a batch of views with the gradients summed into ``accumulate_into`` (dense tensors shaped
    like the parameters, e.g. ``GradAccumulator.grads()``).  This is the per-rank body of a data-parallel step.

    ``camera_fn(i)`` -> dict(view, proj, frustumplane) and ``loss_fn(i, img)`` -> scalar loss are called with view i's
    stream current (so H2D copies issued inside them are ordered correctly).  ``loss_fn`` may instead return
    ``(loss, d_img)`` -- the scalar and dloss/dimg computed outside autograd, e.g. ``ssim.l1_ssim_loss_and_grad(img.detach(),
    gt)`` -- in which case the image gradient is fed straight to the rasterizer's backward.  Consecutive views alternate over
    ``n_streams`` CUDA streams: view i+1's forward (bandwidth-bound projection / sort kernels and the one host
    read-back) overlaps view i's backward (issue-bound raster kernel).  Views only interact through the dense
    accumulate, which is ordered by an event.  Returns the list of (detached) per-view losses.

    ``loss_and_grad_fn(i, img) -> (loss, d_img)`` (with ``loss_fn=None``) skips autograd altogether: the pipeline's forward
    and backward are called directly (no autograd Function, no engine hop: ~0.1 ms less host time per view), the image
    handed to the function is the kernel's clamp(0,1) output and its gradient goes straight to the raster backward.

    ``camera_grads`` (optional contiguous f32[n_views,2,4,4] CUDA tensor): slot i receives (d view_matrix, d proj_matrix) of view i
    (pipeline.render_view_backward), on every path; it is complete when this function returns (the current stream waits).

    ``filter_3d`` (f32[1,C,S] or None): the 3D smoothing filter every view of the batch is drawn with (see render_view).

    ``pp.render_depth`` (absent = False): every view also renders its depth (see render_view), and the callbacks take it with the
    transmittance: ``loss_fn(i, img, depth, trans)`` -> scalar (autograd over the three [1,C,H,W] inputs) or ``(loss, d_img,
    d_depth, d_trans)``, and ``loss_and_grad_fn(i, img, depth, trans) -> (loss, d_img, d_depth, d_trans)``, where d_depth and
    d_trans may be None.  An expected-depth loss uses depth / (1 - trans).  Without the flag both callbacks are called as above.

    ``pp.render_normal`` (absent = False): every view also renders its normal (see render_view), and the callbacks take it
    appended to the depth form: ``loss_fn(i, img, depth, trans, normal)`` -> scalar or ``(loss, d_img, d_depth, d_trans,
    d_normal)``, and ``loss_and_grad_fn(i, img, depth, trans, normal) -> (loss, d_img, d_depth, d_trans, d_normal)``; depth (and
    d_depth) is None unless ``pp.render_depth`` is set.  Without the flag the callbacks are called as above."""
    dev = xyz.device
    filter_3d = pipeline.check_filter_3d(filter_3d, xyz)
    if camera_grads is not None and not (camera_grads.is_cuda and camera_grads.dtype == torch.float32 and camera_grads.is_contiguous()
                                         and tuple(camera_grads.shape) == (n_views, 2, 4, 4)):
        raise RuntimeError(f"camera_grads must be a contiguous float32 CUDA tensor of shape [{n_views},2,4,4]")
    slot = (lambda i: None) if camera_grads is None else (lambda i: camera_grads[i])
    losses = []
    H, W = int(output_shape[0]), int(output_shape[1])
    th, tw = int(pp.tile_size[0]), int(pp.tile_size[1])
    aa, exact, dep, nrm = _modes(pp)
    direct = loss_and_grad_fn is not None or _DIRECT_VIEWS
    if direct:
        params = dict(xyz=xyz.detach(), scale=scale.detach(), rot=rot.detach(), sh_0=sh_0.detach(), sh_rest=sh_rest.detach(),
                      opacity=opacity.detach())
        stat = bool(StatisticsHelperInst.bStart)

    def callback_args(img, depth, trans, normal):
        """What the callbacks take after i: the image, then (depth, trans) with depth or normals on, then the normal with normals on."""
        return [img] + ([depth, trans] if dep or nrm else []) + ([normal] if nrm else [])

    def loss_and_grads(i, img_p, depth_p, T_p, normal_p):
        """Either callback on view i's padded outputs -> (loss, d_img, d_depth, d_trans, d_normal); every gradient but d_img may be
        None.  Autograd runs through the caller's loss only, never through the render kernels."""
        ins = [None if t is None else t[..., :H, :W] for t in callback_args(img_p, depth_p, T_p, normal_p)]
        if loss_and_grad_fn is not None:
            out = tuple(loss_and_grad_fn(i, *ins))
        else:
            leaves = [None if t is None else t.detach().requires_grad_(True) for t in ins]
            out = loss_fn(i, *leaves)
            if not isinstance(out, tuple):
                gs = iter(torch.autograd.grad(out, [t for t in leaves if t is not None], allow_unused=True))
                out = (out, *(None if t is None else next(gs) for t in leaves))
        loss, d_img, d_depth, d_trans, d_normal = out + (None,) * (5 - len(out))
        return loss, (torch.zeros_like(ins[0]) if d_img is None else d_img), d_depth, d_trans, d_normal

    def one_direct(i, wait_ev):
        cam = camera_fn(i)
        img_p, state, stats = pipeline.render_view_forward(params, cluster_origin, cluster_extend, cam["frustumplane"], cam["view"],
                                                           cam["proj"], int(actived_sh_degree), (H, W), (th, tw), enable_statistic=stat,
                                                           clamp_zero=True, antialiased=aa, filter_3d=filter_3d, render_depth=dep,
                                                           render_normal=nrm)
        loss, d_img, d_depth, d_trans, d_normal = loss_and_grads(i, img_p, state.depth, state.T, state.normal)
        if d_img.shape[-2:] != img_p.shape[-2:]:                        # image padded to whole tiles: pad the gradient with zeros
            d_img = torch.nn.functional.pad(d_img, (0, img_p.shape[-1] - W, 0, img_p.shape[-2] - H))
        if d_trans is not None:
            d_trans = pipeline._padded(d_trans, state.T.shape)
        if wait_ev is not None:
            torch.cuda.current_stream(dev).wait_event(wait_ev)
        _, pg_ = pipeline.render_view_backward(params, state, d_img, d_trans, enable_statistic=stat, accumulate_into=accumulate_into,
                                               clamped_img=img_p, camera_grad=slot(i), exact_grad=exact, d_depth=d_depth,
                                               d_normal=d_normal)
        if stat:
            _feed_statistics(state, stats, pg_, (th, tw))
        losses.append(loss.detach())
        return state

    def one_autograd(i, wait_ev):
        cam = camera_fn(i)
        view, proj = cam["view"], cam["proj"]
        if camera_grads is not None:              # leaves of this call: their .grad is view i's camera gradient
            view, proj = view.detach().requires_grad_(True), proj.detach().requires_grad_(True)
        pp_i = pp
        if (dep or nrm) and not pp.enable_transmitance:    # the depth / normal callbacks take the transmittance
            pp_i = copy.copy(pp)
            pp_i.enable_transmitance = True
        img, trans, depth, normal, _ = render_view(cluster_origin, cluster_extend, cam["frustumplane"], view, proj, xyz, scale, rot,
                                                   sh_0, sh_rest, opacity, actived_sh_degree, output_shape, pp_i,
                                                   accumulate_into=accumulate_into, filter_3d=filter_3d)
        ins = callback_args(img, depth, trans, normal)
        loss = loss_fn(i, *ins)
        if wait_ev is not None:          # the previous view's accumulate (other stream) must have landed
            torch.cuda.current_stream(dev).wait_event(wait_ev)
        if isinstance(loss, tuple):
            loss, *gs = loss
            pairs = [(t, g) for t, g in zip(ins, gs) if t is not None and g is not None]
            torch.autograd.backward([t for t, _ in pairs], [g for _, g in pairs])
        else:
            loss.backward()
        if camera_grads is not None:
            camera_grads[i, 0].copy_(view.grad.reshape(4, 4)); camera_grads[i, 1].copy_(proj.grad.reshape(4, 4))
        losses.append(loss.detach())

    # GPU-driven path (default): one preallocated ViewWorkspace per stream slot, no host synchronisation inside the batch, the
    # per-view forward / backward replayed as CUDA graphs.  The first batch of a configuration goes through the synchronising
    # path and measures the capacities (the reference's cold first epoch); statistics runs keep the synchronising path.
    slots = None
    if direct and pipeline.SYNC_FREE and not stat:
        slots = _view_slots(params, (H, W), (th, tw), max(1, n_streams), aa, filter_3d is not None)
        if slots.big:
            slots = None
    probe = {"pairs": 0, "bits": 1} if (slots is not None and slots.ws is None) else None

    def one_ws(i, wait_ev):
        ws = slots.ws[i % max(1, n_streams)]
        cam = camera_fn(i)
        img_p = ws.forward(params, cluster_origin, cluster_extend, cam, int(actived_sh_degree), clamp_zero=True, antialiased=aa,
                           filter_3d=filter_3d, render_depth=dep, render_normal=nrm)
        loss, d_img, d_depth, d_trans, d_normal = loss_and_grads(i, img_p, ws.depth if dep else None, ws.T, ws.normal)
        if wait_ev is not None:
            torch.cuda.current_stream(dev).wait_event(wait_ev)
        ws.backward(params, d_img, int(actived_sh_degree), accumulate_into, use_clamp=True, camera_grad=slot(i), antialiased=aa,
                    filter_3d=filter_3d, exact_grad=exact, d_depth=d_depth, d_trans=d_trans, d_normal=d_normal)
        losses.append(loss.detach())

    def one_probe(i, wait_ev):
        state = one_direct(i, wait_ev)
        probe["pairs"] = max(probe["pairs"], state.n_pairs); probe["bits"] = max(probe["bits"], state.depth_bits)

    use_ws = slots is not None and slots.ws is not None
    if use_ws:
        slots.check()
        one = one_ws
    elif probe is not None:
        one = one_probe
    else:
        one = one_direct if direct else one_autograd
    if n_streams <= 1:
        for i in range(n_views):
            one(i, None)
        if use_ws:
            slots.ws[0].post_flags()
        elif probe is not None:
            slots.size(probe["pairs"], probe["bits"])
        return losses
    cur = torch.cuda.current_stream(dev)
    side = _streams(dev, n_streams)
    for s in side:
        s.wait_stream(cur)
    prev = None
    for i in range(n_views):
        s = side[i % n_streams]
        with torch.cuda.stream(s):
            one(i, prev)
            prev = torch.cuda.Event()
            prev.record(s)
    if use_ws:
        for k, s in enumerate(side[: min(n_streams, n_views)]):
            with torch.cuda.stream(s):
                slots.ws[k].post_flags()
    elif probe is not None:
        slots.size(probe["pairs"], probe["bits"])
    for s in side:
        cur.wait_stream(s)
    return losses


class _ViewSlots:
    """The per-configuration state of render_views' GPU-driven path: capacities measured by the first (synchronising) batch and
    one ViewWorkspace per stream slot, created from them.  The antialiased mode and the use of a 3D filter are part of the
    configuration: both change the pair count, so capacities measured with one setting could overflow with another."""

    def __init__(self, params, hw, tile):
        self.params_like, self.hw, self.tile = params, hw, tile
        self.ws = None
        self.big = False
        self.cap, self.bits = 0, 24

    def size(self, max_pairs, max_bits):
        """Capacities from the measured maxima: 30 % head-room on the pairs, the depth range rounded up to whole 8-bit passes (a
        view that needs more is flagged and the step redone)."""
        self.cap = int(max_pairs * 1.3) + 65536
        self.bits = min(32, 8 * ((max_bits + 7) // 8))
        H, W = self.hw
        ntile = ((W + self.tile[1] - 1) // self.tile[1]) * ((H + self.tile[0] - 1) // self.tile[0])
        # very large pair lists with 8-bit tile digits (4K frames): the library's onesweep, which needs the count on the host,
        # beats the own passes (csrc/sort.cu: sort_impl_for) and such views are device-bound anyway -> stay on the synchronising path
        self.ws = None if (ntile.bit_length() > 14 and max_pairs > (8 << 20)) else []
        self.big = self.ws is None

    def ensure(self, n_slots):
        """One workspace per stream slot (created on demand once the capacities are known)."""
        while self.ws is not None and len(self.ws) < n_slots:
            self.ws.append(pipeline.ViewWorkspace(self.params_like, self.hw, self.tile, self.cap, self.bits))

    def check(self):
        """Overflow flags of the earlier batches that have landed (the others stay queued for the next check): on overflow drop the
        workspaces -- the next batch measures again -- and tell the caller to redo the step."""
        try:
            for w in self.ws:
                w.check(wait=False)
        except pipeline.CapacityExceeded:
            self.ws = None
            raise


_slot_cache: dict = {}


def _view_slots(params, hw, tile, n_slots, antialiased=False, filtered=False):
    xyz = params["xyz"]
    key = (xyz.device, tuple(xyz.shape[-2:]), hw, tile, params["sh_rest"].shape[0], bool(antialiased), bool(filtered))
    ent = _slot_cache.get(key)
    if ent is None:
        ent = _slot_cache[key] = _ViewSlots(params, hw, tile)
    ent.ensure(n_slots)
    return ent


def check_views(wait: bool = True):
    """Explicit form of the lazy overflow check of render_views' GPU-driven path: raises pipeline.CapacityExceeded if a view of
    any batch whose flags were not read yet overflowed its workspace -- redo that step.  wait: wait for the flags of every batch
    enqueued so far (else only those that have landed are read; the rest stay queued)."""
    for ent in _slot_cache.values():
        if ent.ws is not None:
            try:
                for w in ent.ws:
                    w.check(wait=wait)
            except pipeline.CapacityExceeded:
                ent.ws = None
                raise


def reset_view_workspaces():
    """Forget every cached workspace / CUDA graph (call after the scene's size changed, e.g. densification)."""
    _slot_cache.clear()
