"""Differentiable operators of the render path -- the surface of the reference's ``litegs/utils/wrapper.py``
(same class / function names and call signatures) on top of ``litegs_b200.fused``.

Each operator is a ``torch.autograd.Function`` whose forward and backward are single calls into the CUDA
library.  There are deliberately no "script" (pure PyTorch) twins here: the reference uses those only to
validate its kernels (wrapper.py:21-164); that job belongs to the CPU oracle under ``oracle/`` and the
tests.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import fused as litegs_fused
from .compacted import CompactedTensor
from .statistics import StatisticsHelperInst


def set_backend(module) -> None:
    """Route every operator of this module (and render.render_preprocess / render) to another object with the
    ``litegs_fused`` surface.  Used by tests and bench.py to run the SAME orchestration on the reference's own
    kernels (oracle/_ref) for the Tier-2 comparison; the default is ``litegs_b200.fused``."""
    global litegs_fused
    litegs_fused = module


class _Op:
    """call_fused / call, as on the reference's BaseWrapper (wrapper.py:149-159)."""
    @classmethod
    def call_fused(cls, *args, **kwargs):
        return cls._fused(*args, **kwargs)

    @classmethod
    def call(cls, *args, **kwargs):
        return cls._fused(*args, **kwargs)


class MVPTransform(torch.autograd.Function):
    """world [4,N] -> (view_pos, ndc_pos) [V,4,N]   (wrapper.py:270-285)."""
    @staticmethod
    def forward(ctx, position, view_matrix, proj_matrix, valid_length=None):
        view_pos, ndc_pos = litegs_fused.mvp_transform_forward(position, view_matrix, proj_matrix, valid_length)
        ctx.save_for_backward(view_pos, view_matrix, proj_matrix, valid_length)
        return view_pos, ndc_pos

    @staticmethod
    def backward(ctx, grad_view_pos, grad_ndc_pos):
        view_pos, view_matrix, proj_matrix, valid_length = ctx.saved_tensors
        if grad_view_pos is None:
            grad_view_pos = torch.zeros_like(view_pos)
        if grad_ndc_pos is None:
            grad_ndc_pos = torch.zeros_like(view_pos)
        g = litegs_fused.mvp_transform_backward(grad_ndc_pos, grad_view_pos, view_matrix, proj_matrix, view_pos, valid_length)
        return g, None, None, None


class _TransformMatrixFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, quaternion, scale, valid_length):
        ctx.save_for_backward(quaternion, scale, valid_length)
        return litegs_fused.createTransformMatrix_forward(quaternion, scale, valid_length)

    @staticmethod
    def backward(ctx, grad_T):
        quaternion, scale, valid_length = ctx.saved_tensors
        gq, gs = litegs_fused.createTransformMatrix_backward(grad_T, quaternion, scale, valid_length)
        return gq, gs, None


class CreateTransformMatrix(_Op):
    """T = diag(scale) R(quaternion), [3,3,N]   (wrapper.py:166-225); note the (scale, rot) argument order."""
    @staticmethod
    def _fused(scaling_vec, rotator_vec, valid_length=None):
        return _TransformMatrixFn.apply(rotator_vec, scaling_vec, valid_length)


class CreateRaySpaceTransformMatrix(_Op):
    """Perspective Jacobian [V,3,3,N]; carries no gradient (wrapper.py:257-260)."""
    @staticmethod
    @torch.no_grad()
    def _fused(view_pos, proj_matrix, output_shape, valid_length=None):
        return litegs_fused.jacobianRayspace(view_pos, proj_matrix, output_shape[0], output_shape[1], valid_length)


class _Cov2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, J, view_matrix, transform_matrix, valid_length):
        ctx.save_for_backward(J, view_matrix, transform_matrix, valid_length)
        return litegs_fused.createCov2dDirectly_forward(J, view_matrix, transform_matrix, valid_length)

    @staticmethod
    def backward(ctx, grad_cov2d):
        J, view_matrix, transform_matrix, valid_length = ctx.saved_tensors
        gT = litegs_fused.createCov2dDirectly_backward(grad_cov2d, J, view_matrix, transform_matrix, valid_length)
        return None, None, gT, None


class CreateCov2dDirectly(_Op):
    """cov2d = (T V J)^T (T V J) + 0.3 I, [V,2,2,N]   (wrapper.py:373-410)."""
    @staticmethod
    def _fused(J, view_matrix, transform_matrix, valid_length=None):
        return _Cov2dFn.apply(J, view_matrix, transform_matrix, valid_length)


class _EighInvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, matrix, valid_length):
        val, vec, inv = litegs_fused.eigh_and_inv_2x2matrix_forward(matrix, valid_length)
        ctx.save_for_backward(inv, valid_length)
        ctx.mark_non_differentiable(val, vec)
        return val, vec, inv

    @staticmethod
    def backward(ctx, _gval, _gvec, grad_inv):
        inv, valid_length = ctx.saved_tensors
        g = litegs_fused.inv_2x2matrix_backward(inv, grad_inv, valid_length)
        g.nan_to_num_(0)          # wrapper.py:591
        return g, None


class EighAndInverse2x2Matrix(_Op):
    """(eigenvalues, eigenvectors, inverse) of the 2x2 covariance; only the inverse is differentiable
    (wrapper.py:579-593)."""
    @staticmethod
    def _fused(cov2d, valid_length=None):
        return _EighInvFn.apply(cov2d, valid_length)


class _Sh2RgbFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, deg, sh_base, sh_rest, dirs):
        ctx.save_for_backward(dirs, sh_base, sh_rest)
        ctx.deg = deg
        return litegs_fused.sh2rgb_forward(deg, sh_base, sh_rest, dirs)

    @staticmethod
    def backward(ctx, grad_rgb):
        dirs, sh_base, sh_rest = ctx.saved_tensors
        g0, gr, gd = litegs_fused.sh2rgb_backward(ctx.deg, grad_rgb, sh_rest.shape[0], dirs, sh_base, sh_rest)
        return None, g0, gr, gd


class SphericalHarmonicToRGB(_Op):
    """SH -> RGB for the cluster_size=0 path, clamped at 0 (wrapper.py:541-558, SURVEY Q13)."""
    @staticmethod
    def _fused(deg, sh_base, sh_rest, dirs):
        return _Sh2RgbFn.apply(deg, sh_base, sh_rest, dirs).clamp_min(0)


class Binning(_Op):
    """Visibility table: count -> depth sort -> scan -> emit -> tile sort -> ranges   (wrapper.py:717-763).
    Returns (tile_start_index i32[V,tiles+2], sorted_pointId i32[V,alloc], per-point visible-view count)."""
    @staticmethod
    @torch.no_grad()
    def _fused(ndc, view_depth, inv_cov2d, opacity, valid_length, feedback_binning_allocate_size, idx_tensor,
               img_pixel_shape, tile_size):
        H, W = int(img_pixel_shape[0]), int(img_pixel_shape[1])
        th, tw = int(tile_size[0]), int(tile_size[1])
        tiles_num = math.ceil(H / th) * math.ceil(W / tw)
        _, _, allocate_size = litegs_fused.get_allocate_size(ndc, view_depth, inv_cov2d, opacity, H, W, th, tw, valid_length)
        b_visible = allocate_size != 0
        if StatisticsHelperInst.bStart and StatisticsHelperInst.on_visible is not None:
            StatisticsHelperInst.on_visible(b_visible)
        _, depth_sorted_index = view_depth.sort(dim=-1, descending=False, stable=True)
        sorted_size = torch.gather(allocate_size, 1, depth_sorted_index)
        prefix_sum = sorted_size.cumsum(1, dtype=torch.int32)
        tile_ids, point_ids = litegs_fused.create_table(ndc, inv_cov2d, opacity, prefix_sum, depth_sorted_index,
                                                        feedback_binning_allocate_size, idx_tensor, H, W, th, tw)
        tile_start_index = litegs_fused.tileRange(tile_ids, tiles_num)
        return tile_start_index, point_ids, b_visible.sum(0)


class GaussiansRasterFunc(torch.autograd.Function):
    """Tile rasteriser (wrapper.py:444-524): returns (img, transmittance|None, depth|None, normal=None,
    last_contributor)."""
    @staticmethod
    def forward(ctx, sorted_pointId, tile_start_index, ndc, cov2d_inv, color, opacities, tiles,
                img_h, img_w, tile_h, tile_w, enable_transmitance=False, enable_depth=False):
        stat = bool(StatisticsHelperInst.bStart)
        img, transmitance, depth, last, packed, frag_count, frag_weight = litegs_fused.rasterize_forward(
            sorted_pointId, tile_start_index, ndc, cov2d_inv, color, opacities, tiles, img_h, img_w, tile_h, tile_w,
            stat, enable_transmitance, enable_depth)
        ctx.save_for_backward(sorted_pointId, tile_start_index, transmitance, last, packed, tiles, frag_count, frag_weight)
        ctx.geom = (int(img_h), int(img_w), int(tile_h), int(tile_w))
        ctx.stat = stat
        ctx.mark_non_differentiable(last)
        if not enable_depth:
            depth = None
        out_T = transmitance if enable_transmitance else None
        return img, out_T, depth, None, last

    @staticmethod
    def backward(ctx, grad_img, grad_T, grad_depth, grad_normal, _):
        sorted_pointId, tile_start_index, transmitance, last, packed, tiles, frag_count, frag_weight = ctx.saved_tensors
        img_h, img_w, tile_h, tile_w = ctx.geom
        # the reference max-normalises the image gradient for its fp16 kernel and undoes it afterwards
        # (wrapper.py:490-494); kept so that the C entry point sees the same contract.
        gmax = grad_img.abs().max().clamp_min(1e-30)
        d_ndc, d_cov, d_color, d_opacity, _, err_sq = litegs_fused.rasterize_backward(
            sorted_pointId, tile_start_index, packed, tiles, transmitance, last, grad_img / gmax,
            None if grad_T is None else grad_T / gmax, grad_depth, gmax.reshape(1), img_h, img_w, tile_h, tile_w, ctx.stat)
        if ctx.stat:
            if StatisticsHelperInst.on_fragment_weight is not None:
                StatisticsHelperInst.on_fragment_weight(frag_weight, frag_count)
            if StatisticsHelperInst.on_fragment_err is not None:
                StatisticsHelperInst.on_fragment_err(d_opacity.unsqueeze(0), err_sq * gmax * gmax, frag_count)
        return None, None, d_ndc, d_cov, d_color, d_opacity, None, None, None, None, None, None, None


class CreateViewProj(torch.autograd.Function):
    """Learnable cameras (wrapper.py:772-791): view_params f32[V,7], recp_tan_half_fov_x f32[1] -> view, proj, viewproj,
    frustumplane.  The Level A operators above return no view-matrix gradient, as the reference's do; the camera gradient
    comes from render.render_view (Level B)."""

    @staticmethod
    def forward(ctx, view_params, proj_params, img_h: int, img_w: int, z_near: float, z_far: float):
        view_matrix, proj_matrix, viewproj_matrix, frustumplane = litegs_fused.create_viewproj_forward(view_params, proj_params, img_h, img_w,
                                                                                                      z_near, z_far)
        ctx.save_for_backward(view_params, proj_params)
        ctx.geom = (img_h, img_w, z_near, z_far)
        ctx.mark_non_differentiable(frustumplane)
        return view_matrix, proj_matrix, viewproj_matrix, frustumplane

    @staticmethod
    def backward(ctx, view_matrix_grad, proj_matrix_grad, viewproj_matrix_grad, frustumplane_grad):
        view_params, proj_params = ctx.saved_tensors
        g_view, g_proj = litegs_fused.create_viewproj_backward(view_matrix_grad, proj_matrix_grad, viewproj_matrix_grad, view_params,
                                                               proj_params, *ctx.geom)
        return g_view, g_proj, None, None, None, None


class CullCompactActivateWithSparseGrad(torch.autograd.Function):
    """Gather visible chunks, activate, SH->RGB; gradients come back chunk-compacted
    (wrapper.py:793-845).  With b_sparse_grad=False they are scattered into dense tensors (the
    reference's dense branch is broken, SURVEY Q9)."""
    @staticmethod
    def forward(ctx, b_sparse_grad, sh_degree, visible_chunkid, visible_chunk_num, view_matrix,
                xyz, scale, rot, sh_0, sh_rest, opacity):
        ctx.meta = (bool(b_sparse_grad), int(sh_degree), xyz.shape[-2], xyz.shape[-1])
        out = litegs_fused.cull_compact_activate(sh_degree, visible_chunkid, visible_chunk_num, view_matrix,
                                                 xyz, scale, rot, sh_0, sh_rest, opacity)
        ctx.save_for_backward(visible_chunkid, visible_chunk_num, view_matrix, xyz, scale, rot, sh_0, sh_rest, opacity)
        return tuple(out)

    @staticmethod
    def backward(ctx, g_pos, g_scale, g_rot, g_color, g_opacity):
        sparse, sh_degree, chunk_num, chunk_size = ctx.meta
        visible_chunkid, visible_chunk_num, view_matrix, xyz, scale, rot, sh_0, sh_rest, opacity = ctx.saved_tensors
        zeros = lambda ref, g: torch.zeros_like(ref) if g is None else g
        A = visible_chunkid.shape[0]
        shape = lambda c: (c, A, chunk_size)
        dev = xyz.device
        g_pos = torch.zeros(shape(4), device=dev) if g_pos is None else g_pos
        g_scale = torch.zeros(shape(3), device=dev) if g_scale is None else g_scale
        g_rot = torch.zeros(shape(4), device=dev) if g_rot is None else g_rot
        g_color = torch.zeros((view_matrix.shape[0], 3, A, chunk_size), device=dev) if g_color is None else g_color
        g_opacity = torch.zeros(shape(1), device=dev) if g_opacity is None else g_opacity
        compact = litegs_fused.activate_backward(sh_degree, visible_chunkid, visible_chunk_num, view_matrix,
                                                 xyz, scale, rot, sh_0, sh_rest, opacity,
                                                 g_pos, g_scale, g_rot, g_color, g_opacity)
        grads = []
        for g in compact:
            full = (*g.shape[:-2], chunk_num, chunk_size)
            ct = CompactedTensor(full, visible_chunkid, g)
            grads.append(ct if sparse else ct.to_dense(int(visible_chunk_num.item())))
        return (None, None, None, None, None, *grads)


def sparse_adam_update(param, grad, exp_avg, exp_avg_sq, visible_index, valid_length, lr, b1, b2, eps):
    """wrapper.py:847-855."""
    if param.shape[0] != 0:
        litegs_fused.adamUpdate(param, grad, exp_avg, exp_avg_sq, visible_index, valid_length, lr, b1, b2, eps)
