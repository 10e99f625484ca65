"""Depth-normal consistency (2DGS, PGSR, RaDe-GS) on the fused path's depth, transmittance and normal images, on the kernel of
csrc/geometry.cu (DESIGN.md section 1, "Depth-normal consistency").

    depth_normal(depth, trans, proj, alpha_min=0.5)                          -> (n_d [1,3,H,W], mask [1,1,H,W] bool)
    depth_normal_loss_and_grad(depth, trans, normal, proj, weight, upstream=1.0, alpha_min=0.5)
                                                                             -> (loss f32[], d_depth, d_trans, d_normal)
    depth_normal_loss(depth, trans, normal, proj, weight, alpha_min=0.5)     -> loss f32[] (autograd)

depth, trans: the depth mode's D and the transmittance T, f32[1,1,H,W]; normal: the normal mode's N, f32[1,3,H,W]; proj: the
view's projection matrix f32[4,4] or [1,4,4] on the device.  The [..., :H, :W] views render_views hands its callbacks are read in
place.  The loss is weight * mean over all H W pixels of 1 - n_d . N / |N| where n_d and N are defined; n_d is the normal of
the surface the expected depth ED = D / (1 - T) unprojects to.  CUDA float32 only; there is no CPU path.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from .fused import _on, _ptr, _stream


def _plane(t: torch.Tensor, name: str, channels: int, hw=None) -> torch.Tensor:
    if t is None:
        raise RuntimeError(f"depth_normal (litegs_b200): {name} is None")
    if not t.is_cuda or t.dtype != torch.float32:
        raise RuntimeError(f"depth_normal (litegs_b200): {name} must be a float32 CUDA tensor, got {t.dtype} on {t.device}")
    if t.dim() != 4 or t.shape[0] != 1 or t.shape[1] != channels or (hw is not None and tuple(t.shape[-2:]) != hw):
        want = f"[1,{channels},{hw[0]},{hw[1]}]" if hw is not None else f"[1,{channels},H,W]"
        raise RuntimeError(f"depth_normal (litegs_b200): {name} must be {want}, got {list(t.shape)}")
    return t if t.stride(-1) == 1 else t.contiguous()


def _proj(proj: torch.Tensor, dev) -> torch.Tensor:
    if not (isinstance(proj, torch.Tensor) and proj.is_cuda and proj.dtype == torch.float32 and proj.numel() == 16
            and proj.shape[-2:] == (4, 4)):
        raise RuntimeError("depth_normal (litegs_b200): proj must be a float32 CUDA tensor of shape [4,4] or [1,4,4]")
    if proj.device != dev:
        raise RuntimeError(f"depth_normal (litegs_b200): proj is on {proj.device}, the images on {dev}")
    return proj.contiguous()


def _run(depth, trans, normal, proj, alpha_min, want_map=False, want_loss=False, grad_scale=None):
    """One launch of lgs_depth_normal -> (n_d or None, block sums or None, (d_depth, d_trans, d_normal) or None)."""
    D = _plane(depth, "depth", 1)
    H, W = D.shape[-2:]
    T = _plane(trans, "trans", 1, (H, W))
    N = None if normal is None else _plane(normal, "normal", 3, (H, W))
    dev = D.device
    if T.device != dev or (N is not None and N.device != dev):
        raise RuntimeError("depth_normal (litegs_b200): depth, trans and normal must be on one device")
    P = _proj(proj, dev)
    if not 0.0 <= float(alpha_min) < 1.0:
        raise RuntimeError(f"depth_normal (litegs_b200): alpha_min = {alpha_min} outside [0, 1)")
    with _on(dev):
        nd = torch.empty((1, 3, H, W), dtype=torch.float32, device=dev) if want_map else None
        sums = grads = None
        if want_loss:
            n = ctypes.c_int(0)
            _lib.call("lgs_depth_normal_num_block_sums", H, W, ctypes.byref(n))
            sums = torch.empty(n.value, dtype=torch.float32, device=dev)
        if grad_scale is not None:
            grads = (torch.empty((1, 1, H, W), dtype=torch.float32, device=dev), torch.empty((1, 1, H, W), dtype=torch.float32, device=dev),
                     torch.empty((1, 3, H, W), dtype=torch.float32, device=dev))
        ns, ncs = (N.stride(-2), N.stride(1)) if N is not None else (W, H * W)
        _lib.call("lgs_depth_normal", _ptr(D), D.stride(-2), _ptr(T), T.stride(-2), _ptr(N), ns, ncs, _ptr(P), H, W, float(alpha_min),
                  float(grad_scale or 0.0), _ptr(nd), *(_ptr(g) for g in (grads or (None,) * 3)), _ptr(sums), _stream(dev))
    return nd, sums, grads


def _loss(sums, weight, H, W):
    # fixed-order reduction of the per-CTA partials: deterministic
    return sums.sum(dtype=torch.float64).mul_(float(weight) / (H * W)).to(torch.float32)


def depth_normal(depth, trans, proj, alpha_min: float = 0.5):
    """The normal of the unprojected expected depth -> (n_d f32[1,3,H,W], mask bool[1,1,H,W]); n_d is a unit vector where mask
    holds and zero elsewhere (border pixels, alpha <= alpha_min at the pixel or a neighbour, a degenerate cross product)."""
    nd, _, _ = _run(depth, trans, None, proj, alpha_min, want_map=True)
    return nd, (nd != 0).any(dim=1, keepdim=True)


def depth_normal_loss_and_grad(depth, trans, normal, proj, weight: float, upstream: float = 1.0, alpha_min: float = 0.5):
    """L = weight * mean_p (1 - n_d . N_p / |N_p|) over all H W pixels (terms where n_d or N is undefined count as zero) and
    upstream * dL/d(depth, trans, normal), in one kernel without autograd: the form for render_views(loss_and_grad_fn=...).
    Returns (loss f32[] on the device, d_depth f32[1,1,H,W], d_trans f32[1,1,H,W], d_normal f32[1,3,H,W])."""
    H, W = depth.shape[-2:]
    _, sums, grads = _run(depth, trans, normal, proj, alpha_min, want_loss=True, grad_scale=float(weight) * float(upstream) / (H * W))
    return (_loss(sums, weight, H, W), *grads)


class _LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, trans, normal, proj, weight, alpha_min):
        H, W = depth.shape[-2:]
        want_grad = any(ctx.needs_input_grad[:3])
        _, sums, grads = _run(depth, trans, normal, proj, alpha_min, want_loss=True,
                              grad_scale=float(weight) / (H * W) if want_grad else None)
        if want_grad:
            ctx.save_for_backward(*grads)
        return _loss(sums, weight, H, W)

    @staticmethod
    def backward(ctx, g):
        dD, dT, dN = ctx.saved_tensors
        return dD * g, dT * g, dN * g, None, None, None


def depth_normal_loss(depth, trans, normal, proj, weight: float, alpha_min: float = 0.5):
    """depth_normal_loss_and_grad's L as a differentiable scalar, for render_view users and render_views(loss_fn=...); the
    gradient is computed with the loss, by the same kernel, and scaled by the incoming gradient in the backward."""
    for t, name, flag in ((depth, "depth", "pp.render_depth"), (trans, "trans", "pp.enable_transmitance"),
                          (normal, "normal", "pp.render_normal")):
        if t is None:
            raise RuntimeError(f"depth_normal_loss: {name} is None; render with {flag} = True")
    return _LossFn.apply(depth, trans, normal, proj, weight, alpha_min)
