"""Host mirror of the reference's ``fused_ssim`` package (fused_ssim/fused_ssim/__init__.py:1-90 above the pybind module
fused_ssim/ext.cpp:4-9) on the kernels of csrc/ssim.cu.

Same names, argument order and semantics:

    fusedssim(C1, C2, img1, img2, train)                       -> (ssim_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)
    fusedssim_backward(C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12) -> dL_dimg1
    fusedl1ssim_loss(ssim_weight, C1, C2, img1, img2, train)   -> (loss_map, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)
    fusedl1ssim_loss_backward(ssim_weight, C1, C2, img1, img2, dL_dmap, ...) -> dL_dimg1
    FusedSSIMMap / FusedL1SSIMLossMap (autograd), fused_ssim(img1, img2, padding, train), fused_l1_ssim_loss(...)

plus one entry the reference does not have, for the training loop: ``l1_ssim_loss_and_grad`` computes the scalar loss
and dL/dimg1 in two kernels without materialising the loss map (the mean only needs per-CTA partial sums) and without
an autograd round trip.  CUDA float32 only; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from .fused import _on, _ptr, _stream

allowed_padding = ["same", "valid"]


def _check(img1: torch.Tensor, img2: torch.Tensor):
    if not (img1.is_cuda and img2.is_cuda):
        raise RuntimeError("fused_ssim (litegs_b200) only supports CUDA tensors")
    if img1.dtype != torch.float32 or img2.dtype != torch.float32:
        raise RuntimeError("fused_ssim (litegs_b200): float32 images expected")
    if img1.dim() != 4 or img1.shape != img2.shape:
        raise RuntimeError(f"fused_ssim (litegs_b200): two [B,CH,H,W] images of one shape expected, got {tuple(img1.shape)} "
                           f"and {tuple(img2.shape)}")
    return img1.contiguous(), img2.contiguous()


def _forward(l1_mode: int, ssim_weight: float, C1: float, C2: float, img1, img2, train: bool, want_map=True, want_sums=False):
    a, b = _check(img1, img2)
    B, CH, H, W = a.shape
    dev = a.device
    with _on(dev):
        out = torch.empty_like(a) if want_map else None
        if train:
            d0, d1, d2 = torch.empty_like(a), torch.empty_like(a), torch.empty_like(a)
        else:
            d0 = d1 = d2 = None
        sums = None
        if want_sums:
            n = ctypes.c_int(0)
            _lib.call("lgs_ssim_num_block_sums", B, CH, H, W, ctypes.byref(n))
            sums = torch.empty(n.value, dtype=torch.float32, device=dev)
        _lib.call("lgs_ssim_forward", _ptr(a), _ptr(b), B, CH, H, W, float(C1), float(C2), int(l1_mode), float(ssim_weight), _ptr(out),
                  _ptr(d0), _ptr(d1), _ptr(d2), _ptr(sums), _stream(dev))
    if not train:
        e = torch.empty((0,), dtype=a.dtype, device=dev)
        d0 = d1 = d2 = e
    return out, d0, d1, d2, sums


def _backward(l1_mode: int, ssim_weight: float, img1, img2, dL_dmap, uniform_chain: float, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    a, b = _check(img1, img2)
    B, CH, H, W = a.shape
    dev = a.device
    with _on(dev):
        if dL_dmap is not None:
            if dL_dmap.shape != a.shape or not dL_dmap.is_cuda or dL_dmap.dtype != torch.float32:
                raise RuntimeError("fused_ssim (litegs_b200): dL_dmap must be a float32 CUDA tensor shaped like the images")
            dL_dmap = dL_dmap.contiguous()
        g = torch.empty_like(a)
        _lib.call("lgs_ssim_backward", _ptr(a), _ptr(b), _ptr(dL_dmap), float(uniform_chain), _ptr(dm_dmu1.contiguous()),
                  _ptr(dm_dsigma1_sq.contiguous()), _ptr(dm_dsigma12.contiguous()), B, CH, H, W, int(l1_mode), float(ssim_weight), _ptr(g),
                  _stream(dev))
    return g


# ---- the four functions of the reference's pybind module (fused_ssim/ext.cpp:4-9) ------------------------------------

def fusedssim(C1, C2, img1, img2, train=True):
    return _forward(0, 0.0, C1, C2, img1, img2, bool(train))[:4]


def fusedssim_backward(C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    return _backward(0, 0.0, img1, img2, dL_dmap, 0.0, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)


def fusedl1ssim_loss(ssim_weight, C1, C2, img1, img2, train=True):
    return _forward(1, ssim_weight, C1, C2, img1, img2, bool(train))[:4]


def fusedl1ssim_loss_backward(ssim_weight, C1, C2, img1, img2, dL_dmap, dm_dmu1, dm_dsigma1_sq, dm_dsigma12):
    return _backward(1, ssim_weight, img1, img2, dL_dmap, 0.0, dm_dmu1, dm_dsigma1_sq, dm_dsigma12)


# ---- the Python layer of the reference package (fused_ssim/fused_ssim/__init__.py:16-90) -----------------------------
# One autograd node serves both maps; the two public Function classes only fix the mode and the reference's argument order.

def _crop(t, padding):
    return t[:, :, 5:-5, 5:-5] if padding == "valid" else t


class _MapFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, l1_mode, ssim_weight, C1, C2, img1, img2, padding, train):
        out, d0, d1, d2, _ = _forward(l1_mode, ssim_weight, C1, C2, img1, img2, bool(train))
        ctx.save_for_backward(img1.detach(), img2, d0, d1, d2)
        ctx.cfg = (l1_mode, ssim_weight, padding)
        return _crop(out, padding)

    @staticmethod
    def backward(ctx, g_map):
        img1, img2, d0, d1, d2 = ctx.saved_tensors
        l1_mode, ssim_weight, padding = ctx.cfg
        if padding == "valid":                      # gradient of the crop: zero border (reference __init__.py:34-37)
            full = torch.zeros_like(img1)
            full[:, :, 5:-5, 5:-5] = g_map
            g_map = full
        g = _backward(l1_mode, ssim_weight, img1, img2, g_map, 0.0, d0, d1, d2)
        return None, None, None, None, g, None, None, None


class FusedSSIMMap:
    """FusedSSIMMap.apply(C1, C2, img1, img2, padding="same", train=True) -> SSIM map (reference __init__.py:16-42)."""

    @staticmethod
    def apply(C1, C2, img1, img2, padding="same", train=True):
        return _MapFn.apply(0, 0.0, C1, C2, img1, img2, padding, train)


class FusedL1SSIMLossMap:
    """FusedL1SSIMLossMap.apply(ssim_weight, C1, C2, img1, img2, padding="same", train=True) -> loss map (:53-80)."""

    @staticmethod
    def apply(ssim_weight, C1, C2, img1, img2, padding="same", train=True):
        return _MapFn.apply(1, ssim_weight, C1, C2, img1, img2, padding, train)


def _consts():
    return 0.01 ** 2, 0.03 ** 2


def fused_ssim(img1, img2, padding="same", train=True):
    """Mean SSIM (reference __init__.py:44-51)."""
    if padding not in allowed_padding:
        raise AssertionError(f"padding must be one of {allowed_padding}")
    C1, C2 = _consts()
    return FusedSSIMMap.apply(C1, C2, img1.contiguous(), img2, padding, train).mean()


def fused_l1_ssim_loss(img1, img2, ssim_weight=0.2, padding="same", train=True):
    """mean(w (1 - SSIM) + (1 - w) |img1 - img2|) (reference __init__.py:82-90; what trainer.py:145 calls)."""
    if padding not in allowed_padding:
        raise AssertionError(f"padding must be one of {allowed_padding}")
    C1, C2 = _consts()
    return FusedL1SSIMLossMap.apply(ssim_weight, C1, C2, img1, img2, padding, train).mean()


# ---- fused training entry (ours) ----------------------------------------------------------------------------------------

def l1_ssim_loss_and_grad(img1, img2, ssim_weight=0.2, upstream: float = 1.0):
    """loss = mean(w (1 - SSIM) + (1 - w) |img1 - img2|) over all B*CH*H*W elements (= fused_l1_ssim_loss(img1, img2, w),
    padding "same") and upstream * dloss/dimg1, in two kernels: no loss map, no autograd graph.  Returns
    (loss f32[] on the device, dL_dimg1 f32[B,CH,H,W])."""
    C1, C2 = _consts()
    _, d0, d1, d2, sums = _forward(1, ssim_weight, C1, C2, img1, img2, True, want_map=False, want_sums=True)
    n = img1.numel()
    loss = sums.sum(dtype=torch.float64).div_(n).to(torch.float32)      # fixed-order reduction of ~1e3 partials: deterministic
    grad = _backward(1, ssim_weight, img1, img2, None, float(upstream) / n, d0, d1, d2)
    return loss, grad
