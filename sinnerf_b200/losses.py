"""kornia 0.6.3's `inverse_depth_smoothness_loss` and `ssim_loss` with kornia's signatures, executed by
libsinnerf_b200's sm_90a kernels (csrc/patch_loss.cu) forward and backward.

The reference training step puts them on (B,C,H,W) patches of render_rays' outputs (models/sinnerf.py:370-373,
:395-398; losses.py:105 under --patch_loss l2_ssim).  A SinNeRF maintainer swaps two imports:

    from sinnerf_b200.losses import inverse_depth_smoothness_loss   # models/sinnerf.py:23
    from sinnerf_b200.losses import ssim_loss                       # losses.py:2

Inputs are read through their strides, so the '(b p q) c -> b c p q' views of the ray-major outputs are not copied,
and gradients come back with the inputs' strides (autograd's backward of the rearrange is then a view).  Both losses
compute in fp32 (SSIM's window sums in fp64) whatever the autocast state; kornia's conv2d would run in half precision
under fp16 autocast.  fp32 CUDA tensors only: there is no CPU path.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .rendering import _loss_workspace

__all__ = ["inverse_depth_smoothness_loss", "ssim_loss"]


def _strides(t: torch.Tensor):
    return (C.c_int64 * 4)(*t.stride())


def _check_shape(t, name: str, what: str) -> None:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what}: {name} is not a torch.Tensor (got {type(t)})")
    if t.dim() != 4:
        raise ValueError(f"{what}: invalid {name} shape, we expect BxCxHxW. Got: {tuple(t.shape)}")


def _check_storage(t, name: str, what: str) -> None:
    _lib.require_device(t, what)
    if t.dtype != torch.float32:
        raise TypeError(f"{what}: {name} must be float32 (got {t.dtype})")


class _DepthSmooth(torch.autograd.Function):
    @staticmethod
    def forward(ctx, idepth, image):
        lib = _lib.load()
        B, Cc, H, W = image.shape
        loss = torch.empty((), device=image.device, dtype=torch.float32)
        st = _lib.stream_ptr(image.device)
        _lib.check(lib.snb_depth_smooth_forward(_lib.ptr(idepth), _strides(idepth), _lib.ptr(image), _strides(image),
                                                B, Cc, H, W, _lib.ptr(loss), _lib.ptr(_loss_workspace(image.device)), st),
                   "snb_depth_smooth_forward")
        ctx.save_for_backward(idepth, image)
        return loss

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        idepth, image = ctx.saved_tensors
        B, Cc, H, W = image.shape
        g = g.detach().to(torch.float32).contiguous()
        # empty_like keeps the input's strides (a permuted view stays permuted) whenever they are non-overlapping
        g_d = torch.empty_like(idepth) if ctx.needs_input_grad[0] else None
        g_i = torch.empty_like(image) if ctx.needs_input_grad[1] else None
        _lib.check(lib.snb_depth_smooth_backward(
            _lib.ptr(idepth), _strides(idepth), _lib.ptr(image), _strides(image), B, Cc, H, W, _lib.ptr(g),
            _lib.ptr(g_d), None if g_d is None else _strides(g_d), _lib.ptr(g_i), None if g_i is None else _strides(g_i),
            _lib.stream_ptr(image.device)), "snb_depth_smooth_backward")
        return g_d, g_i


def inverse_depth_smoothness_loss(idepth: torch.Tensor, image: torch.Tensor) -> torch.Tensor:
    """kornia.losses.inverse_depth_smoothness_loss (0.6.3): idepth (B,1,H,W), image (B,C,H,W) ->
    mean |dx(idepth) exp(-mean_c |dx(image)|)| + mean |dy(idepth) exp(-mean_c |dy(image)|)|, a 0-d tensor.
    Differentiable in both inputs.  kornia's shape errors are ValueError; an idepth with more than one channel
    (which kornia would broadcast and the reference never passes) is NotImplementedError; H or W below 2 (where
    kornia returns the NaN of an empty mean) is ValueError."""
    what = "inverse_depth_smoothness_loss"
    _check_shape(idepth, "idepth", what)
    _check_shape(image, "image", what)
    if idepth.shape[-2:] != image.shape[-2:]:
        raise ValueError(f"{what}: idepth and image shapes must be the same. Got: {tuple(idepth.shape)} and "
                         f"{tuple(image.shape)}")
    if idepth.device != image.device:
        raise ValueError(f"{what}: idepth and image must be in the same device. Got: {idepth.device} and {image.device}")
    if idepth.shape[0] != image.shape[0]:
        raise ValueError(f"{what}: idepth and image batch sizes differ: {idepth.shape[0]} and {image.shape[0]}")
    if idepth.shape[1] != 1:
        raise NotImplementedError(f"{what}: idepth must have one channel (got {idepth.shape[1]})")
    if min(image.shape[-2:]) < 2:
        raise ValueError(f"{what}: needs H, W >= 2 (got {tuple(image.shape[-2:])})")
    _check_storage(idepth, "idepth", what)
    _check_storage(image, "image", what)
    return _DepthSmooth.apply(idepth, image)


class _Ssim(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, max_val, eps):
        lib = _lib.load()
        B, Cc, H, W = img1.shape
        dev = img1.device
        loss = torch.empty((), device=dev, dtype=torch.float32)
        # per-pixel coefficient maps of the backward (dL/dmu1, dL/df(x^2), dL/df(xy)), fp64
        coef = torch.empty(3 * img1.numel(), device=dev, dtype=torch.float64) if ctx.needs_input_grad[0] else None
        _lib.check(lib.snb_ssim_loss_forward(_lib.ptr(img1), _strides(img1), _lib.ptr(img2), _strides(img2), B, Cc, H, W,
                                             11, max_val, eps, _lib.ptr(loss), _lib.ptr(coef),
                                             _lib.ptr(_loss_workspace(dev)), _lib.stream_ptr(dev)),
                   "snb_ssim_loss_forward")
        if coef is not None:
            ctx.save_for_backward(img1, img2, coef)
        return loss

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        img1, img2, coef = ctx.saved_tensors
        B, Cc, H, W = img1.shape
        g = g.detach().to(torch.float32).contiguous()
        g1 = torch.empty_like(img1)
        _lib.check(lib.snb_ssim_loss_backward(_lib.ptr(img1), _strides(img1), _lib.ptr(img2), _strides(img2), B, Cc, H,
                                              W, _lib.ptr(coef), _lib.ptr(g), _lib.ptr(g1), _strides(g1),
                                              _lib.stream_ptr(img1.device)), "snb_ssim_loss_backward")
        return g1, None, None, None


def ssim_loss(img1: torch.Tensor, img2: torch.Tensor, window_size: int, max_val: float = 1.0, eps: float = 1e-12,
              reduction: str = "mean") -> torch.Tensor:
    """kornia.losses.ssim_loss (0.6.3): mean clamp((1 - SSIM(img1, img2)) / 2, 0, 1) with an 11x11 Gaussian window
    (sigma 1.5) over reflect-padded (B,C,H,W) images, a 0-d tensor.  Built for what the reference uses:
    window_size 11, reduction 'mean', gradients into img1 only (the reference's img2 is a target); other values, or
    an img2 that requires grad, raise NotImplementedError.  H, W >= 6 (reflect padding needs pad < size)."""
    what = "ssim_loss"
    _check_shape(img1, "img1", what)
    _check_shape(img2, "img2", what)
    if img1.shape != img2.shape:
        raise ValueError(f"{what}: img1 and img2 shapes must be the same. Got: {tuple(img1.shape)} and "
                         f"{tuple(img2.shape)}")
    if img1.device != img2.device:
        raise ValueError(f"{what}: img1 and img2 must be in the same device. Got: {img1.device} and {img2.device}")
    if window_size != 11:
        raise NotImplementedError(f"{what}: only window_size=11 is built (got {window_size})")
    if reduction != "mean":
        raise NotImplementedError(f"{what}: only reduction='mean' is built (got {reduction!r})")
    if img2.requires_grad:
        raise NotImplementedError(f"{what}: no gradient into img2 (the target); pass img2.detach()")
    if min(img1.shape[-2:]) < 6:
        raise ValueError(f"{what}: needs H, W >= 6 for reflect padding of 5 (got {tuple(img1.shape[-2:])})")
    _check_storage(img1, "img1", what)
    _check_storage(img2, "img2", what)
    return _Ssim.apply(img1, img2, float(max_val), float(eps))
