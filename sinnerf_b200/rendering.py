"""`render_rays`, `sample_pdf`, `eval_points` with the reference's signatures
(reference models/rendering.py:15-61, :64-123, :126-335), executed by libsinnerf_b200's
sm_90a kernels through the C ABI in include/sinnerf_b200.h.

Host side only: argument checks, output allocation from PyTorch's caching allocator, the
reference's random draws (same shapes, same order, same torch generator, so a seeded run
consumes the RNG exactly like the reference on that device), and one `snb_render_forward`
call that enqueues every stage on the current CUDA stream.  No stage has a PyTorch or CPU
fallback.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Dict, List, Optional, Sequence, Union

import torch

from . import _lib
from . import config
from .nerf import NeRF

__all__ = ["render_rays", "render_rays_multi", "sample_pdf", "eval_points", "RayLosses"]

# The reference draws `randn` for the sigma noise even when noise_std == 0
# (models/rendering.py:224).  Keep the draw (generator state parity) unless disabled.
DRAW_UNUSED_NOISE = True

_linspace_cache: Dict[tuple, torch.Tensor] = {}


def _linspace01(n: int, device) -> torch.Tensor:
    """torch.linspace(0, 1, n) in the default dtype (rendering.py:264-265 / :40), cached per
    device.  Computed on the host so the values equal the CPU reference's bit for bit."""
    key = (n, str(device))
    t = _linspace_cache.get(key)
    if t is None:
        t = torch.linspace(0, 1, n, dtype=torch.float32).to(device)
        _linspace_cache[key] = t
    return t


# --------------------------------------------------------------------------- training path
@dataclasses.dataclass
class RayLosses:
    """Losses SinNeRF puts directly on render_rays' outputs (reference models/sinnerf.py:310-319), evaluated
    inside the compositing kernels (SURVEY 8f-3) for the coarse AND the fine pass:
      rgb term   = sum_ray rgb_weight   * |rgb - target_rgb|^2       (MSELoss, losses.py:12-22)
      depth term = sum_ray depth_weight * smooth_l1(depth - target_depth)   (SL1Loss, models/sinnerf.py:32-42)
    Weights: None -> 'mean' normalisation (1/(3N) and 1/N, what nn.MSELoss / nn.SmoothL1Loss compute), a float,
    or an (N,) tensor of per-ray weights (0 = this ray has no target)."""
    target_rgb: Optional[torch.Tensor] = None
    target_depth: Optional[torch.Tensor] = None
    rgb_weight: Union[None, float, torch.Tensor] = None
    depth_weight: Union[None, float, torch.Tensor] = None

    def resolved(self, n: int, dev):
        """-> (target_rgb, target_depth, rgb_weight tensor|None, depth_weight tensor|None, wr0, wd0), fp32 on dev."""
        def tens(x, shape, what):
            if x is None:
                return None
            x = x.detach().to(dev, torch.float32).reshape(shape).contiguous()
            return x
        trgb = tens(self.target_rgb, (n, 3), "target_rgb")
        tdep = tens(self.target_depth, (n,), "target_depth")
        if trgb is None and tdep is None:
            raise ValueError("RayLosses: give target_rgb and/or target_depth")
        wr = wd = None
        wr0, wd0 = 1.0 / (3 * max(n, 1)), 1.0 / max(n, 1)
        if isinstance(self.rgb_weight, torch.Tensor):
            wr = tens(self.rgb_weight, (n,), "rgb_weight")
        elif self.rgb_weight is not None:
            wr0 = float(self.rgb_weight)
        if isinstance(self.depth_weight, torch.Tensor):
            wd = tens(self.depth_weight, (n,), "depth_weight")
        elif self.depth_weight is not None:
            wd0 = float(self.depth_weight)
        return trgb, tdep, wr, wd, wr0, wd0


_loss_ws: Dict[str, torch.Tensor] = {}


def _loss_workspace(dev) -> torch.Tensor:
    ws = _loss_ws.get(str(dev))
    if ws is None:
        ws = torch.zeros(_lib.LOSS_WS_FLOATS, device=dev, dtype=torch.float32)
        _loss_ws[str(dev)] = ws
    return ws


def _loss_struct(spec):
    if spec is None:
        return None
    trgb, tdep, wr, wd, wr0, wd0 = spec
    ls = _lib.SnbLossSpec()
    ls.target_rgb, ls.target_depth = _lib.ptr(trgb), _lib.ptr(tdep)
    ls.rgb_weight, ls.depth_weight = _lib.ptr(wr), _lib.ptr(wd)
    ls.rgb_weight0, ls.depth_weight0 = wr0, wd0
    return ls


class _RenderPass(torch.autograd.Function):
    """(rgb, depth, weights, loss) = composite(field(rays, z; params)) for one pass (coarse or fine).

    Forward: snb_field_forward_train (keeps the activations) + snb_composite_forward[_loss].
    Backward: snb_composite_backward_loss (closed form; the fused loss terms' derivatives are formed per ray
    in registers, no g_rgb / g_depth tensors) + snb_field_backward.  Differentiable in the 24 parameter
    tensors only -- the reference propagates nothing into rays / z either (rendering.py:311-313).
    `loss` is a (2,) tensor [rgb term, depth term] (zeros without a loss spec)."""

    @staticmethod
    def forward(ctx, model: "NeRF", prec: int, rays, z, noise, noise_std, white_back, spec, *params):
        lib = _lib.load()
        dev = rays.device
        n, S = z.shape
        P = n * S
        img = model.packed_weights(prec)
        raw = torch.empty(n, S, 4, device=dev, dtype=torch.float32)
        store16 = prec != _lib.PRECISIONS["fp32"] and config.get_train_storage() == "fp16"
        if store16:
            # one fp16 copy of everything the backward streams, in the MMA-ready tile layout (csrc/act16.cuh)
            act16 = torch.empty(lib.snb_act16_bytes(P), device=dev, dtype=torch.uint8)
            save_enc = save_dir = save_h = save_g = raw.new_empty(0)
        else:
            act16 = raw.new_empty(0)
            save_enc = torch.empty(P, 64, device=dev, dtype=torch.float32)
            save_dir = torch.empty(P, 32, device=dev, dtype=torch.float32)
            save_h = torch.empty(8, P, 256, device=dev, dtype=torch.float32)
            save_g = torch.empty(P, 128, device=dev, dtype=torch.float32)
        rgb = torch.empty(n, 3, device=dev, dtype=torch.float32)
        depth = torch.empty(n, device=dev, dtype=torch.float32)
        w = torch.empty(n, S, device=dev, dtype=torch.float32)
        loss = torch.zeros(2, device=dev, dtype=torch.float32) if spec is None else torch.empty(2, device=dev)
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            if store16:
                _lib.check(lib.snb_field_forward_train16(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S,
                                                         _lib.ptr(raw), _lib.ptr(act16), st), "snb_field_forward_train16")
            else:
                _lib.check(lib.snb_field_forward_train(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, _lib.ptr(raw),
                                                       _lib.ptr(save_enc), _lib.ptr(save_dir), _lib.ptr(save_h),
                                                       _lib.ptr(save_g), st), "snb_field_forward_train")
            if spec is None:
                _lib.check(lib.snb_composite_forward(_lib.ptr(raw), 4, _lib.ptr(z), _lib.ptr(rays), _lib.ptr(noise),
                                                     noise_std, int(white_back), n, S, _lib.ptr(rgb), _lib.ptr(depth),
                                                     _lib.ptr(w), st), "snb_composite_forward")
            else:
                ls = _loss_struct(spec)
                _lib.check(lib.snb_composite_forward_loss(_lib.ptr(raw), _lib.ptr(z), _lib.ptr(rays), _lib.ptr(noise),
                                                          noise_std, int(white_back), n, S, C.byref(ls), _lib.ptr(rgb),
                                                          _lib.ptr(depth), _lib.ptr(w), _lib.ptr(loss),
                                                          _lib.ptr(_loss_workspace(dev)), st), "snb_composite_forward_loss")
        ctx.save_for_backward(raw, z, rays, noise if noise is not None else raw.new_empty(0), rgb, depth,
                              save_enc, save_dir, save_h, save_g, act16, *params)
        ctx.cfg = (float(noise_std), int(white_back), noise is not None, int(model.use_new_activation), store16)
        ctx.spec = spec          # plain (non-differentiable) tensors + floats
        if spec is None:
            ctx.mark_non_differentiable(loss)
        return rgb, depth, w, loss

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_w, g_loss):
        lib = _lib.load()
        raw, z, rays, noise, rgb, depth, save_enc, save_dir, save_h, save_g, act16, *params = ctx.saved_tensors
        noise_std, white_back, has_noise, new_activation, store16 = ctx.cfg
        dev = raw.device
        n, S = z.shape
        P = n * S
        g_raw = torch.empty_like(raw)
        keep = [t.contiguous().to(torch.float32) if t is not None else None for t in (g_rgb, g_depth, g_w)]
        ls = _loss_struct(ctx.spec)
        gl = g_loss.contiguous().to(torch.float32) if (ls is not None and g_loss is not None) else None
        if ls is not None and g_loss is None:
            ls = None            # the loss output was not used: only the explicit gradients flow
        ps = [p.detach().contiguous() for p in params]
        # one zero-filled buffer for all 24 gradient tensors (the kernels accumulate into them); every view
        # starts on a 16-byte boundary
        offs, total = [], 0
        for p in ps:
            offs.append(total)
            total += (p.numel() + 3) // 4 * 4
        flat = torch.zeros(total, device=dev, dtype=torch.float32)
        grads = [flat[o:o + p.numel()].view_as(p) for o, p in zip(offs, ps)]
        parr = (C.c_void_p * 24)(*[p.data_ptr() for p in ps])
        garr = (C.c_void_p * 24)(*[g.data_ptr() for g in grads])
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            g_amax = torch.zeros(1, device=dev, dtype=torch.float32) if store16 else None     # bit pattern of max |g_raw|
            _lib.check(lib.snb_composite_backward_loss(_lib.ptr(raw), _lib.ptr(z), _lib.ptr(rays),
                                                       _lib.ptr(noise) if has_noise else None, noise_std, white_back,
                                                       _lib.ptr(keep[0]), _lib.ptr(keep[1]), _lib.ptr(keep[2]),
                                                       C.byref(ls) if ls is not None else None, _lib.ptr(rgb),
                                                       _lib.ptr(depth), _lib.ptr(gl), n, S, _lib.ptr(g_raw), _lib.ptr(g_amax), st),
                       "snb_composite_backward_loss")
            if store16:
                ws = torch.empty(lib.snb_bwd16_workspace_bytes(P), device=dev, dtype=torch.uint8)
                _lib.check(lib.snb_field_backward16(parr, garr, new_activation, _lib.ptr(g_raw), _lib.ptr(raw), _lib.ptr(act16),
                                                    P, _lib.ptr(ws), _lib.ptr(g_amax), st), "snb_field_backward16")
            else:
                ws_a = torch.empty(P, 256, device=dev, dtype=torch.float32)
                ws_b = torch.empty(P, 256, device=dev, dtype=torch.float32)
                ws_s = torch.empty(P, 128, device=dev, dtype=torch.float32)
                ws_w = torch.empty(_lib.BWD_WS_FLOATS, device=dev, dtype=torch.float32)
                ws_m = torch.empty(P, 8, device=dev, dtype=torch.int32)
                _lib.check(lib.snb_field_backward(parr, garr, new_activation, _lib.ptr(g_raw), _lib.ptr(raw),
                                                  _lib.ptr(save_enc), _lib.ptr(save_dir), _lib.ptr(save_h),
                                                  _lib.ptr(save_g), P, _lib.ptr(ws_a), _lib.ptr(ws_b), _lib.ptr(ws_s),
                                                  _lib.ptr(ws_w), _lib.ptr(ws_m), st), "snb_field_backward")
        return (None, None, None, None, None, None, None, None, *grads)


# the parameter tensors a sigma-only pass reads: xyz_encoding_1..8 and sigma (state-dict indices 0-15, 20, 21)
_SIGMA_PASS_TENSORS = tuple(range(16)) + (20, 21)


class _SigmaPass(torch.autograd.Function):
    """One sigma-only field pass: layers 1-8 and the sigma head (models/nerf.py:105-136 with sigma_only=True), and with
    `composite` the weights-only compositing after it (models/rendering.py:215-238 with weights_only=True).

    composite=True returns the weights (N,S): render_rays(test_time=True)'s coarse pass (rendering.py:287-292).
    composite=False returns sigma (N,S): eval_points (rendering.py:64-123), whose points are staged as rays.
    Forward: snb_field_forward_train[16]_sigma (+ snb_composite_forward with raw_channels = 1).  Backward:
    (snb_composite_backward_weights +) snb_field_backward[16]_sigma.  Differentiable in the parameter tensors only;
    xyz_encoding_final, dir_encoding and rgb, which the pass never reads, get None, as autograd through the reference
    leaves them."""

    @staticmethod
    def forward(ctx, model: "NeRF", prec: int, rays, z, noise, noise_std, composite, *params):
        lib = _lib.load()
        dev = rays.device
        n, S = z.shape
        P = n * S
        img = model.packed_weights(prec)
        sigma = torch.empty(n, S, device=dev, dtype=torch.float32)
        store16 = prec != _lib.PRECISIONS["fp32"] and config.get_train_storage() == "fp16"
        if store16:
            act16 = torch.empty(lib.snb_act16_bytes(P), device=dev, dtype=torch.uint8)
            save_enc = save_h = sigma.new_empty(0)
        else:
            act16 = sigma.new_empty(0)
            save_enc = torch.empty(P, 64, device=dev, dtype=torch.float32)
            save_h = torch.empty(8, P, 256, device=dev, dtype=torch.float32)
        w = torch.empty(n, S, device=dev, dtype=torch.float32) if composite else None
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            if store16:
                _lib.check(lib.snb_field_forward_train16_sigma(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S,
                                                               _lib.ptr(sigma), _lib.ptr(act16), st),
                           "snb_field_forward_train16_sigma")
            else:
                _lib.check(lib.snb_field_forward_train_sigma(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S,
                                                             _lib.ptr(sigma), _lib.ptr(save_enc), _lib.ptr(save_h), st),
                           "snb_field_forward_train_sigma")
            if composite:
                _lib.check(lib.snb_composite_forward(_lib.ptr(sigma), 1, _lib.ptr(z), _lib.ptr(rays), _lib.ptr(noise),
                                                     noise_std, 0, n, S, None, None, _lib.ptr(w), st),
                           "snb_composite_forward")
        ctx.save_for_backward(sigma, z, rays, noise if noise is not None else sigma.new_empty(0), save_enc, save_h,
                              act16, *params)
        ctx.cfg = (float(noise_std), noise is not None, store16, bool(composite))
        return w if composite else sigma

    @staticmethod
    def backward(ctx, g_out):
        lib = _lib.load()
        sigma, z, rays, noise, save_enc, save_h, act16, *params = ctx.saved_tensors
        noise_std, has_noise, store16, composite = ctx.cfg
        dev = sigma.device
        n, S = z.shape
        P = n * S
        ps = [p.detach().contiguous() for p in params]
        # one zero-filled buffer for the gradients the pass produces (the kernels accumulate into them)
        offs, total = {}, 0
        for i in _SIGMA_PASS_TENSORS:
            offs[i] = total
            total += (ps[i].numel() + 3) // 4 * 4
        flat = torch.zeros(total, device=dev, dtype=torch.float32)
        grads = [flat[offs[i]:offs[i] + p.numel()].view_as(p) if i in offs else None for i, p in enumerate(ps)]
        parr = (C.c_void_p * 24)(*[p.data_ptr() for p in ps])
        garr = (C.c_void_p * 24)(*[g.data_ptr() if g is not None else None for g in grads])
        g = g_out.contiguous().to(torch.float32)
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            g_amax = None
            if composite:
                g_amax = torch.zeros(1, device=dev, dtype=torch.float32) if store16 else None   # bit pattern of max |g_sigma|
                g_sigma = torch.empty_like(sigma)
                _lib.check(lib.snb_composite_backward_weights(_lib.ptr(sigma), _lib.ptr(z), _lib.ptr(rays),
                                                              _lib.ptr(noise) if has_noise else None, noise_std,
                                                              _lib.ptr(g), n, S, _lib.ptr(g_sigma), _lib.ptr(g_amax), st),
                           "snb_composite_backward_weights")
            else:
                g_sigma = g
            if store16:
                ws = torch.empty(lib.snb_bwd16_workspace_bytes(P), device=dev, dtype=torch.uint8)
                _lib.check(lib.snb_field_backward16_sigma(parr, garr, _lib.ptr(g_sigma), _lib.ptr(act16), P, _lib.ptr(ws),
                                                          _lib.ptr(g_amax), st), "snb_field_backward16_sigma")
            else:
                ws_a = torch.empty(P, 256, device=dev, dtype=torch.float32)
                ws_b = torch.empty(P, 256, device=dev, dtype=torch.float32)
                ws_m = torch.empty(P, 8, device=dev, dtype=torch.int32)
                _lib.check(lib.snb_field_backward_sigma(parr, garr, _lib.ptr(g_sigma), _lib.ptr(save_enc), _lib.ptr(save_h),
                                                        P, _lib.ptr(ws_a), _lib.ptr(ws_b), _lib.ptr(ws_m), st),
                           "snb_field_backward_sigma")
        return (None, None, None, None, None, None, None, *grads)


class _Composite(torch.autograd.Function):
    """(rgb, depth, weights) = composite(raw, z, ...), backward = snb_composite_backward (closed form).
    Stand-alone differentiable compositing of a given raw tensor (stage tests; the training path uses _RenderPass)."""

    @staticmethod
    def forward(ctx, raw, z, rays, noise, noise_std, white_back):
        lib = _lib.load()
        dev = raw.device
        n, S = z.shape
        rgb = torch.empty(n, 3, device=dev, dtype=torch.float32)
        depth = torch.empty(n, device=dev, dtype=torch.float32)
        w = torch.empty(n, S, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(lib.snb_composite_forward(_lib.ptr(raw), 4, _lib.ptr(z), _lib.ptr(rays), _lib.ptr(noise),
                                                 noise_std, int(white_back), n, S, _lib.ptr(rgb), _lib.ptr(depth),
                                                 _lib.ptr(w), _lib.stream_ptr(dev)), "snb_composite_forward")
        ctx.save_for_backward(raw, z, rays, noise if noise is not None else raw.new_empty(0))
        ctx.cfg = (float(noise_std), int(white_back), noise is not None)
        return rgb, depth, w

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_w):
        lib = _lib.load()
        raw, z, rays, noise = ctx.saved_tensors
        noise_std, white_back, has_noise = ctx.cfg
        dev = raw.device
        n, S = z.shape
        g_raw = torch.empty_like(raw)
        keep = [t.contiguous().to(torch.float32) if t is not None else None for t in (g_rgb, g_depth, g_w)]
        with torch.cuda.device(dev):
            _lib.check(lib.snb_composite_backward(_lib.ptr(raw), _lib.ptr(z), _lib.ptr(rays),
                                                  _lib.ptr(noise) if has_noise else None, noise_std, white_back,
                                                  _lib.ptr(keep[0]), _lib.ptr(keep[1]), _lib.ptr(keep[2]), n, S,
                                                  _lib.ptr(g_raw), _lib.stream_ptr(dev)), "snb_composite_backward")
        return g_raw, None, None, None, None, None


def _field_composite_nograd(model, prec, rays, z, noise, noise_std, white_back):
    """One field pass + compositing with the inference kernels (snb_field_forward + snb_composite_forward)."""
    lib = _lib.load()
    dev = rays.device
    n, S = z.shape
    raw = torch.empty(n, S, 4, device=dev, dtype=torch.float32)
    rgb = torch.empty(n, 3, device=dev, dtype=torch.float32)
    depth = torch.empty(n, device=dev, dtype=torch.float32)
    w = torch.empty(n, S, device=dev, dtype=torch.float32)
    img = model.packed_weights(prec)
    with torch.cuda.device(dev):
        st = _lib.stream_ptr(dev)
        _lib.check(lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, 0, _lib.ptr(raw), st),
                   "snb_field_forward")
        _lib.check(lib.snb_composite_forward(_lib.ptr(raw), 4, _lib.ptr(z), _lib.ptr(rays), _lib.ptr(noise), noise_std,
                                             int(white_back), n, S, _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(w), st),
                   "snb_composite_forward")
    return rgb, depth, w


def _weights_nograd(model, prec, rays, z, noise, noise_std):
    """A sigma-only field pass + weights-only compositing with the inference kernels."""
    lib = _lib.load()
    dev = rays.device
    n, S = z.shape
    sigma = torch.empty(n, S, device=dev, dtype=torch.float32)
    w = torch.empty(n, S, device=dev, dtype=torch.float32)
    img = model.packed_weights(prec)
    with torch.cuda.device(dev):
        st = _lib.stream_ptr(dev)
        _lib.check(lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, 1, _lib.ptr(sigma), st),
                   "snb_field_forward")
        _lib.check(lib.snb_composite_forward(_lib.ptr(sigma), 1, _lib.ptr(z), _lib.ptr(rays), _lib.ptr(noise), noise_std,
                                             0, n, S, None, None, _lib.ptr(w), st), "snb_composite_forward")
    return w


def _needs_grad(models) -> bool:
    return torch.is_grad_enabled() and any(p.requires_grad for m in models for p in m.parameters())


def _render_rays_train(models, r, S, Ni, use_disp, perturb, noise_std, white_back, detach_coarse, rng_draw,
                       return_intermediates=False, prec: int = 0, losses: Optional[RayLosses] = None,
                       test_time: bool = False):
    """render_rays with autograd (reference models/rendering.py:126-335 under grad mode): same
    kernels for sampling / importance sampling, the field pass that keeps activations (in the
    arithmetic of `prec`: tensor-core modes or the fp32 FFMA kernel), the closed-form compositing
    backward and the tensor-core / FFMA MLP backward.  Gradients reach the NeRF parameters only.
    test_time: the coarse pass is sigma-only (rendering.py:287-292) and yields only its weights; the loss terms
    come from the fine pass alone."""
    lib = _lib.load()
    dev = r.device
    n = r.shape[0]
    st = _lib.stream_ptr(dev)

    def new(*shape):
        return torch.empty(*shape, device=dev, dtype=torch.float32)

    perturb_u = rng_draw("perturb_u", torch.rand, n, S) if perturb > 0 else None
    noise_c = rng_draw("noise_coarse", torch.randn, n, S) if (noise_std != 0 or DRAW_UNUSED_NOISE) else None
    z_steps = _linspace01(S, dev)
    z_c = new(n, S)
    with torch.cuda.device(dev):
        _lib.check(lib.snb_sample_coarse(_lib.ptr(r), _lib.ptr(z_steps), _lib.ptr(perturb_u), perturb, int(use_disp),
                                         n, S, _lib.ptr(z_c), st), "snb_sample_coarse")

    spec = losses.resolved(n, dev) if losses is not None else None
    loss_terms = {}

    def field_pass(model, z, noise, which):
        nz = noise if noise_std != 0 else None
        if not (torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())):
            # nothing to differentiate in this pass (detach_coarse, a frozen model): the inference kernels,
            # no saved activations
            return _field_composite_nograd(model, prec, r, z, nz, noise_std, white_back)
        rgb, depth, w, loss = _RenderPass.apply(model, prec, r, z, nz, noise_std, white_back, spec, *model._param_list())
        if spec is not None:
            loss_terms[which] = loss
        return rgb, depth, w

    def sigma_pass(model, z, noise):
        nz = noise if noise_std != 0 else None
        if not (torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())):
            return _weights_nograd(model, prec, r, z, nz, noise_std)
        return _SigmaPass.apply(model, prec, r, z, nz, noise_std, True, *model._param_list())

    coarse_pass = (lambda: (None, None, sigma_pass(models[0], z_c, noise_c))) if test_time else \
        (lambda: field_pass(models[0], z_c, noise_c, "coarse"))
    if detach_coarse:
        with torch.no_grad():
            rgb_c, depth_c, w_c = coarse_pass()
    else:
        rgb_c, depth_c, w_c = coarse_pass()
    result = {"opacity_coarse": w_c} if test_time else {"rgb_coarse": rgb_c, "depth_coarse": depth_c, "opacity_coarse": w_c}
    if Ni > 0:
        det = not (perturb > 0)
        pdf_u = None if det else rng_draw("pdf_u", torch.rand, n, Ni)
        noise_f = rng_draw("noise_fine", torch.randn, n, S + Ni) if (noise_std != 0 or DRAW_UNUSED_NOISE) else None
        u = _linspace01(Ni, dev) if det else pdf_u
        z_f = new(n, S + Ni)
        w_det = w_c.detach().contiguous()       # sample_pdf(...).detach(), rendering.py:311-313
        with torch.cuda.device(dev):
            _lib.check(lib.snb_importance_merge(_lib.ptr(z_c), _lib.ptr(w_det), _lib.ptr(u), 0 if det else Ni, n, S, Ni,
                                                1e-5, _lib.ptr(z_f), None, st), "snb_importance_merge")
        rgb_f, depth_f, w_f = field_pass(models[1], z_f, noise_f, "fine")
        result["rgb_fine"], result["depth_fine"], result["opacity_fine"] = rgb_f, depth_f, w_f
    else:
        z_f = None
        result["rgb_fine"], result["depth_fine"], result["opacity_fine"] = rgb_c, depth_c, w_c
    if spec is not None:
        # (2,) tensors [rgb term, depth term] per pass; "loss_rgb" / "loss_depth" = coarse + fine, which is what
        # MSELoss (losses.py:17-20) and the two s1 calls (models/sinnerf.py:310-311) add up to
        tot = None
        for which, t in loss_terms.items():
            result[f"loss_{which}"] = t
            tot = t if tot is None else tot + t
        if tot is not None:
            result["loss_rgb"], result["loss_depth"] = tot[0], tot[1]
    if return_intermediates:
        result["_inter"] = {"z_coarse": z_c, "z_fine": z_f}
    return result


def _as_rays(rays: torch.Tensor) -> torch.Tensor:
    _lib.require_device(rays, "render_rays")
    if rays.dim() != 2 or rays.shape[1] != 8:
        raise ValueError(f"render_rays: rays must be (N_rays, 8) [o, d, near, far], got {tuple(rays.shape)}")
    return rays.detach().to(torch.float32).contiguous()


def sample_pdf(bins, weights, N_importance, det=False, eps=1e-5, *, _u: Optional[torch.Tensor] = None):
    """Inverse-CDF sampling, reference models/rendering.py:15-61.
    bins (N, M+1), weights (N, M) -> (N, N_importance)."""
    _lib.require_device(bins, "sample_pdf")
    n, m = weights.shape
    if bins.shape != (n, m + 1):
        raise ValueError(f"sample_pdf: bins must be (N, M+1) = ({n}, {m + 1}), got {tuple(bins.shape)}")
    b = bins.detach().to(torch.float32)
    w = weights.detach().to(torch.float32)
    if b.stride(1) != 1:
        b = b.contiguous()
    if w.stride(1) != 1:
        w = w.contiguous()
    if det:
        u, u_stride = _linspace01(N_importance, bins.device), 0
    else:
        u = torch.rand(n, N_importance, device=bins.device) if _u is None else _u.to(bins.device, torch.float32)
        u, u_stride = u.contiguous(), N_importance
    out = torch.empty(n, N_importance, device=bins.device, dtype=torch.float32)
    with torch.cuda.device(bins.device):
        _lib.check(_lib.load().snb_sample_pdf(_lib.ptr(b), b.stride(0), _lib.ptr(w), w.stride(0), _lib.ptr(u),
                                              u_stride, n, m, N_importance, float(eps), _lib.ptr(out),
                                              _lib.stream_ptr(bins.device)), "snb_sample_pdf")
    return out


def eval_points(points, models, embeddings):
    """sigma (B,1) of the fine model at 3-D points (B,3), reference models/rendering.py:64-123
    (imported by models/sinnerf.py:13, never called there).

    Under autograd (grad mode on and a parameter of the fine model requiring grad) the gradients reach that model's
    parameters, through the sigma-only training kernels: each point is staged as a ray [x, 0, 0, 0, 0, 0] with one
    sample at z = 0, so the kernel's o + d z is exactly x.  The points themselves are not differentiated."""
    model = models[-1]
    if not _needs_grad([model]):
        return model(embeddings[0](points), sigma_only=True)
    _lib.require_device(points, "eval_points")
    if points.requires_grad:
        raise NotImplementedError("sinnerf_b200.eval_points is not differentiable in the points (as Embedding.forward); "
                                  "detach them")
    emb = embeddings[0]
    if (emb.N_freqs, emb.in_channels, emb._logscale) != (10, 3, True):
        raise NotImplementedError("eval_points: the training kernels are built for Embedding(3, 10) (logscale)")
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"eval_points: expected points (B, 3), got {tuple(points.shape)}")
    n = points.shape[0]
    rays = torch.zeros(n, 8, device=points.device, dtype=torch.float32)
    rays[:, :3] = points.detach()
    z = torch.zeros(n, 1, device=points.device, dtype=torch.float32)
    prec = config.resolve_precision()
    return _SigmaPass.apply(model, prec, rays, z, None, 0.0, False, *model._param_list())


def render_rays(models,
                embeddings,
                rays,
                N_samples=64,
                use_disp=False,
                perturb=0,
                noise_std=1,
                N_importance=0,
                chunk=1024 * 32,
                white_back=False,
                test_time=False,
                detach_coarse=False,
                noisy_coarse=True,
                *,
                precision: Optional[str] = None,
                losses: Optional[RayLosses] = None,
                pixel_scatter=None,
                _rng: Optional[Dict[str, torch.Tensor]] = None,
                _return_intermediates: bool = False,
                ):
    """Render rays -- same arguments, defaults and result keys as reference
    models/rendering.py:126-139.

    models [coarse(, fine)] are sinnerf_b200.NeRF; embeddings [xyz, dir] must be the L=10 / L=4
    logscale embeddings SinNeRF builds (models/sinnerf.py:131-132) -- the kernels compute them
    on the fly, the modules are only inspected.  `chunk` is accepted and ignored: no (P,256)
    activation ever reaches HBM in inference, so there is nothing to chunk.  Under autograd (grad
    mode on and a model parameter requiring grad) the call runs the training path: the field
    pass that also keeps activations + hand-written tensor-core backward kernels; gradients reach
    the NeRF parameters only, as in the reference; with `test_time=True` the coarse pass is the
    sigma-only one there too (its `opacity_coarse` differentiates into the coarse trunk and sigma
    head, the loss terms come from the fine pass).  `noisy_coarse` is ignored exactly
    as in the reference (:138).  Keyword-only extras: `precision` overrides
    sinnerf_b200.config (a mode name, or 'autocast': the mode follows CUDA autocast); `losses` (a RayLosses, training path only) evaluates the MSE-rgb / SmoothL1-depth
    terms of models/sinnerf.py:310-319 inside the compositing kernels and adds `loss_rgb`, `loss_depth`
    (0-dim, differentiable; coarse + fine) and `loss_coarse` / `loss_fine` ((2,) each) to the result;
    `pixel_scatter` (inference only; `(destination addresses, row offset)`, see distributed.PeerPixels) makes the last
    pass's compositing kernel also store each ray's [r, g, b, depth] row into frame buffers on other GPUs;
    `_rng` injects the four random tensors (tests).
    """
    if len(embeddings) != 2 or (embeddings[0].N_freqs, embeddings[0].in_channels) != (10, 3) or \
            (embeddings[1].N_freqs, embeddings[1].in_channels) != (4, 3):
        raise NotImplementedError("render_rays: kernels are built for Embedding(3,10) / Embedding(3,4)")
    r = _as_rays(rays)
    dev = r.device
    n = r.shape[0]
    S, Ni = int(N_samples), int(N_importance)
    coarse: NeRF = models[0]
    if Ni > 0 and len(models) < 2:
        raise ValueError("render_rays: N_importance > 0 needs a fine model (models[1])")
    if test_time and Ni == 0:
        # the reference fails at models/rendering.py:331 (rgb_coarse is never bound)
        raise UnboundLocalError("render_rays(test_time=True) requires N_importance > 0, as in the reference")
    prec = config.resolve_precision(precision)
    rng = dict(_rng or {})
    perturb = float(perturb)
    noise_std = float(noise_std)

    def new(*shape):
        return torch.empty(*shape, device=dev, dtype=torch.float32)

    def rnd(name, fn, *shape):
        t = rng.get(name)
        if t is None:
            return fn(*shape, device=dev)
        if tuple(t.shape) != shape:
            raise ValueError(f"_rng['{name}'] must be {shape}, got {tuple(t.shape)}")
        return t.to(dev, torch.float32).contiguous()

    if _needs_grad(models[:2 if Ni > 0 else 1]):
        if pixel_scatter is not None:
            raise ValueError("render_rays(pixel_scatter=...) is an inference feature: call it under torch.no_grad()")
        return _render_rays_train(models, r, S, Ni, bool(use_disp), perturb, noise_std, bool(white_back),
                                  bool(detach_coarse), rnd, _return_intermediates, prec, losses, bool(test_time))
    if losses is not None:
        raise ValueError("render_rays(losses=...) is the training path: it needs grad mode and trainable NeRF parameters")
    scatter = None
    if pixel_scatter is not None:
        if test_time:
            raise ValueError("render_rays(pixel_scatter=...) needs rgb / depth of the last pass: not with test_time")
        dsts, row_offset = pixel_scatter
        if not 1 <= len(dsts) <= _lib.MAX_PIXEL_DST:
            raise ValueError(f"pixel_scatter: 1..{_lib.MAX_PIXEL_DST} destinations, got {len(dsts)}")
        scatter = _lib.SnbPixelScatter()
        for i, d in enumerate(dsts):
            scatter.dst[i] = int(d)
        scatter.n_dst, scatter.row_offset = len(dsts), int(row_offset)

    # random draws in the reference's order (rendering.py:281, :224, :43, :224)
    perturb_u = rnd("perturb_u", torch.rand, n, S) if perturb > 0 else None
    noise_c = rnd("noise_coarse", torch.randn, n, S) if (noise_std != 0 or DRAW_UNUSED_NOISE) else None
    pdf_u = noise_f = None

    a = _lib.SnbRenderArgs()
    a.rays, a.n_rays, a.n_samples, a.n_importance = _lib.ptr(r), n, S, Ni
    a.use_disp, a.perturb, a.noise_std = int(bool(use_disp)), perturb, noise_std
    a.white_back, a.test_time, a.precision = int(bool(white_back)), int(bool(test_time)), prec
    img_c = coarse.packed_weights(prec)
    a.packed_coarse = _lib.ptr(img_c)
    z_steps = _linspace01(S, dev)
    a.z_steps = _lib.ptr(z_steps)
    a.perturb_u = _lib.ptr(perturb_u)
    a.noise_coarse = _lib.ptr(noise_c) if noise_std != 0 else None
    z_c = new(n, S)
    raw_c = new(n, S) if test_time else new(n, S, 4)
    w_c = new(n, S)
    rgb_c = None if test_time else new(n, 3)
    depth_c = None if test_time else new(n)
    a.z_coarse, a.raw_coarse, a.weights_coarse = _lib.ptr(z_c), _lib.ptr(raw_c), _lib.ptr(w_c)
    a.rgb_coarse, a.depth_coarse = _lib.ptr(rgb_c), _lib.ptr(depth_c)
    keep = [r, img_c, z_steps, perturb_u, noise_c]
    z_f = raw_f = None
    if Ni > 0:
        fine: NeRF = models[1]
        img_f = fine.packed_weights(prec)
        if perturb > 0:
            pdf_u = rnd("pdf_u", torch.rand, n, Ni)
        noise_f = rnd("noise_fine", torch.randn, n, S + Ni) if (noise_std != 0 or DRAW_UNUSED_NOISE) else None
        u_steps = _linspace01(Ni, dev)
        z_f, raw_f = new(n, S + Ni), new(n, S + Ni, 4)
        rgb_f, depth_f, w_f = new(n, 3), new(n), new(n, S + Ni)
        a.packed_fine, a.u_steps, a.pdf_u = _lib.ptr(img_f), _lib.ptr(u_steps), _lib.ptr(pdf_u)
        a.noise_fine = _lib.ptr(noise_f) if noise_std != 0 else None
        a.z_fine, a.raw_fine = _lib.ptr(z_f), _lib.ptr(raw_f)
        a.rgb_fine, a.depth_fine, a.weights_fine = _lib.ptr(rgb_f), _lib.ptr(depth_f), _lib.ptr(w_f)
        keep += [img_f, u_steps, pdf_u, noise_f]

    if scatter is not None:
        a.pixel_scatter = C.pointer(scatter)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().snb_render_forward(C.byref(a), _lib.stream_ptr(dev)), "snb_render_forward")

    if test_time:
        result = {"opacity_coarse": w_c}
    else:
        result = {"rgb_coarse": rgb_c, "depth_coarse": depth_c, "opacity_coarse": w_c}
    if Ni > 0:
        result["rgb_fine"], result["depth_fine"], result["opacity_fine"] = rgb_f, depth_f, w_f
    else:  # the fine keys alias the coarse tensors (rendering.py:330-333)
        result["rgb_fine"], result["depth_fine"], result["opacity_fine"] = rgb_c, depth_c, w_c
    if _return_intermediates:
        result["_inter"] = {"z_coarse": z_c, "raw_coarse": raw_c, "z_fine": z_f, "raw_fine": raw_f}
    return result


_weight_cache: Dict[tuple, tuple] = {}


def _combine_losses(batch_losses: Sequence[Optional[RayLosses]], sizes: List[int], dev) -> Optional[RayLosses]:
    """One RayLosses over the concatenated rays: per-ray weight vectors carry each batch's own normalisation
    (default 'mean' over THAT batch) and are zero where a batch has no target.  The weight vectors depend only
    on the batch sizes and scalar weights, so they are built once and cached."""
    if batch_losses is None or all(b is None for b in batch_losses):
        return None
    if len(batch_losses) != len(sizes):
        raise ValueError("render_rays_multi: `batch_losses` needs one entry (RayLosses or None) per ray batch")
    any_rgb = any(b is not None and b.target_rgb is not None for b in batch_losses)
    any_dep = any(b is not None and b.target_depth is not None for b in batch_losses)

    def scalar_key(b, which):
        if b is None or getattr(b, "target_" + which) is None:
            return 0.0
        w = getattr(b, which + "_weight")
        if isinstance(w, torch.Tensor):
            return None          # per-ray weights given: no caching
        return ("mean",) if w is None else float(w)

    keys = tuple((scalar_key(b, "rgb"), scalar_key(b, "depth")) for b in batch_losses)
    cacheable = all(k[0] is not None and k[1] is not None for k in keys)
    ck = (tuple(sizes), keys, str(dev))
    hit = _weight_cache.get(ck) if cacheable else None
    if hit is None:
        def weights(which, denom_mul):
            parts = []
            for b, nb in zip(batch_losses, sizes):
                if b is None or getattr(b, "target_" + which) is None:
                    parts.append(torch.zeros(nb, device=dev))
                    continue
                w = getattr(b, which + "_weight")
                if isinstance(w, torch.Tensor):
                    parts.append(w.detach().to(dev, torch.float32).reshape(nb))
                else:
                    parts.append(torch.full((nb,), (1.0 / (denom_mul * max(nb, 1))) if w is None else float(w), device=dev))
            return torch.cat(parts)
        hit = (weights("rgb", 3) if any_rgb else None, weights("depth", 1) if any_dep else None)
        if cacheable:
            if len(_weight_cache) > 64:
                _weight_cache.clear()
            _weight_cache[ck] = hit
    wr, wd = hit

    def targets(which, tail):
        parts = []
        for b, nb in zip(batch_losses, sizes):
            t = None if b is None else getattr(b, "target_" + which)
            parts.append(torch.zeros((nb,) + tail, device=dev) if t is None
                         else t.detach().to(dev, torch.float32).reshape((nb,) + tail))
        return torch.cat(parts)
    return RayLosses(targets("rgb", (3,)) if any_rgb else None, targets("depth", ()) if any_dep else None, wr, wd)


def render_rays_multi(models, embeddings, ray_batches, *args, batch_losses: Optional[Sequence[Optional[RayLosses]]] = None,
                      **kwargs):
    """Several `render_rays` calls with the same models and settings as ONE pass (SURVEY 8f-2).

    SinNeRF's training step renders four ray sets back to back (reference models/sinnerf.py:304-307:
    the reference-view patch, an unseen-view patch and two random sets) -- eight field passes and, under
    autograd, eight backward passes, each with its own launches, weight conversions and split-P
    reductions.  Rays are independent, so the batches are concatenated, rendered once and the result
    dict is split again; the values of every ray are those of a separate call except that with
    `perturb > 0` / `noise_std > 0` the random tensors are drawn once for the concatenation (same
    distribution, different consumption of the generator than four separate calls).
    `batch_losses` (one RayLosses or None per batch): the per-ray losses of models/sinnerf.py:310-319 evaluated
    inside the compositing kernels, each batch with its own 'mean' normalisation; the totals over all batches
    (`loss_rgb`, `loss_depth`, `loss_coarse`, `loss_fine`) are put into every result dict.
    Returns a list of result dicts, one per batch, in order."""
    batches = [_as_rays(r) for r in ray_batches]
    if not batches:
        return []
    sizes = [int(r.shape[0]) for r in batches]
    if batch_losses is not None:
        kwargs["losses"] = _combine_losses(batch_losses, sizes, batches[0].device)
    out = render_rays(models, embeddings, torch.cat(batches, 0), *args, **kwargs)
    per_key = {k: torch.split(v, sizes, 0) for k, v in out.items() if not k.startswith(("_", "loss"))}
    results = [dict() for _ in sizes]
    for k, parts in per_key.items():
        for i, part in enumerate(parts):
            results[i][k] = part
    for k, v in out.items():
        if k.startswith("loss"):
            for res in results:
                res[k] = v
    # the reference aliases the fine keys to the coarse tensors when N_importance == 0 (rendering.py:330-333)
    if out.get("rgb_fine") is out.get("rgb_coarse"):
        for res in results:
            for k in ("rgb", "depth", "opacity"):
                if f"{k}_coarse" in res:
                    res[f"{k}_fine"] = res[f"{k}_coarse"]
    return results
