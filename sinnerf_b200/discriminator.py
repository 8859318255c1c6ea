"""SinNeRF's adversarial-loss discriminator (models/discriminator.py with models/diff_aug.py), forward and both
backwards executed by libsinnerf_b200's sm_90a kernels (csrc/disc.cu).

    from sinnerf_b200.discriminator import Discriminator      # models/sinnerf.py:12, nothing else changes

`Discriminator(conditional, policy, ndf=64, imsize=64)` builds its parameters and buffers from the same
`nn.Conv2d` + `torch.nn.utils.spectral_norm` containers, in the same order, as the reference: the state-dict keys
(`main.{i}.weight_orig`, `.weight_u`, `.weight_v`) and, under the same torch seed, the initial values are the
reference's, so a SinNeRF checkpoint's `D.*` loads with strict=True.  The submodules only hold parameters; their
forward hooks never run.

`forward(input, y=None)` makes the reference's random draws itself -- `np.random.random()` twice for the gates, then
DiffAugment's `torch.rand` / `torch.randint` calls on the input's device -- and hands the drawn device tensors to the
kernels.  In training mode each call advances every weight_u / weight_v in place by one power iteration, as
spectral_norm does, also under torch.no_grad(); the backward uses the call's own sigma, u and v, so the
discriminator step's two calls before one backward are handled as the reference handles them.  In eval mode the
stored u and v are used.  Nothing synchronises with the host.

Inputs are (B, 3, H, W) fp32 CUDA tensors read through their strides; the input gradient comes back with the input's
strides.  Gradients flow to the input and to every weight_orig.  The backward is once-differentiable: back-propagating
through it raises, so compute_grad2(create_graph=True) on D(x) does too.  The gradient penalty of dloss='wgan_gp'
comes instead from `forward_with_penalty(input)`, which returns D(input) and compute_grad2's per-image penalty of
the same call, both differentiable to first order (the penalty's gradients are second-order in the discriminator).
The GEMM arithmetic follows `precision=` or the process setting (config.resolve_precision), as in
sinnerf_b200.vit: the fp16 hi + lo three-product split by default, 'f16' / 'bf16' single products, and under
'autocast' fp16 autocast gives 'f16', the arithmetic of the reference's cuDNN convolutions under Lightning's
precision=16.  There is no CPU path.

`DiffAugment(x, policy, channels_first)` is models/diff_aug.py's standalone augmentation (any policy, translation
included) on the library's kernels, for dloss='relavistic''s `self.D(DiffAugment(real_patch))`:

    from sinnerf_b200.discriminator import DiffAugment        # models/sinnerf.py:14
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from .config import resolve_precision

__all__ = ["Discriminator", "DiffAugment", "layer_schedule", "output_sizes", "draw_augment", "diff_augment_draws"]

POLICIES = (None, "", "color,cutout")

# (in, out, InstanceNorm after) of each convolution of Discriminator.__init__'s branches for ndf = 64; every
# convolution but the last (stride 1, pad 0) has stride 2 and pad 1, and every one but the last is followed by
# LeakyReLU(0.2)
_BRANCHES = {
    128: [(3, 32, False), (32, 64, True), (64, 128, True), (128, 256, True), (256, 512, True), (512, 1, False)],
    64: [(3, 64, False), (64, 128, True), (128, 256, True), (256, 512, True), (512, 1, False)],
    32: [(3, 128, True), (128, 256, True), (256, 512, True), (512, 1, False)],
    None: [(3, 256, True), (256, 512, True), (512, 1, False)],
}


def layer_schedule(imsize):
    """[(in, out, instance norm after)] of the branch `imsize` selects (any size but 128, 64 or 32: the last)."""
    return _BRANCHES.get(imsize, _BRANCHES[None])


def output_sizes(imsize, h: int, w: int):
    """[(h_l, w_l)] of every convolution's output for an h x w input; ValueError where the reference cannot run
    (a convolution whose output would be empty, or an InstanceNorm over a single element)."""
    spec = layer_schedule(imsize)
    sizes = []
    for i, (_, _, inorm) in enumerate(spec):
        last = i == len(spec) - 1
        s, p = (1, 0) if last else (2, 1)
        if h + 2 * p < 4 or w + 2 * p < 4:
            raise ValueError(f"Discriminator(imsize={imsize}): layer {i}'s input is {h} x {w}, smaller than its 4 x 4 "
                             "kernel (the convolution's output would be empty)")
        h, w = (h + 2 * p - 4) // s + 1, (w + 2 * p - 4) // s + 1
        if inorm and h * w == 1:
            raise ValueError(f"Discriminator(imsize={imsize}): layer {i}'s InstanceNorm would normalise a single "
                             "spatial element (torch: 'Expected more than 1 spatial element when training')")
        sizes.append((h, w))
    return sizes


def _draw_color(B, H, W, device):
    # rand_brightness, rand_saturation, rand_contrast
    return tuple(torch.rand(B, 1, 1, 1, dtype=torch.float32, device=device).reshape(B) for _ in range(3))


def _draw_translation(B, H, W, device):
    # rand_translation: the shifts of dim 2 (rows) and of dim 3 (columns)
    sy, sx = int(H * 0.125 + 0.5), int(W * 0.125 + 0.5)
    ty = torch.randint(-sy, sy + 1, size=[B, 1, 1], device=device)
    tx = torch.randint(-sx, sx + 1, size=[B, 1, 1], device=device)
    return ty.reshape(B), tx.reshape(B)


def _draw_cutout(B, H, W, device):
    # rand_cutout: the offsets along the rows and the columns
    ch, cw = int(H * 0.5 + 0.5), int(W * 0.5 + 0.5)
    oy = torch.randint(0, H + (1 - ch % 2), size=[B, 1, 1], device=device)
    ox = torch.randint(0, W + (1 - cw % 2), size=[B, 1, 1], device=device)
    return oy.reshape(B), ox.reshape(B)


_DRAWS = {"color": _draw_color, "translation": _draw_translation, "cutout": _draw_cutout}


def diff_augment_draws(policy, shape, device):
    """The random draws of models/diff_aug.py DiffAugment(x, policy) for x of shape (B, C, H, W), made with the same
    calls in the same order: its gate np.random.random() < 0.5 gives None (DiffAugment returns x), else the list
    [(op, draws)] over the policy's ops in order -- empty for an empty or None policy -- with draws (brightness,
    saturation, contrast), (row shift, column shift) or (cutout row offset, cutout column offset), each of (B,)
    device tensors.  An unknown op raises KeyError once the draws before it are made, as AUGMENT_FNS[p] does."""
    if np.random.random() < 0.5:
        return None
    B, _, H, W = shape
    return [(p, _DRAWS[p](B, H, W, device)) for p in policy.split(",")] if policy else []


def draw_augment(policy, shape, device):
    """The random draws of Discriminator.forward + DiffAugment (models/discriminator.py:159, models/diff_aug.py),
    made with the same calls in the same order: None when no augmentation applies, else the tuple (brightness,
    saturation, contrast, cutout row offset, cutout column offset) of (B,) device tensors."""
    if policy is None or not np.random.random() > 0.5:
        return None
    draws = diff_augment_draws(policy, shape, device)
    if not draws:
        return None
    (_, color), (_, cutout) = draws
    return color + cutout


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


class _DiscFn(torch.autograd.Function):
    """D(x) for one call; backward to x and / or the weight_origs with this call's sigma, u and v"""

    @staticmethod
    def forward(ctx, cfg, x, *weights):
        imsize, mode, training, save, us, vs, aug, out_hw = cfg
        lib = _lib.load()
        B, _, H, W = x.shape
        dev = x.device
        ws = torch.empty(lib.snb_disc_workspace_bytes(imsize, B, H, W, int(save)), device=dev, dtype=torch.uint8)
        out = torch.empty(B, 1, *out_hw, device=dev, dtype=torch.float32)
        a = None if aug is None else _lib.SnbDiscAug(*[t.data_ptr() for t in aug])
        _lib.check(lib.snb_disc_forward(imsize, mode, int(training), _ptrs(weights), _ptrs(us), _ptrs(vs),
                                        _lib.ptr(x), (C.c_int64 * 4)(*x.stride()), B, H, W,
                                        None if a is None else C.byref(a), _lib.ptr(out), _lib.ptr(ws),
                                        _lib.stream_ptr(dev)), "snb_disc_forward")
        if save:
            ctx.save_for_backward(ws, x, *weights)
            ctx.cfg = (imsize, mode)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        lib = _lib.load()
        ws, x, *weights = ctx.saved_tensors
        imsize, mode = ctx.cfg
        g = g.detach().to(torch.float32).contiguous()
        # empty_like keeps the input's strides (a permuted view stays permuted); the kernels write every element
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        dws = [torch.empty_like(w) if need else None for w, need in zip(weights, ctx.needs_input_grad[2:])]
        B, _, H, W = x.shape
        strides = None if dx is None else (C.c_int64 * 4)(*dx.stride())
        _lib.check(lib.snb_disc_backward(imsize, mode, _ptrs(weights), B, H, W, _lib.ptr(g), _lib.ptr(dx), strides,
                                         _ptrs(dws), _lib.ptr(ws), _lib.stream_ptr(g.device)), "snb_disc_backward")
        return (None, dx, *dws)


class _PenaltyFn(torch.autograd.Function):
    """(D(x), compute_grad2(D(x), x)) for one call; backward from either or both with this call's sigma, u and v"""

    @staticmethod
    def forward(ctx, cfg, x, *weights):
        imsize, mode, training, save, us, vs, aug, out_hw = cfg
        lib = _lib.load()
        B, _, H, W = x.shape
        dev = x.device
        ws = torch.empty(lib.snb_disc_penalty_workspace_bytes(imsize, B, H, W), device=dev, dtype=torch.uint8)
        out = torch.empty(B, 1, *out_hw, device=dev, dtype=torch.float32)
        reg = torch.empty(B, device=dev, dtype=torch.float32)
        a = None if aug is None else _lib.SnbDiscAug(*[t.data_ptr() for t in aug])
        _lib.check(lib.snb_disc_penalty_forward(imsize, mode, int(training), _ptrs(weights), _ptrs(us), _ptrs(vs),
                                                _lib.ptr(x), (C.c_int64 * 4)(*x.stride()), B, H, W,
                                                None if a is None else C.byref(a), _lib.ptr(out), _lib.ptr(reg),
                                                _lib.ptr(ws), _lib.stream_ptr(dev)), "snb_disc_penalty_forward")
        ctx.set_materialize_grads(False)
        if save:
            ctx.save_for_backward(ws, x, *weights)
            ctx.cfg = (imsize, mode)
        return out, reg

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, g_reg):
        ws, x, *weights = ctx.saved_tensors
        if g_out is None and g_reg is None:
            return (None, None, *[None] * len(weights))
        lib = _lib.load()
        imsize, mode = ctx.cfg
        g_out = None if g_out is None else g_out.detach().to(torch.float32).contiguous()
        g_reg = None if g_reg is None else g_reg.detach().to(torch.float32).contiguous()
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        dws = [torch.empty_like(w) if need else None for w, need in zip(weights, ctx.needs_input_grad[2:])]
        B, _, H, W = x.shape
        strides = None if dx is None else (C.c_int64 * 4)(*dx.stride())
        _lib.check(lib.snb_disc_penalty_backward(imsize, mode, _ptrs(weights), B, H, W, _lib.ptr(g_out),
                                                 _lib.ptr(g_reg), _lib.ptr(dx), strides, _ptrs(dws), _lib.ptr(ws),
                                                 _lib.stream_ptr(x.device)), "snb_disc_penalty_backward")
        return (None, dx, *dws)


class Discriminator(nn.Module):
    """models/discriminator.py Discriminator(conditional=False, policy, ndf=64, imsize) on the library's kernels.

    `precision` (not a reference argument): the GEMM arithmetic, as for render_rays; None follows the process
    setting.  conditional=True, ndf != 64 and policies other than 'color,cutout', '' and None raise
    NotImplementedError."""

    def __init__(self, conditional, policy, ndf=64, imsize=64, precision=None):
        super().__init__()
        if conditional:
            raise NotImplementedError("Discriminator: the conditional head is not implemented (SinNeRF builds "
                                      "conditional=False)")
        if ndf != 64:
            raise NotImplementedError(f"Discriminator: ndf={ndf} is not implemented (SinNeRF uses 64)")
        if policy not in POLICIES:
            raise NotImplementedError(f"Discriminator: policy {policy!r} is not implemented; choose one of {POLICIES}")
        self.conditional = conditional
        self.policy = policy
        self.imsize = imsize
        self.precision = precision
        SN = torch.nn.utils.spectral_norm
        spec = layer_schedule(imsize)
        blocks = []
        for i, (cin, cout, inorm) in enumerate(spec):
            last = i == len(spec) - 1
            blocks.append(SN(nn.Conv2d(cin, cout, (4, 4), (1, 1) if last else (2, 2), (0, 0) if last else (1, 1),
                                       bias=False)))
            if inorm:
                blocks.append(nn.InstanceNorm2d(cout))
            if not last:
                blocks.append(nn.LeakyReLU(0.2, inplace=True))
        self.main = nn.Sequential(*blocks)

    def convs(self):
        return [m for m in self.main if isinstance(m, nn.Conv2d)]

    def _call_args(self, x, what):
        """the input checks of a call, then its draws: (cfg prefix, weights)"""
        if not isinstance(x, torch.Tensor):
            raise TypeError(f"{what}: input is not a torch.Tensor (got {type(x)})")
        if x.dim() != 4 or x.shape[0] < 1 or x.shape[1] != 3:
            raise ValueError(f"{what}: invalid input shape, we expect Bx3xHxW with B >= 1. Got: {tuple(x.shape)}")
        _lib.require_device(x, what)
        if x.dtype != torch.float32:
            raise TypeError(f"{what}: input must be float32 (got {x.dtype})")
        out_hw = output_sizes(self.imsize, x.shape[2], x.shape[3])[-1]
        convs = self.convs()
        weights = [m.weight_orig for m in convs]
        us, vs = [m.weight_u for m in convs], [m.weight_v for m in convs]
        for t in weights + us + vs:
            if t.device != x.device or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError(f"{what}: parameters and buffers must be contiguous float32 on {x.device} "
                                   f"(got {t.dtype} on {t.device}); move the module with .to(device)")
        aug = draw_augment(self.policy, tuple(x.shape), x.device)
        mode = resolve_precision(self.precision)
        save = torch.is_grad_enabled() and (x.requires_grad or any(w.requires_grad for w in weights))
        cfg = (self.imsize if self.imsize in (128, 64, 32) else -1, mode, self.training, save, us, vs, aug, out_hw)
        return cfg, weights

    def forward(self, input, y=None):
        cfg, weights = self._call_args(input, "Discriminator")
        return _DiscFn.apply(cfg, input, *weights)

    def forward_with_penalty(self, input, y=None):
        """(out, reg): out is D(input) -- the same draws, bits and weight_u / weight_v update -- and reg (B,) is
        models/sinnerf.py's compute_grad2(out, input) for this call, reg[b] = sum (d sum(out) / d input[b])^2 through
        DiffAugment and every spectral-norm layer with this call's sigma, u and v.  Both are differentiable to first
        order: reg back-propagates to every weight_orig (through sigma, as spectral_norm does) and to the input when
        it requires grad.  input need not require grad.  The wgan_gp discriminator step:

            pred_real, reg_real = D.forward_with_penalty(real_patch)
            loss_d += 10 * reg_real.mean()
        """
        cfg, weights = self._call_args(input, "Discriminator.forward_with_penalty")
        return _PenaltyFn.apply(cfg, input, *weights)


class _DiffAugFn(torch.autograd.Function):
    """DiffAugment's ops with the given draws; backward to x through the same draws"""

    @staticmethod
    def forward(ctx, x, channels_first, draws):
        lib = _lib.load()
        if channels_first:
            B, Ch, H, W = x.shape
            out = torch.empty(B, Ch, H, W, device=x.device, dtype=torch.float32)
        else:
            B, H, W, Ch = x.shape
            out = torch.empty(B, H, W, Ch, device=x.device, dtype=torch.float32)
        ops, d, _ = _diff_aug_args(draws, B)
        ws = torch.empty(B * _lib.DIFF_AUG_WS_FLOATS, device=x.device, dtype=torch.float32)
        _lib.check(lib.snb_diff_augment_forward(ops, len(draws), C.byref(d), _lib.ptr(x), _nchw_strides(x, channels_first),
                                                B, Ch, H, W, _lib.ptr(out), _nchw_strides(out, channels_first),
                                                _lib.ptr(ws), _lib.stream_ptr(x.device)), "snb_diff_augment_forward")
        # the gradient's layout: x's strides where empty_like keeps them (a permuted view stays permuted)
        ctx.args = (channels_first, draws, (B, Ch, H, W), torch.empty_like(x, device="meta"))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        channels_first, draws, (B, Ch, H, W), like = ctx.args
        if not ctx.needs_input_grad[0]:
            return None, None, None
        lib = _lib.load()
        g = g.detach().to(torch.float32)
        dx = torch.empty_strided(like.shape, like.stride(), device=g.device, dtype=torch.float32)   # all written
        ops, d, _ = _diff_aug_args(draws, B)
        ws = torch.empty(B * _lib.DIFF_AUG_WS_FLOATS, device=g.device, dtype=torch.float32)
        _lib.check(lib.snb_diff_augment_backward(ops, len(draws), C.byref(d), _lib.ptr(g), _nchw_strides(g, channels_first),
                                                 B, Ch, H, W, _lib.ptr(dx), _nchw_strides(dx, channels_first),
                                                 _lib.ptr(ws), _lib.stream_ptr(g.device)), "snb_diff_augment_backward")
        return dx, None, None


def _nchw_strides(t, channels_first):
    """t's element strides in (image, channel, row, column) order"""
    s = t.stride()
    return (C.c_int64 * 4)(*(s if channels_first else (s[0], s[3], s[1], s[2])))


def _diff_aug_args(draws, B):
    """(op codes, SnbDiffAugDraws, the tensors it points into): an op's k-th occurrence reads row k of its draws"""
    fields = {"color": ("brightness", "saturation", "contrast"), "translation": ("translation_y", "translation_x"),
              "cutout": ("cutout_y", "cutout_x")}
    rows = {}
    for op, ts in draws:
        rows.setdefault(op, []).append(ts)
    d, keep = _lib.SnbDiffAugDraws(), []
    for op, occ in rows.items():
        for name, ts in zip(fields[op], zip(*occ)):
            t = ts[0] if len(ts) == 1 else torch.stack(ts)
            keep.append(t)
            setattr(d, name, t.data_ptr())
    ops = (C.c_int * max(len(draws), 1))(*[_lib.DIFF_AUG_OPS[op] for op, _ in draws])
    return ops, d, keep


def DiffAugment(x, policy="color,cutout", channels_first=True):
    """models/diff_aug.py DiffAugment(x, policy, channels_first) on the library's kernels (csrc/disc.cu).

    x: fp32 CUDA (B, C, H, W), or (B, H, W, C) with channels_first=False, any C >= 1, read through its strides (a
    permuted view is not copied).  The reference's draws are made with the same calls in the same order (see
    diff_augment_draws): on its gate, or for an empty or None policy, x itself is returned; otherwise a new
    contiguous tensor of x's shape, with the policy's ops ('color', 'translation', 'cutout', in the order given)
    applied, and an unknown op raises KeyError.  The arithmetic is fp32 whatever the autocast state or precision
    setting, and where the policy is 'color,cutout' the values are the ones Discriminator(policy='color,cutout')
    feeds its first convolution for the same draws, bit for bit.  Differentiable in x, once: the gradient comes back
    with x's strides.  Nothing synchronises with the host."""
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"DiffAugment: input is not a torch.Tensor (got {type(x)})")
    if x.dim() != 4 or min(x.shape) < 1:
        raise ValueError(f"DiffAugment: invalid input shape, we expect a non-empty 4-d tensor. Got: {tuple(x.shape)}")
    _lib.require_device(x, "DiffAugment")
    if x.dtype != torch.float32:
        raise TypeError(f"DiffAugment: input must be float32 (got {x.dtype})")
    B, Ch, H, W = x.shape if channels_first else (x.shape[0], x.shape[3], x.shape[1], x.shape[2])
    draws = diff_augment_draws(policy, (B, Ch, H, W), x.device)
    if not draws:
        return x
    if len(draws) > _lib.DIFF_AUG_MAX_OPS:
        raise ValueError(f"DiffAugment: policy {policy!r} has {len(draws)} ops, more than {_lib.DIFF_AUG_MAX_OPS}")
    return _DiffAugFn.apply(x, bool(channels_first), draws)
