"""The CPU oracle's restatement of the single-product fp16 mode (SNB_PREC_F16, the reference's arithmetic under
Lightning's precision=16): nn.Linear operands rounded to fp16 with fp32 accumulation and the bottleneck folded into the
direction layer, exactly as oracle.render_oracle restates the bf16 mode (`linear_dtype`, `fold_bottleneck`), plus the
kernels' saturation of fp16 operands at +-65504, where a plain conversion to fp16 overflows to inf.

oracle/ is the yardstick every test shares and stays as it is, so the saturation is added here: for the duration of a
call the oracle's operand-rounding helper is replaced by one that clamps fp16 operands first (straight-through in the
backward, like the rounding itself).  bf16 operands pass through unchanged."""
import contextlib

import torch

from oracle import render_oracle as orc

F16_MAX = 65504.0
F16 = dict(linear_dtype=torch.float16, fold_bottleneck=True)
_round_st = orc._round_st


def _round_st_saturating(x, dt):
    if dt is torch.float16:
        x = x + (x.clamp(-F16_MAX, F16_MAX) - x).detach()
    return _round_st(x, dt)


@contextlib.contextmanager
def fp16_saturation():
    orc._round_st = _round_st_saturating
    try:
        yield
    finally:
        orc._round_st = _round_st


def affine(p, name, x, linear_dtype=torch.float16):
    """One nn.Linear of the restatement (oracle _affine with saturating fp16 operands)."""
    with fp16_saturation():
        return orc._affine(p, name, x, linear_dtype)


def field_mlp(p, xyz_enc, dir_enc, **kw):
    with fp16_saturation():
        return orc.field_mlp(p, xyz_enc, dir_enc, **F16, **kw)


def render_rays(coarse, fine, rays, **kw):
    with fp16_saturation():
        return orc.render_rays(coarse, fine, rays, **F16, **kw)
