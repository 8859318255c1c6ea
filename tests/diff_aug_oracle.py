"""Float64 restatement of SinNeRF's standalone DiffAugment (models/diff_aug.py) after its gate, with the random draws
as explicit arguments, in the dtype and on the device of its input: the tests run it in float64 on the CPU,
tools/time_diff_aug.py as fp32 PyTorch on the GPU.

`diff_augment(x, draws, channels_first)` applies any policy in any op order (color, translation, cutout, repeats
included) to any channel count.  draws is [(op, draws)] in policy order, as
sinnerf_b200.discriminator.diff_augment_draws returns them.  It is differentiable in x through autograd.
"""
import torch



def _color(x, rb, rs, rc):
    B = x.shape[0]
    rb, rs, rc = (t.reshape(B, 1, 1, 1).to(x) for t in (rb, rs, rc))
    x = x + (rb - 0.5)
    m = x.mean(1, keepdim=True)
    x = (x - m) * (rs * 2) + m
    m = x.mean((1, 2, 3), keepdim=True)
    return (x - m) * (rc + 0.5) + m


def _translation(x, ty, tx):
    # rand_translation: output pixel (i, j) reads the zero-padded input at clamp(i + ty + 1, 0, H + 1), i.e. input
    # row i + ty (and column j + tx), zero where that falls outside the image
    B, _, H, W = x.shape
    r = torch.arange(H, device=x.device).view(1, H, 1) + ty.reshape(B, 1, 1).to(x.device)
    c = torch.arange(W, device=x.device).view(1, 1, W) + tx.reshape(B, 1, 1).to(x.device)
    inside = (r >= 0) & (r < H) & (c >= 0) & (c < W)
    b = torch.arange(B, device=x.device).view(B, 1, 1)
    g = x[b, :, r.clamp(0, H - 1), c.clamp(0, W - 1)].permute(0, 3, 1, 2)
    return torch.where(inside.unsqueeze(1), g, torch.zeros((), dtype=x.dtype, device=x.device))


def _cutout(x, oy, ox):
    # rand_cutout zeroes the clamped index range of a ch x cw window centred on the offsets
    B, _, H, W = x.shape
    oy, ox = (t.reshape(B, 1, 1).to(x.device) for t in (oy, ox))
    ch, cw = int(H * 0.5 + 0.5), int(W * 0.5 + 0.5)
    y0, y1 = (oy - ch // 2).clamp(0, H - 1), (oy - ch // 2 + ch - 1).clamp(0, H - 1)
    x0, x1 = (ox - cw // 2).clamp(0, W - 1), (ox - cw // 2 + cw - 1).clamp(0, W - 1)
    r = torch.arange(H, device=x.device).view(1, H, 1)
    c = torch.arange(W, device=x.device).view(1, 1, W)
    cut = (r >= y0) & (r <= y1) & (c >= x0) & (c <= x1)
    return x * (~cut).to(x.dtype).unsqueeze(1)


_OPS = {"color": _color, "translation": _translation, "cutout": _cutout}


def diff_augment(x, draws, channels_first=True):
    """models/diff_aug.py DiffAugment after its gate, with the given draws -- [(op, draws)] in policy order, as
    sinnerf_b200.discriminator.diff_augment_draws returns them -- in x's dtype and on x's device: any policy and op
    order, any channel count; x is (B, C, H, W), or (B, H, W, C) with channels_first=False, and so is the result
    (contiguous)"""
    if not channels_first:
        x = x.permute(0, 3, 1, 2)
    for op, ts in draws:
        x = _OPS[op](x, *ts)
    if not channels_first:
        x = x.permute(0, 2, 3, 1)
    return x.contiguous()


