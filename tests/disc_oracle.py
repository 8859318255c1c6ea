"""Restatement of SinNeRF's discriminator forward (models/discriminator.py, models/diff_aug.py) with the random draws
as explicit arguments, in the dtype and on the device of its input: the tests run it in float64 on the CPU,
tools/time_discriminator.py as fp32 PyTorch on the GPU.

`forward(weights, us, vs, x, imsize, training, aug)` returns (out, us', vs', sigmas): the output, the power-iterated
u and v of every layer (training) or the given ones (eval), and the sigma each layer's weight was divided by.  It is
differentiable in x and in the weight_origs through autograd; u and v are constants of the call, as in
torch.nn.utils.spectral_norm.  `near_kink` = (tau, list) collects the LeakyReLU inputs within tau of zero, and
`flips` {layer: bool mask} puts chosen inputs on the other branch of their LeakyReLU (for a gradient taken by an
arithmetic that rounded them across the kink).  aug is None or (brightness, saturation, contrast, cutout row offset, cutout column
offset), each of B values, as sinnerf_b200.discriminator.draw_augment returns them.
"""
import torch
import torch.nn.functional as F

from sinnerf_b200.discriminator import layer_schedule


def _normalize(t, eps=1e-12):
    return t / t.norm().clamp_min(eps)


def augment(x, aug):
    """DiffAugment 'color,cutout' with the given draws, in x's dtype and on x's device (no host round trip)"""
    B, _, H, W = x.shape
    rb, rs, rc = (t.reshape(B, 1, 1, 1).to(x) for t in aug[:3])
    oy, ox = (t.reshape(B, 1, 1).to(x.device) for t in aug[3:])
    x = x + (rb - 0.5)
    m = x.mean(1, keepdim=True)
    x = (x - m) * (rs * 2) + m
    m = x.mean((1, 2, 3), keepdim=True)
    x = (x - m) * (rc + 0.5) + m
    # rand_cutout zeroes the clamped index range of a ch x cw window centred on the offsets
    ch, cw = int(H * 0.5 + 0.5), int(W * 0.5 + 0.5)
    y0, y1 = (oy - ch // 2).clamp(0, H - 1), (oy - ch // 2 + ch - 1).clamp(0, H - 1)
    x0, x1 = (ox - cw // 2).clamp(0, W - 1), (ox - cw // 2 + cw - 1).clamp(0, W - 1)
    r = torch.arange(H, device=x.device).view(1, H, 1)
    c = torch.arange(W, device=x.device).view(1, 1, W)
    cut = (r >= y0) & (r <= y1) & (c >= x0) & (c <= x1)
    return x * (~cut).to(x.dtype).unsqueeze(1)


def forward(weights, us, vs, x, imsize, training=True, aug=None, near_kink=None, flips=None):
    spec = layer_schedule(imsize)
    assert len(weights) == len(spec)
    if aug is not None:
        x = augment(x, aug)
    us2, vs2, sigmas = [], [], []
    for i, ((_, cout, inorm), w) in enumerate(zip(spec, weights)):
        last = i == len(spec) - 1
        wm = w.reshape(cout, -1)
        with torch.no_grad():
            u, v = us[i].to(x), vs[i].to(x)
            if training:
                v = _normalize(wm.detach().t() @ u)
                u = _normalize(wm.detach() @ v)
        sigma = torch.dot(u, wm @ v)
        x = F.conv2d(x, w / sigma, stride=1 if last else 2, padding=0 if last else 1)
        if inorm:
            mean = x.mean((2, 3), keepdim=True)
            var = ((x - mean) ** 2).mean((2, 3), keepdim=True)
            x = (x - mean) / torch.sqrt(var + 1e-5)
        if not last:
            if near_kink is not None:
                # (layer, flat index, |input|, numel) of every LeakyReLU input within near_kink[0] of the kink (not at it)
                a = x.detach().abs().reshape(-1)
                idx = torch.nonzero((a > 0) & (a < near_kink[0])).reshape(-1)
                near_kink[1].extend((i, int(j), float(a[j]), a.numel()) for j in idx)
            pos = x > 0
            if flips is not None and i in flips:
                pos = pos ^ flips[i].view(x.shape)
            x = torch.where(pos, x, 0.2 * x)
        us2.append(u)
        vs2.append(v)
        sigmas.append(sigma.detach())
    return x, us2, vs2, sigmas
