"""GPU tests of sinnerf_b200.losses (csrc/patch_loss.cu) against the float64 restatement of kornia 0.6.3's
inverse_depth_smoothness_loss and ssim_loss (tests/patch_loss_oracle.py), on contiguous NCHW tensors and on the
'(b p q) c -> b c p q' views of ray-major tensors the training step passes, plus one end-to-end check through
render_rays' training path."""
import contextlib

import pytest
import torch

from sinnerf_b200 import config, synthetic
from sinnerf_b200.losses import inverse_depth_smoothness_loss, ssim_loss
from sinnerf_b200.nerf import NeRF, Embedding
from sinnerf_b200.rendering import render_rays
from tests import patch_loss_oracle as plo
from tests._common import assert_close, max_rel, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D = torch.float64

SMOOTH_SHAPES = [(1, 64, 64), (1, 63, 84), (1, 56, 70), (2, 64, 64), (1, 2, 2)]       # (B, H, W)
SSIM_SHAPES = [(1, 64, 64), (1, 63, 84), (1, 56, 70), (2, 64, 64), (1, 6, 7)]
LAYOUTS = ["nchw", "rays"]


@contextlib.contextmanager
def no_tf32():
    """The fp32 oracle's conv2d in true fp32: cuDNN would otherwise run it in TF32."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def as_layout(x, layout, requires_grad=False):
    """-> (leaf, view): x (B,C,H,W) as a contiguous tensor, or as the '(b p q) c -> b c p q' view of a ray-major
    (B*H*W, C) tensor (the leaf), the way models/sinnerf.py rearranges render_rays' outputs."""
    B, Cc, H, W = x.shape
    if layout == "nchw":
        leaf = x.detach().clone().contiguous().requires_grad_(requires_grad)
        return leaf, leaf
    leaf = x.detach().permute(0, 2, 3, 1).reshape(B * H * W, Cc).contiguous().requires_grad_(requires_grad)
    return leaf, leaf.view(B, H, W, Cc).permute(0, 3, 1, 2)


def smooth_inputs(B, H, W, seed):
    """Depth 2..6 with a flat run, rgb in [0,1] with a white block: exactly equal neighbours in both (sign(0) = 0)."""
    g = torch.Generator().manual_seed(seed)
    d = torch.rand(B, 1, H, W, generator=g) * 4 + 2
    img = torch.rand(B, 3, H, W, generator=g)
    img[:, :, : H // 2, : W // 3] = 1.0
    d[:, :, H // 3:, W // 2:] = 3.5
    return d.to(DEV), img.to(DEV)


def smooth_run(d, img, layout):
    (dl, dv), (il, iv) = as_layout(d, layout, True), as_layout(img, layout, True)
    loss = inverse_depth_smoothness_loss(dv, iv)
    gd, gi = torch.autograd.grad(loss, [dv, iv])
    assert gd.stride() == dv.stride() and gi.stride() == iv.stride()
    return loss.detach(), gd, gi


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("shape", SMOOTH_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_smoothness_vs_float64(shape, layout):
    B, H, W = shape
    d, img = smooth_inputs(B, H, W, seed=H * W + B)
    loss, gd, gi = smooth_run(d, img, layout)
    d64, i64 = d.double().requires_grad_(True), img.double().requires_grad_(True)
    ref = plo.inverse_depth_smoothness_loss(d64, i64)
    rd, ri = torch.autograd.grad(ref, [d64, i64])
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)), (float(loss), float(ref))
    assert_close(gd, rd, 1e-4, "g_idepth")
    assert_close(gi, ri, 1e-4, "g_image")


def ssim_inputs(B, Cc, H, W, seed, depth=False):
    g = torch.Generator().manual_seed(seed)
    if not depth:
        x = torch.rand(B, Cc, H, W, generator=g)
        y = (x + 0.2 * torch.rand(B, Cc, H, W, generator=g)).clamp(0, 1)
        x[:, :, : H // 3, : W // 2] = 1.0       # flat white background in both
        y[:, :, : H // 3, : W // 2] = 1.0
        return x.to(DEV), y.to(DEV)
    # depth-valued (values 2..6, max_val = 1): a smooth surface plus a little noise, the target close to it
    ii, jj = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    surf = 2 + 4 * torch.sigmoid(3 * (ii - jj)) * (0.6 + 0.4 * torch.cos(3 * ii))
    x = surf.expand(B, 1, H, W) + 0.01 * torch.rand(B, 1, H, W, generator=g)
    y = surf.expand(B, 1, H, W) + 0.01 * torch.rand(B, 1, H, W, generator=g)
    return x.to(DEV), y.to(DEV)


def ssim_run(x, y, layout):
    xl, xv = as_layout(x, layout, True)
    _, yv = as_layout(y, layout)
    loss = ssim_loss(xv, yv, 11)
    (gx,) = torch.autograd.grad(loss, [xv])
    assert gx.stride() == xv.stride()
    return loss.detach(), gx


def ssim_ref(x, y, dtype):
    xr = x.to(dtype).requires_grad_(True)
    with no_tf32():
        loss = plo.ssim_loss(xr, y.to(dtype), 11)
        (g,) = torch.autograd.grad(loss, [xr])
    return loss.detach(), g


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("shape", SSIM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_ssim_rgb_vs_float64(shape, channels, layout):
    B, H, W = shape
    x, y = ssim_inputs(B, channels, H, W, seed=H * W + channels)
    loss, gx = ssim_run(x, y, layout)
    ref, rg = ssim_ref(x, y, D)
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)), (float(loss), float(ref))
    assert_close(gx, rg, 1e-4, "g_img1")


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("shape", SSIM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_ssim_depth_vs_float64(shape, layout):
    """Depth-valued SSIM is ill-conditioned in fp32 (sigma^2 = f(x^2) - mu^2 cancels): the kernels are held to twice the
    fp32 oracle's own deviation from float64 on the same inputs, floored at 1e-5."""
    B, H, W = shape
    x, y = ssim_inputs(B, 1, H, W, seed=7 + H * W, depth=True)
    loss, gx = ssim_run(x, y, layout)
    ref, rg = ssim_ref(x, y, D)
    l32, g32 = ssim_ref(x, y, torch.float32)
    bar_loss = max(2 * abs(float(l32) - float(ref)) / abs(float(ref)), 1e-5)
    bar_l2 = max(2 * rel_l2(g32, rg), 1e-5)
    bar_max = max(2 * max_rel(g32, rg), 1e-5)
    err = abs(float(loss) - float(ref)) / abs(float(ref))
    print(f"depth ssim {shape} {layout}: kernel loss {err:.2e} grad {rel_l2(gx, rg):.2e}/{max_rel(gx, rg):.2e}; "
          f"fp32 oracle loss {abs(float(l32) - float(ref)) / abs(float(ref)):.2e} grad {rel_l2(g32, rg):.2e}/"
          f"{max_rel(g32, rg):.2e}")
    assert err <= bar_loss, (err, bar_loss)
    assert rel_l2(gx, rg) <= bar_l2 and max_rel(gx, rg) <= bar_max, (rel_l2(gx, rg), max_rel(gx, rg), bar_l2, bar_max)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_bitwise_repeatable_and_upstream_scaling(layout):
    d, img = smooth_inputs(2, 63, 84, seed=11)
    x, y = ssim_inputs(2, 3, 63, 84, seed=12)

    def grads(scale):
        (dl, dv), (il, iv), (xl, xv) = (as_layout(t, layout, True) for t in (d, img, x))
        _, yv = as_layout(y, layout)
        ls, lq = inverse_depth_smoothness_loss(dv, iv), ssim_loss(xv, yv, 11)
        (scale * ls + scale * lq).backward()
        return ls.detach(), lq.detach(), dl.grad, il.grad, xl.grad

    a, b = grads(1.0), grads(1.0)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    z = grads(0.0)
    for t in z[2:]:
        assert int(torch.count_nonzero(t)) == 0
    s = grads(3.7)
    for u, v in zip(a[2:], s[2:]):
        assert torch.equal(v, 3.7 * u)


def test_fp32_under_fp16_autocast():
    x, y = ssim_inputs(1, 3, 64, 64, seed=13)
    d, img = smooth_inputs(1, 64, 64, seed=14)
    want = (ssim_loss(x, y, 11), inverse_depth_smoothness_loss(d, img))
    with torch.autocast("cuda", dtype=torch.float16):
        got = (ssim_loss(x, y, 11), inverse_depth_smoothness_loss(d, img))
    for u, v in zip(want, got):
        assert v.dtype == torch.float32 and torch.equal(u, v)


def test_argument_errors():
    x = torch.rand(1, 3, 8, 8, device=DEV)
    with pytest.raises(NotImplementedError, match="window_size"):
        ssim_loss(x, x, 7)
    with pytest.raises(NotImplementedError, match="reduction"):
        ssim_loss(x, x, 11, reduction="sum")
    with pytest.raises(NotImplementedError, match="img2"):
        ssim_loss(x, x.clone().requires_grad_(True), 11)
    with pytest.raises(ValueError, match="H, W >= 6"):
        ssim_loss(x[:, :, :5], x[:, :, :5], 11)
    with pytest.raises(NotImplementedError, match="one channel"):
        inverse_depth_smoothness_loss(x, x)
    with pytest.raises(ValueError, match="H, W >= 2"):
        inverse_depth_smoothness_loss(x[:, :1, :, :1], x[:, :, :, :1])
    with pytest.raises(ValueError, match="shapes must be the same"):
        inverse_depth_smoothness_loss(x[:, :1, :7], x)
    with pytest.raises(TypeError, match="float32"):
        ssim_loss(x.double(), x.double(), 11)


def _models():
    models = []
    for seed in (0, 1):
        m = NeRF(use_new_activation=True)
        m.load_state_dict(synthetic.default_init_params(seed))
        models.append(m.to(DEV))
    return models, [Embedding(3, 10), Embedding(3, 4)]


@pytest.mark.parametrize("storage", ["fp32", "fp16"])
def test_end_to_end_training_patch_terms(storage):
    """render_rays' training path on two 64x64 stride-6 patches (perturb = noise_std = 0), the four smoothness terms of
    models/sinnerf.py:370-373, 395-398 plus ssim_loss(rgb_fine, target, 11): every NeRF parameter gradient matches the
    same graph with the oracle losses evaluated in float64 on the rendered fp32 outputs.
    - With fp32 activation storage the bar is 1e-4 rel-L2, or 3x the backward's own run-to-run spread where that is
      larger: single-element bias gradients are sums of ~10^6 per-point terms added with fp32 atomics, and move by up to
      ~4e-5 between two runs of the same graph.
    - With the default 16-bit storage the bar is the 16-bit backward's 1e-3: its power-of-two gradient scale is a step
      function of max |g_raw|, so last-bit differences in the upstream gradients can change the fp16 rounding of
      every gradient plane (measured 2.4e-4 on the fine model's bottleneck bias, against any reference).
    - With the oracle in fp32, as kornia computes, the fine model's bottleneck gradients move by ~5e-4: the default-init
      render is nearly flat, and SSIM's variances of a flat patch are rounding noise in fp32.  That is printed, not held."""
    models, emb = _models()
    full = synthetic.patch_rays("lego", 64, 64, 6, seed=1).to(DEV)
    side = synthetic.patch_rays("lego", 64, 64, 6, seed=2).to(DEV)
    target = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3)).to(DEV)

    def rgb(out):
        return out["rgb_fine"].view(1, 64, 64, 3).permute(0, 3, 1, 2)

    def depth(out, k):
        return out[k].view(1, 64, 64, 1).permute(0, 3, 1, 2)

    def grads(smooth, ssim):
        for m in models:
            m.zero_grad(set_to_none=True)
        rf = render_rays(models, emb, full, 64, False, 0, 0, 64, 32768, True)
        rs = render_rays(models, emb, side, 64, False, 0, 0, 64, 32768, True)
        loss = smooth(depth(rf, "depth_fine"), rgb(rf)) + smooth(depth(rf, "depth_coarse"), rgb(rf)) \
            + smooth(depth(rs, "depth_coarse"), rgb(rs)) + smooth(depth(rs, "depth_fine"), rgb(rs)) \
            + ssim(rgb(rf), target, 11)
        loss.backward()
        return float(loss), [{k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
                             for m in models]

    def f64(smooth, ssim):
        return (lambda d, i: smooth(d.double(), i.double())), (lambda a, b, w: ssim(a.double(), b.double(), w))

    old = config.get_train_storage()
    config.set_train_storage(storage)
    try:
        lf, gf = grads(inverse_depth_smoothness_loss, ssim_loss)
        lo, go = grads(*f64(plo.inverse_depth_smoothness_loss, plo.ssim_loss))
        _, go2 = grads(*f64(plo.inverse_depth_smoothness_loss, plo.ssim_loss))
        with no_tf32():
            _, g32 = grads(plo.inverse_depth_smoothness_loss, plo.ssim_loss)
    finally:
        config.set_train_storage(old)
    assert abs(lf - lo) <= 1e-5 * abs(lo), (lf, lo)
    n, worst, worst32 = 0, 0.0, 0.0
    for a, b, b2, c in zip(gf, go, go2, g32):
        assert a.keys() == b.keys()
        for k in a:
            if float(b[k].norm()) == 0.0:
                continue
            bar = max(1e-4, 3 * rel_l2(b2[k], b[k])) if storage == "fp32" else 1e-3
            assert rel_l2(a[k], b[k]) <= bar, (k, rel_l2(a[k], b[k]), bar)
            worst, worst32 = max(worst, rel_l2(a[k], b[k])), max(worst32, rel_l2(c[k], b[k]))
            n += 1
    print(f"end to end ({storage} storage): worst parameter-gradient rel-L2 {worst:.2e} (fused losses), "
          f"{worst32:.2e} (fp32 oracle losses)")
    assert n >= 30
