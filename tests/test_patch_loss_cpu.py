"""CPU tests of the patch losses: the float64 restatement of kornia's inverse_depth_smoothness_loss / ssim_loss
(tests/patch_loss_oracle.py), the reflect-pad adjoint the SSIM backward kernel applies, and the C ABI's argument
checks.  No GPU: sinnerf_b200.losses itself is checked on the H100 by tests/test_gpu_patch_loss.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sinnerf_b200 import _lib, build
from tests import patch_loss_oracle as plo

D = torch.float64


def test_gaussian_taps():
    g = plo.gaussian_1d(11, 1.5)
    assert g.shape == (11,)
    assert torch.equal(g, g.flip(0))
    assert abs(float(g.sum()) - 1.0) < 1e-15
    want = 1.0 / sum(math.exp(-x * x / 4.5) for x in range(-5, 6))
    assert abs(float(g[5]) - want) < 1e-15
    g2 = plo.gaussian_2d(11, 1.5)
    assert abs(float(g2.sum()) - 1.0) < 1e-14 and torch.equal(g2, g2.t())


def _reflect(k, n):
    return -k if k < 0 else (2 * (n - 1) - k if k >= n else k)


@pytest.mark.parametrize("hw", [(6, 7), (9, 13), (17, 6)])
def test_reflect_filter_matches_direct_sum(hw):
    """filter2d == F.pad(reflect) + conv2d == the direct sum over reflected indices the forward kernel stages."""
    h, w = hw
    x = torch.rand(2, 3, h, w, dtype=D, generator=torch.Generator().manual_seed(h * w))
    k = plo.gaussian_2d(11, 1.5)
    got = plo.filter2d(x, k)
    ref = F.conv2d(F.pad(x, [5, 5, 5, 5], mode="reflect"), k.expand(3, 1, 11, 11), groups=3)
    assert torch.equal(got, ref)
    xn, kn = x.numpy(), k.numpy()
    direct = np.zeros_like(xn)
    for i in range(h):
        for j in range(w):
            for a in range(-5, 6):
                for b in range(-5, 6):
                    direct[:, :, i, j] += kn[a + 5, b + 5] * xn[:, :, _reflect(i + a, h), _reflect(j + b, w)]
    assert np.abs(direct - got.numpy()).max() < 1e-14


def _adj_weight(g, p, q, n):
    """patch_loss.cu adj_weight: the weight with which output p of 'reflect-pad by 5, correlate' reads input q."""
    def tap(k):
        return float(g[k + 5]) if -5 <= k <= 5 else 0.0
    w = tap(q - p)
    if 1 <= q <= 5:
        w += tap(-q - p)
    if n - 6 <= q <= n - 2:
        w += tap(2 * (n - 1) - q - p)
    return w


@pytest.mark.parametrize("n", [6, 7, 8, 11, 12, 20])
def test_reflect_adjoint_fold(n):
    """The backward kernel's 1-D weights (incl. the fold of padded positions onto their mirror pixels, which covers
    most of the image at these sizes) are the matrix of pad-then-correlate, and vanish for |p - q| > 5."""
    g = plo.gaussian_1d(11, 1.5)
    M = torch.zeros(n, n, dtype=D)
    for p in range(n):
        for k in range(-5, 6):
            M[p, _reflect(p + k, n)] += g[k + 5]
    W = torch.tensor([[_adj_weight(g, p, q, n) if abs(p - q) <= 5 else 0.0 for q in range(n)] for p in range(n)], dtype=D)
    assert (M - W).abs().max() < 1e-16
    for p in range(n):
        for q in range(n):
            if abs(p - q) > 5:
                assert _adj_weight(g, p, q, n) == 0.0
    # and the 2-D filter is the separable product of it: f(x) = M x M^T per plane
    x = torch.rand(1, 1, n, n + 1, dtype=D, generator=torch.Generator().manual_seed(n))
    Mw = torch.zeros(n + 1, n + 1, dtype=D)
    for p in range(n + 1):
        for k in range(-5, 6):
            Mw[p, _reflect(p + k, n + 1)] += g[k + 5]
    assert (plo.filter2d(x, plo.gaussian_2d()) [0, 0] - M @ x[0, 0] @ Mw.t()).abs().max() < 1e-15


def test_ssim_of_identical_images_is_zero():
    x = torch.rand(2, 3, 16, 20, dtype=D, generator=torch.Generator().manual_seed(1))
    assert abs(float(plo.ssim_loss(x, x.clone(), 11))) < 1e-9


@pytest.mark.parametrize("slope", [0.25, -1.5])
def test_smoothness_closed_forms(slope):
    h, w = 7, 9
    img = torch.full((2, 3, h, w), 0.4, dtype=D)
    ramp_w = (slope * torch.arange(w, dtype=D)).expand(2, 1, h, w)
    # along W: |dx| = |slope| with unit weights over every x edge; dy = 0
    assert abs(float(plo.inverse_depth_smoothness_loss(ramp_w, img)) - abs(slope)) < 1e-14
    ramp_h = (slope * torch.arange(h, dtype=D)[:, None]).expand(2, 1, h, w)
    assert abs(float(plo.inverse_depth_smoothness_loss(ramp_h, img)) - abs(slope)) < 1e-14
    assert float(plo.inverse_depth_smoothness_loss(torch.full((2, 1, h, w), 3.0, dtype=D), img)) == 0.0


def _flat_patches(g):
    """Images with exactly equal neighbours (white background next to content) and depth with flat runs."""
    img = torch.rand(1, 3, 6, 7, dtype=D, generator=g)
    img[:, :, :3, :4] = 1.0
    d = torch.rand(1, 1, 6, 7, dtype=D, generator=g) * 4 + 2
    d[:, :, 2:5, 1:4] = 3.0
    return d, img


def test_smoothness_gradcheck():
    g = torch.Generator().manual_seed(2)
    d = (torch.rand(2, 1, 5, 6, dtype=D, generator=g) * 4 + 2).requires_grad_(True)
    img = torch.rand(2, 3, 5, 6, dtype=D, generator=g).requires_grad_(True)
    assert torch.autograd.gradcheck(plo.inverse_depth_smoothness_loss, (d, img))
    d, img = _flat_patches(g)
    d.requires_grad_(True)
    img.requires_grad_(True)
    assert torch.autograd.gradcheck(plo.inverse_depth_smoothness_loss, (d, img))
    # sign(0) = 0: an image gradient through an edge whose channel difference is exactly 0 is exactly 0
    plo.inverse_depth_smoothness_loss(d, img).backward()
    assert float(img.grad[0, :, 0, 1].abs().max()) == 0.0     # all four incident edges lie in the flat block


def test_ssim_gradcheck():
    g = torch.Generator().manual_seed(3)
    x = torch.rand(1, 2, 6, 7, dtype=D, generator=g).requires_grad_(True)
    y = torch.rand(1, 2, 6, 7, dtype=D, generator=g)
    assert torch.autograd.gradcheck(lambda a: plo.ssim_loss(a, y, 11), (x,))
    d, _ = _flat_patches(g)
    dt = d + 0.1 * torch.rand(d.shape, dtype=D, generator=g)
    d.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a: plo.ssim_loss(a, dt, 11), (d,))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_cabi_argument_validation_without_gpu(lib):
    s = (C.c_int64 * 4)(12, 12, 4, 1)
    p = C.c_void_p(16)   # never dereferenced: every failing check comes before any CUDA call
    # smoothness: H, W >= 2, non-null operands and outputs
    assert lib.snb_depth_smooth_forward(p, s, p, s, 1, 3, 1, 4, p, p, None) == -1
    assert b"H, W >= 2" in lib.snb_last_error()
    assert lib.snb_depth_smooth_forward(None, s, p, s, 1, 3, 4, 4, p, p, None) == -1
    assert b"null pointer" in lib.snb_last_error() and b"idepth" in lib.snb_last_error()
    assert lib.snb_depth_smooth_forward(p, s, p, None, 1, 3, 4, 4, p, p, None) == -1
    assert b"image" in lib.snb_last_error()
    assert lib.snb_depth_smooth_forward(p, s, p, s, 1, 3, 4, 4, None, p, None) == -1
    assert b"workspace" in lib.snb_last_error()
    assert lib.snb_depth_smooth_forward(p, s, p, s, 0, 3, 4, 4, p, p, None) == -1
    assert b"batch" in lib.snb_last_error()
    assert lib.snb_depth_smooth_backward(p, s, p, s, 1, 3, 4, 4, None, p, s, p, s, None) == -1
    assert b"g_loss" in lib.snb_last_error()
    assert lib.snb_depth_smooth_backward(p, s, p, s, 1, 3, 4, 4, p, p, None, None, None, None) == -1
    assert b"g_idepth" in lib.snb_last_error()
    assert lib.snb_depth_smooth_backward(p, s, p, s, 1, 3, 4, 1, p, p, s, p, s, None) == -1
    assert b"H, W >= 2" in lib.snb_last_error()
    neg = (C.c_int64 * 4)(12, -1, 4, 1)
    assert lib.snb_depth_smooth_forward(p, s, p, neg, 1, 3, 4, 4, p, p, None) == -1
    assert b"negative stride" in lib.snb_last_error()
    # ssim: window 11 only (unsupported, -3), H, W >= 6, non-null operands, outputs and coefficient maps
    assert lib.snb_ssim_loss_forward(p, s, p, s, 1, 3, 8, 8, 7, 1.0, 1e-12, p, p, p, None) == -3
    assert b"window_size 11" in lib.snb_last_error()
    assert lib.snb_ssim_loss_forward(p, s, p, s, 1, 3, 5, 8, 11, 1.0, 1e-12, p, p, p, None) == -1
    assert b"H, W >= 6" in lib.snb_last_error()
    assert lib.snb_ssim_loss_forward(p, s, None, s, 1, 3, 8, 8, 11, 1.0, 1e-12, p, p, p, None) == -1
    assert b"img2" in lib.snb_last_error()
    assert lib.snb_ssim_loss_forward(p, s, p, s, 1, 3, 8, 8, 11, 1.0, 1e-12, p, p, None, None) == -1
    assert b"workspace" in lib.snb_last_error()
    assert lib.snb_ssim_loss_backward(p, s, p, s, 1, 3, 8, 5, p, p, p, s, None) == -1
    assert b"H, W >= 6" in lib.snb_last_error()
    assert lib.snb_ssim_loss_backward(p, s, p, s, 1, 3, 8, 8, None, p, p, s, None) == -1
    assert b"coef" in lib.snb_last_error()
    assert lib.snb_ssim_loss_backward(p, s, p, s, 1, 3, 8, 8, p, p, None, s, None) == -1
    assert b"g_img1" in lib.snb_last_error()


def test_python_argument_errors_without_gpu():
    from sinnerf_b200.losses import inverse_depth_smoothness_loss, ssim_loss
    x = torch.rand(1, 3, 8, 8)
    with pytest.raises(ValueError, match="BxCxHxW"):
        inverse_depth_smoothness_loss(torch.rand(8, 8), x)
    with pytest.raises(ValueError, match="BxCxHxW"):
        ssim_loss(x, torch.rand(3, 8, 8), 11)
    with pytest.raises(TypeError):
        ssim_loss(x.numpy(), x, 11)
    # well-formed CPU tensors: no CPU path
    with pytest.raises(RuntimeError, match="no CPU path"):
        inverse_depth_smoothness_loss(torch.rand(1, 1, 8, 8), x)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ssim_loss(x, x, 11)


def test_against_kornia():
    """The restatement against kornia itself, wherever kornia 0.6.x is installed."""
    kornia = pytest.importorskip("kornia")
    from kornia.losses import inverse_depth_smoothness_loss as k_smooth, ssim_loss as k_ssim
    g = torch.Generator().manual_seed(5)
    for shape in [(1, 3, 64, 64), (2, 3, 63, 84), (1, 1, 6, 7)]:
        x = torch.rand(shape, dtype=D, generator=g)
        y = torch.rand(shape, dtype=D, generator=g)
        d = torch.rand(shape[0], 1, *shape[2:], dtype=D, generator=g) * 4 + 2
        a = x.clone().requires_grad_(True)
        b = x.clone().requires_grad_(True)
        la, lb = k_ssim(a, y, 11), plo.ssim_loss(b, y, 11)
        (la + k_smooth(d, a)).backward()
        (lb + plo.inverse_depth_smoothness_loss(d, b)).backward()
        assert abs(float(la - lb)) <= 1e-12 * max(1.0, abs(float(la))), kornia.__version__
        assert float((a.grad - b.grad).abs().max()) <= 1e-12 * float(b.grad.abs().max())
        ld = k_ssim(d, d.flip(-1).contiguous(), 11, max_val=1.0)
        assert abs(float(ld - plo.ssim_loss(d, d.flip(-1).contiguous(), 11))) <= 1e-12
