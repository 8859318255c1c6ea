"""The patch-loss kernels of sinnerf_b200/csrc/patch_loss.cu stage by stage through the C ABI, per element against
float64 on the same float32 inputs (tests/patch_loss_emulation.py).

Stages and measures (every error divided by the float64 sum of absolute values of the terms forming the element):
  SSIM forward    loss: |got - ref| / mean(|clamp(u)| + 2^-48 (1 + |ssim| kappa))   (the second term: u's own fp64
                  rounding through the condition kappa of the variance sums; it matters only where u is near 0)
                  coefficient maps dL/dmu1, dL/df(x^2), dL/df(xy): / (sum of |terms| of the closed form x kappa)
  SSIM backward   g_img1 from INJECTED coefficient maps (random, one-hot lattices covering every position, a different
                  map per plane) against the float64 autograd adjoint of reflect-pad + conv2d, / the same adjoint of
                  |maps|; g_loss = 0 gives exact zeros, g_loss = 3.7 and 2^-100 scale the g_loss = 1 result exactly
  smoothness      loss / itself (its terms are |.|); g_idepth / (inv_n sum of incident edge weights); g_image /
                  (inv_n / C sum of |d(p) - d(q)| w over incident edges); each gradient alone gives the same bits
The coefficient and output buffers are NaN-filled before every call, so an element the kernel does not write fails.
Pixels whose u lies within 4 of its rounding scale of the clamp's ends may take either side of the gate; pixels whose
windows are all zero (u = 0 exactly when eps = 0) must pass the gradient.

The checkers are functions of an implementation.  Here it is the library (`Lib`); tests/test_patch_loss_stages_cpu.py
runs the same checkers on the CPU stand-in, faithful and with one planted defect at a time.

Bars: about 4x the largest value measured on an NVIDIA H100 80GB HBM3 at its 700 W power limit, written beside them;
`pytest -s` prints worst / rms per stage at the end of the module.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import patch_loss_emulation as emu
from tests import patch_loss_oracle as plo

pytestmark = pytest.mark.gpu

f32 = np.float32
COEF_TOL = 1.2e-14      # coefficient maps / (sum |terms| x kappa)            (measured 2.9e-15)
SSIM_LOSS_TOL = 7e-7    # SSIM loss / its bound, u away from 0                  (measured 1.8e-7)
SSIM_LOSS_U0_TOL = 4e-4  # the same where the fp64 allowance of u dominates     (measured 9.4e-5)
GX_TOL = 2.4e-7         # g_img1 / adjoint of |maps|: one fp32 rounding         (measured 5.96e-8 = 2^-24)
SM_LOSS_TOL = 6e-7      # smoothness loss / itself                              (measured 1.5e-7)
SM_GD_TOL = 8e-7        # g_idepth / its bound                                  (measured 1.9e-7)
SM_GI_TOL = 1.2e-6      # g_image / its bound                                   (measured 3.1e-7)
FLOOR = 1e-300
MEASURED = {}           # stage -> [worst, sum of squares, count]

HW = (6, 7, 10, 11, 12, 16, 17, 31, 32, 33, 63, 64, 84)
SHAPES = tuple(zip(HW, HW)) + tuple(zip(HW, HW[::-1]))
BC = ((1, 1), (2, 3), (8, 3), (1, 3), (3, 1))
LAYOUTS = ("nchw", "rays", "channels_last", "crop", "expand")


# ------------------------------------------------------------------------------------------------ the library
class Lib:
    """The patch-loss entry points of include/sinnerf_b200.h on cuda:0, outputs caller-owned."""
    device = "cuda:0"

    def __init__(self):
        from sinnerf_b200 import _lib
        self._lib, self.lib = _lib, _lib.load()
        sm = C.c_int(0)
        assert self.lib.snb_device_check(C.byref(sm), None, None) == 0, self.lib.snb_last_error()
        self.sm_count = sm.value
        assert self.sm_count == torch.cuda.get_device_properties(0).multi_processor_count

    def _ok(self, rc):
        assert rc == 0, self.lib.snb_last_error()
        torch.cuda.synchronize()

    @staticmethod
    def _s(t):
        return None if t is None else (C.c_int64 * 4)(*t.stride())

    def ssim_forward(self, x, y, max_val, eps, loss, coef, ws):
        p, (B, Cc, H, W) = self._lib.ptr, x.shape
        self._ok(self.lib.snb_ssim_loss_forward(p(x), self._s(x), p(y), self._s(y), B, Cc, H, W, 11, max_val, eps,
                                                p(loss), p(coef), p(ws), None))

    def ssim_backward(self, x, y, coef, g_loss, g_x):
        p, (B, Cc, H, W) = self._lib.ptr, x.shape
        self._ok(self.lib.snb_ssim_loss_backward(p(x), self._s(x), p(y), self._s(y), B, Cc, H, W, p(coef), p(g_loss),
                                                 p(g_x), self._s(g_x), None))

    def smooth_forward(self, d, img, loss, ws):
        p, (B, Cc, H, W) = self._lib.ptr, img.shape
        self._ok(self.lib.snb_depth_smooth_forward(p(d), self._s(d), p(img), self._s(img), B, Cc, H, W, p(loss), p(ws),
                                                   None))

    def smooth_backward(self, d, img, g_loss, g_d, g_img):
        p, (B, Cc, H, W) = self._lib.ptr, img.shape
        self._ok(self.lib.snb_depth_smooth_backward(p(d), self._s(d), p(img), self._s(img), B, Cc, H, W, p(g_loss),
                                                    p(g_d), self._s(g_d), p(g_img), self._s(g_img), None))


@pytest.fixture(scope="module")
def lib():
    yield Lib()
    for k, (w, ss, n) in sorted(MEASURED.items()):
        print(f"patch-loss stage {k:14s} worst {w:.2e}  rms {math.sqrt(ss / max(n, 1)):.2e}")


# ------------------------------------------------------------------------------------------------ layouts and measures
def place(t, kind):
    """The values of t (B,C,H,W) in a layout: NCHW, the '(b p q) c -> b c p q' view of a ray-major tensor,
    channels_last, a crop of a larger NaN-filled tensor, or (kind 'expand') the first image expanded over the batch
    with stride 0 -- whose values then differ from t's, so use what is returned."""
    B, Cc, H, W = t.shape
    if kind == "nchw":
        return t.clone().contiguous()
    if kind == "rays":
        return t.permute(0, 2, 3, 1).reshape(B * H * W, Cc).contiguous().view(B, H, W, Cc).permute(0, 3, 1, 2)
    if kind == "channels_last":
        return t.contiguous(memory_format=torch.channels_last)
    if kind == "crop":
        big = torch.full((B + 1, Cc + 2, H + 3, W + 5), float("nan"), device=t.device)
        v = big[1:, 1:Cc + 1, 2:H + 2, 3:W + 3]
        v.copy_(t)
        return v
    assert kind == "expand"
    return t[:1].expand(B, Cc, H, W)


def out_like(t):
    """A NaN-filled output with t's strides inside a NaN-filled storage, and the mask of storage elements outside it."""
    extent = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    buf = torch.full((extent + 8,), float("nan"), device=t.device, dtype=t.dtype)
    out = buf.as_strided(t.shape, t.stride(), 4)
    outside = torch.ones(buf.shape, dtype=torch.bool, device=t.device)
    outside.as_strided(t.shape, t.stride(), 4).fill_(False)
    return out, lambda: bool(torch.isnan(buf[outside]).all())


def measure(got, want, bound, tol, stage, what):
    diff = (got.double() - want).abs()
    err = torch.where(diff == 0, torch.zeros_like(diff), diff / (bound + FLOOR))
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    flat = int(err.argmax())
    m = float(err.reshape(-1)[flat])
    rec = MEASURED.setdefault(stage, [0.0, 0.0, 0])
    fin = err[torch.isfinite(err)]
    rec[0], rec[1], rec[2] = max(rec[0], m), rec[1] + float((fin * fin).sum()), rec[2] + err.numel()
    idx = tuple(int(i) for i in np.unravel_index(flat, tuple(err.shape))) if err.dim() else ()
    assert m <= tol, f"{what}: {stage} error / bound = {m:.3e} > {tol:.1e} at {idx}"
    return m


def scalar(v, device):
    return torch.tensor([v], dtype=torch.float32, device=device)


def ticket(ws):
    return int(ws.view(torch.int32)[0])


# ------------------------------------------------------------------------------------------------ inputs
def ssim_case(kind, B, Cc, H, W, device, seed):
    """(x, y, max_val, eps) for one input kind."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)
    mv, eps = 1.0, 1e-12
    if kind == "rgb":                     # 8-bit values: exact ties; a flat white block and a black one in both
        x = torch.floor(r(B, Cc, H, W) * 256) / 255
        y = torch.floor((x + 0.2 * r(B, Cc, H, W)).clamp(0, 1) * 255) / 255
        for t in (x, y):
            t[:, :, : H // 3, : W // 2] = 1.0
            t[:, :, H // 2:, W // 2:] = 0.0
    elif kind in ("depth", "far_depth"):  # a smooth surface plus a little noise, the target close to it
        lo, hi = (2.0, 6.0) if kind == "depth" else (10.0, 100.0)
        ii, jj = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
        surf = lo + (hi - lo) * torch.sigmoid(3 * (ii - jj)) * (0.6 + 0.4 * torch.cos(3 * ii))
        x = surf.expand(B, Cc, H, W) + 0.01 * r(B, Cc, H, W)
        y = surf.expand(B, Cc, H, W) + 0.01 * r(B, Cc, H, W)
    elif kind in ("identical", "identical_eps0"):   # u ~ 0: the lower end of the gate; black windows give u = 0 exactly
        x = r(B, Cc, H, W)
        x[:, :, H // 2:, W // 2:] = 0.0
        y = x.clone()
        eps = 0.0 if kind == "identical_eps0" else eps
    elif kind == "inverse":               # y = 1 - x: u near 1
        x = r(B, Cc, H, W)
        y = 1.0 - x
    else:
        assert kind == "max_val"          # a non-default max_val (not a float32 value) and eps
        x, y = r(B, Cc, H, W) * 0.3, r(B, Cc, H, W) * 0.3
        mv, eps = 0.3, 1e-6
    return x.to(device), y.to(device), mv, eps


SSIM_KINDS = ("rgb", "depth", "far_depth", "identical", "identical_eps0", "inverse", "max_val")


def smooth_case(kind, B, Cc, H, W, device, seed):
    g = torch.Generator().manual_seed(seed)
    lo, hi = {"depth": (2.0, 6.0), "far_depth": (10.0, 100.0)}[kind]
    d = torch.rand(B, 1, H, W, generator=g) * (hi - lo) + lo
    d[:, :, H // 3:, W // 2:] = 0.5 * (lo + hi)                  # a flat run: sign(0) = 0 edges
    img = torch.floor(torch.rand(B, Cc, H, W, generator=g) * 256) / 255
    img[:, :, : H // 2, : W // 3] = 1.0                          # equal neighbours in every channel
    return d.to(device), img.to(device)


# ------------------------------------------------------------------------------------------------ checkers
def check_ssim_forward(impl, x, y, max_val, eps, what):
    """-> the kernel's coefficient maps (3,B,C,H,W).  Loss and every coefficient against float64."""
    B, Cc, H, W = x.shape
    loss = torch.full((1,), float("nan"), device=x.device)
    coef = torch.full((3 * B * Cc * H * W,), float("nan"), device=x.device, dtype=torch.float64)
    ws = torch.zeros(emu.LOSS_WS_FLOATS, device=x.device)
    impl.ssim_forward(x, y, max_val, eps, loss, coef, ws)
    assert ticket(ws) == 0, f"{what}: loss ticket not reset"
    r = emu.ssim64(x, y, float(f32(max_val)), float(f32(eps)))
    # where mean |clamp(u)| is not far above u's fp64 rounding allowance (identical images) the loss measures that
    # allowance, not the summation: those cases are reported apart
    u0 = float(r["loss"]) < 1e3 * float(r["du"].mean())
    measure(loss[0], r["loss"], r["loss_bound"], SSIM_LOSS_U0_TOL if u0 else SSIM_LOSS_TOL,
            "ssim loss, u ~ 0" if u0 else "ssim loss", what)
    cf = coef.view(3, B, Cc, H, W)
    bound = r["coef_bound"]
    err = (cf - r["coef"]).abs()
    u, du = r["u"], 4 * r["du"]
    near = ((u.abs() <= du) | ((1 - u).abs() <= du)) & ~r["exact"]
    either = torch.minimum((cf - r["coef_open"]).abs(), cf.abs())
    err = torch.where(near.expand_as(err), either, err)
    measure(err, torch.zeros_like(err), bound, COEF_TOL, "ssim coef", what)
    return cf


def check_ssim_backward(impl, x, y, coef, what):
    """g_img1 from the coefficient maps `coef` (3,B,C,H,W) against the float64 adjoint, at g_loss 1, 0, 3.7, 2^-100,
    written through x's strides without touching anything else."""
    flat = coef.reshape(-1).contiguous()
    ref, bound = emu.adjoint64(coef, x, y)
    outs = {}
    for gl in (1.0, 0.0, 3.7, 2.0 ** -100):
        gx, untouched = out_like(x)
        impl.ssim_backward(x, y, flat, scalar(gl, x.device), gx)
        assert untouched(), f"{what}: g_img1 written outside its strides"
        outs[gl] = gx
    measure(outs[1.0], ref, bound, GX_TOL, "ssim g_img1", what)
    assert not torch.isnan(outs[0.0]).any() and int(torch.count_nonzero(outs[0.0])) == 0, f"{what}: g_loss = 0"
    for s in (3.7, 2.0 ** -100):
        assert torch.equal(outs[s], outs[1.0] * scalar(s, x.device)), f"{what}: g_loss = {s} is not an exact scale"


def lattice_maps(B, Cc, H, W, device, offset=0):
    """One-hot maps on a lattice of spacing 11 (the adjoint's support is 11 wide, so every output element reads at most
    one non-zero): plane k puts ones at rows = a, columns = b mod 11, (a, b) = divmod(k + offset, 11) mod 11, so 121
    planes cover every position, the edges, the tile seams and the corners included; map m = k mod 3."""
    c = torch.zeros(3, B, Cc, H, W, dtype=torch.float64)
    for k in range(B * Cc):
        a, b = divmod((k + offset) % 121, 11)
        c[k % 3, k // Cc, k % Cc, a::11, b::11] = 1.0
    return c.to(device)


def check_smooth(impl, d, img, what, scales=True):
    B, Cc, H, W = img.shape
    loss = torch.full((1,), float("nan"), device=img.device)
    ws = torch.zeros(emu.LOSS_WS_FLOATS, device=img.device)
    impl.smooth_forward(d, img, loss, ws)
    assert ticket(ws) == 0, f"{what}: loss ticket not reset"
    r = emu.smooth64(d, img)
    measure(loss[0], r["loss"], r["loss_bound"], SM_LOSS_TOL, "smooth loss", what)
    one = scalar(1.0, img.device)
    gd, ud = out_like(d)
    gi, ui = out_like(img)
    impl.smooth_backward(d, img, one, gd, gi)
    assert ud() and ui(), f"{what}: gradient written outside its strides"
    measure(gd, r["g_d"], r["g_d_bound"], SM_GD_TOL, "smooth g_idepth", what)
    measure(gi, r["g_img"], r["g_img_bound"], SM_GI_TOL, "smooth g_image", what)
    gd2, _ = out_like(d)
    impl.smooth_backward(d, img, one, gd2, None)
    gi2, _ = out_like(img)
    impl.smooth_backward(d, img, one, None, gi2)
    assert torch.equal(gd2, gd) and torch.equal(gi2, gi), f"{what}: one gradient alone differs from both together"
    if scales:
        for s in (0.0, 3.7):
            gds, _ = out_like(d)
            gis, _ = out_like(img)
            impl.smooth_backward(d, img, scalar(s, img.device), gds, gis)
            sc = scalar(s, img.device)
            assert torch.equal(gds, gd * sc) and torch.equal(gis, gi * sc), f"{what}: g_loss = {s}"


def ssim_loss_call(impl, x, y, ws, coef=True):
    loss = torch.full((1,), float("nan"), device=x.device)
    cf = torch.full((3 * x.numel(),), float("nan"), device=x.device, dtype=torch.float64) if coef else None
    impl.ssim_forward(x, y, 1.0, 1e-12, loss, cf, ws)
    return (loss,) if cf is None else (loss, cf)


def smooth_loss_call(impl, d, img, ws):
    loss = torch.full((1,), float("nan"), device=img.device)
    impl.smooth_forward(d, img, loss, ws)
    return (loss,)


def check_scratch(impl, calls):
    """`calls`: functions of a scratch tensor returning tensors.  Run each alone on a fresh scratch, then all in turn on
    one scratch, twice: every result bit for bit the same, the ticket word 0 after every call."""
    fresh = lambda: torch.zeros(emu.LOSS_WS_FLOATS, device=impl.device)
    alone = [call(fresh()) for call in calls]
    ws = fresh()
    for rep in range(2):
        for k, call in enumerate(calls):
            got = call(ws)
            assert ticket(ws) == 0, f"call {k}: ticket {ticket(ws)} left in the scratch"
            assert all(torch.equal(a, b) for a, b in zip(got, alone[k])), f"call {k} (pass {rep}) differs from it alone"


def check_nonfinite(impl):
    """A NaN in img1 or img2 makes the SSIM loss NaN and the gradient NaN exactly where torch's is (the pixels whose
    windows reach it), the rest as float64; NaN / inf / -inf in the smoothness inputs give torch's NaN / inf pattern."""
    dev = impl.device
    g = torch.Generator().manual_seed(5)
    for which in ("x", "y"):
        x, y = torch.rand(2, 3, 20, 40, generator=g), torch.rand(2, 3, 20, 40, generator=g)
        (x if which == "x" else y)[1, 2, 7, 33] = float("nan")
        xd, yd = x.to(dev), y.to(dev)
        loss = torch.full((1,), 0.0, device=dev)
        coef = torch.zeros(3 * x.numel(), device=dev, dtype=torch.float64)
        impl.ssim_forward(xd, yd, 1.0, 1e-12, loss, coef, torch.zeros(emu.LOSS_WS_FLOATS, device=dev))
        assert torch.isnan(loss).all(), f"NaN in img{1 if which == 'x' else 2}: SSIM loss {float(loss[0])} is not NaN"
        gx = torch.zeros_like(xd)
        impl.ssim_backward(xd, yd, coef, scalar(1.0, dev), gx)
        xr = x.double().requires_grad_(True)
        (want,) = torch.autograd.grad(plo.ssim_loss(xr, y.double(), 11), xr)
        gx = gx.cpu()
        assert torch.equal(torch.isnan(gx), torch.isnan(want)), f"NaN in {which}: NaN pattern of g_img1 differs from torch"
        fin = ~torch.isnan(want)
        assert float((gx.double() - want)[fin].abs().max()) <= 1e-6 * float(want[fin].abs().max())
    for bad in (float("nan"), float("inf"), -float("inf")):
        for where in ("d", "img", "both"):
            d, img = torch.rand(2, 1, 9, 12, generator=g) * 4 + 2, torch.rand(2, 3, 9, 12, generator=g)
            if where in ("d", "both"):
                d[1, 0, 4, 5] = bad; d[0, 0, 0, 0] = bad; d[0, 0, 0, 1] = bad
            if where in ("img", "both"):
                img[0, 2, 3, 3] = bad; img[1, 0, 8, 11] = bad; img[1, 1, 8, 10] = bad
            loss = torch.zeros(1, device=dev)
            impl.smooth_forward(d.to(dev), img.to(dev), loss, torch.zeros(emu.LOSS_WS_FLOATS, device=dev))
            gd, gi = torch.zeros(d.shape, device=dev), torch.zeros(img.shape, device=dev)
            impl.smooth_backward(d.to(dev), img.to(dev), scalar(1.0, dev), gd, gi)
            r = emu.smooth64(d, img)
            for got, want, name in ((loss.cpu()[0], r["loss"], "loss"), (gd.cpu(), r["g_d"], "g_idepth"),
                                    (gi.cpu(), r["g_img"], "g_image")):
                got = got.double()
                same = torch.equal(torch.isnan(got), torch.isnan(want)) and torch.equal(got.isinf(), want.isinf())
                fin = torch.isfinite(want)
                assert same and bool(((got - want)[fin].abs() <= 1e-5 * (1 + want[fin].abs())).all()), \
                    f"smoothness with {bad} in {where}: {name} differs from torch"


def check_max_val_rounding():
    """The C ABI takes max_val as float32; kornia forms C1, C2 from the Python double.  -> for max_val = 0.3, what
    rounding it to float32 moves, each in this module's measure: the loss (relative), the coefficient maps and the
    gradient (CPU, float64)."""
    x, y, _, _ = ssim_case("max_val", 2, 3, 32, 40, "cpu", 3)
    a, b = emu.ssim64(x, y, 0.3), emu.ssim64(x, y, float(f32(0.3)))
    ga, bound = emu.adjoint64(a["coef"], x, y)
    gb, _ = emu.adjoint64(b["coef"], x, y)
    return (abs(float(a["loss"] - b["loss"])) / float(a["loss"]), float(((a["coef"] - b["coef"]).abs() / a["coef_bound"]).max()),
            float(((ga - gb).abs() / bound).max()))


# ------------------------------------------------------------------------------------------------ the tests
def _bc(k):
    return BC[k % len(BC)]


@pytest.mark.parametrize("hw", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_ssim_forward_and_backward_every_shape(lib, hw):
    """Every input kind at this H x W, the layouts in turn; the backward from the kernel's own coefficient maps."""
    H, W = hw
    for k, kind in enumerate(SSIM_KINDS):
        B, Cc = _bc(H + W + k)
        x, y, mv, eps = ssim_case(kind, B, Cc, H, W, lib.device, 100 * H + W + k)
        lay = LAYOUTS[(H + k) % len(LAYOUTS)]
        x = place(x, lay if lay != "expand" else "nchw")
        y = place(y, lay)
        what = f"ssim {kind} {B}x{Cc}x{H}x{W} {lay}"
        coef = check_ssim_forward(lib, x, y, mv, eps, what)
        check_ssim_backward(lib, x, y, coef, what)


@pytest.mark.parametrize("hw", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_ssim_backward_injected_maps(lib, hw):
    """Random maps, a different one per plane, and one-hot lattices covering every position of 121 planes."""
    H, W = hw
    g = torch.Generator().manual_seed(H * 100 + W)
    B, Cc = _bc(H * W)
    x, y = (torch.rand(B, Cc, H, W, generator=g).to(lib.device) for _ in range(2))
    rnd = torch.randn(3, B, Cc, H, W, generator=g, dtype=torch.float64).to(lib.device) * 1e-4
    check_ssim_backward(lib, place(x, LAYOUTS[H % 4]), y, rnd, f"random maps {B}x{Cc}x{H}x{W}")
    x, y = (torch.rand(121, 1, H, W, generator=g).to(lib.device) for _ in range(2))
    check_ssim_backward(lib, x, y, lattice_maps(121, 1, H, W, lib.device), f"one-hot lattice 121x1x{H}x{W}")
    x, y = (torch.rand(41, 3, H, W, generator=g).to(lib.device) for _ in range(2))
    check_ssim_backward(lib, place(x, "channels_last"), y, lattice_maps(41, 3, H, W, lib.device, 7),
                        f"one-hot lattice 41x3x{H}x{W}")


def test_ssim_depth_target_with_warp_holes(lib):
    """SSIM of a depth patch against a forward-warped depth label, zero where nothing landed (losses.py:105)."""
    from sinnerf_b200.warp import forward_warp
    from tests.warp_scenes import proj, random_poses, scene
    for H, W in ((64, 64), (63, 84)):
        image, depth = scene(H, W, seed=H + W, holes=0.05)
        _, wd, hit = forward_warp(torch.from_numpy(image).to(lib.device), torch.from_numpy(depth).to(lib.device),
                                  proj(H, W), random_poses(H, W, 2, seed=W))
        assert not bool(hit.all())
        x = torch.from_numpy(depth).to(lib.device).expand(2, 1, H, W).contiguous()
        y = wd[:, None]
        what = f"ssim warped depth label 2x1x{H}x{W}"
        coef = check_ssim_forward(lib, x, y, 1.0, 1e-12, what)
        check_ssim_backward(lib, x, y, coef, what)


def past_ssim_caps(impl):
    cap = max(emu.MAX_LOSS_BLOCKS, 8 * impl.sm_count)
    B = -(-(cap + cap // 4) // (3 * 16 * 8))
    n = emu.ssim_tiles(B, 3, 256, 256)
    assert emu.ssim_fwd_grid(n) < n and emu.ssim_bwd_grid(n, impl.sm_count) < n, (n, impl.sm_count)
    return B, 3, 256, 256


def past_smooth_caps(impl):
    cap = max(emu.MAX_LOSS_BLOCKS, 16 * impl.sm_count) * emu.THREADS
    side = math.isqrt(cap + cap // 5) + 1
    n = side * side
    assert emu.smooth_fwd_grid(n) * emu.THREADS < n and emu.smooth_bwd_grid(n, impl.sm_count) * emu.THREADS < n
    return 1, 3, side, side


def test_ssim_past_the_launch_caps(lib):
    B, Cc, H, W = past_ssim_caps(lib)
    x, y, mv, eps = ssim_case("rgb", B, Cc, H, W, lib.device, 1)
    coef = check_ssim_forward(lib, x, y, mv, eps, f"ssim past the caps {B}x{Cc}x{H}x{W}")
    check_ssim_backward(lib, x, y, coef, f"ssim past the caps {B}x{Cc}x{H}x{W}")


@pytest.mark.parametrize("hw", SHAPES[:13] + ((2, 2), (2, 9), (9, 2)), ids=lambda s: f"{s[0]}x{s[1]}")
def test_smoothness_every_shape(lib, hw):
    H, W = hw
    for k, kind in enumerate(("depth", "far_depth")):
        B, Cc = _bc(H + W + k)
        d, img = smooth_case(kind, B, Cc, H, W, lib.device, 10 * H + W + k)
        lay = LAYOUTS[(H + k) % 4]
        check_smooth(lib, place(d, lay), place(img, LAYOUTS[(H + k + 1) % 4]), f"smooth {kind} {B}x{Cc}x{H}x{W} {lay}")


def test_smoothness_past_the_launch_caps(lib):
    B, Cc, H, W = past_smooth_caps(lib)
    d, img = smooth_case("depth", B, Cc, H, W, lib.device, 2)
    check_smooth(lib, d, place(img, "rays"), f"smooth past the caps {B}x{Cc}x{H}x{W}", scales=False)


def test_shared_scratch_protocol(lib):
    from tests import test_gpu_ray_stages as rst
    rays_lib = rst.Lib()
    dev = lib.device
    x1, y1, _, _ = ssim_case("rgb", 1, 3, 64, 64, dev, 4)
    x2, y2, _, _ = ssim_case("rgb", *past_ssim_caps(lib), dev, 5)
    d1, i1 = smooth_case("depth", 1, 3, 64, 64, dev, 6)
    d2, i2 = smooth_case("depth", *past_smooth_caps(lib), dev, 7)

    def composite(n, S):
        sc = rst.scene(n, S, 3, dev)
        spec = dict(trgb=sc["trgb"], tdepth=sc["tdepth"], wr0=1.0 / (3 * n), wd0=1.0 / n)
        return lambda ws: rays_lib.composite_forward_loss(sc["raw"], sc["z"], sc["rays"], sc["noise"], 0.7, True, spec, ws)

    check_scratch(lib, [lambda ws: ssim_loss_call(lib, x1, y1, ws), lambda ws: smooth_loss_call(lib, d2, i2, ws),
                        composite(rst.past_cap(rays_lib, 64), 64), lambda ws: ssim_loss_call(lib, x2, y2, ws),
                        lambda ws: smooth_loss_call(lib, d1, i1, ws), composite(77, 64),
                        lambda ws: ssim_loss_call(lib, x1, y1, ws, coef=False)])


def test_non_finite_inputs(lib):
    check_nonfinite(lib)


def test_max_val_is_taken_as_float32(lib):
    """The kernel is compared against C1, C2 formed from float32(max_val) above.  Against kornia's double max_val = 0.3
    that costs 4.5e-10 of the loss and 8.7e-10 of the gradient's bound (under its one fp32 rounding, 6e-8), but 1.6e-10
    of the coefficient maps' bound, far above COEF_TOL: so the comparison must use the float32 value."""
    dl, dc, dg = check_max_val_rounding()
    print(f"max_val 0.3 as float32: loss {dl:.1e} relative, coefficients {dc:.1e}, gradient {dg:.1e} of their bounds")
    assert dl < 1e-9 and dg < 1e-8 and dc > COEF_TOL
    x, y, _, _ = ssim_case("max_val", 1, 3, 32, 32, lib.device, 3)
    loss = torch.full((1,), float("nan"), device=lib.device)
    lib.ssim_forward(x, y, 0.3, 1e-6, loss, None, torch.zeros(emu.LOSS_WS_FLOATS, device=lib.device))
    want = float(emu.ssim64(x, y, 0.3, float(f32(1e-6)))["loss"])
    assert abs(float(loss[0]) - want) <= SSIM_LOSS_TOL * want
