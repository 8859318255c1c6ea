"""The ray kernels of sinnerf_b200/csrc/ray_kernels.cu, stage by stage through the C ABI: inverse-CDF sampling and
the sorted merge bit for bit against the float32 emulation of tests/ray_emulation.py, compositing forward / backward
and the fused losses per element against float64 on the same float32 inputs.

Measure for the continuous outputs: |got - float64| of every element divided by what bounds that element
  weights: 1        rgb: sum_i T_i |c_i| (+ 1 + sum T with white_back)        depth: sum_i T_i |z_i|
  g_raw:   the float64 sum of absolute values of the terms of its closed form (ray_emulation.g_raw_bound64)
(T_i, not w_i = alpha_i T_i, in the sums: alpha = 1 - exp(-x) is rounded to an ulp of 1 however small alpha is, so a
ray of faint samples has errors of 2^-24 T_i per sample, which sum_i w_i |c_i| does not bound)
and the maximum is taken per element, so a kernel that is wrong in one sample slot of each ray (last sample, first
sample of a quad, first sample after a 32-sample step) fails whatever the other slots hold; a failure names the ray
and the slot.  Whole-tensor rel-L2, which tests/test_gpu_parity.py and tests/test_gpu_backward.py use, moves by less
than their bars when such a slot carries little weight.

The checkers are functions of an implementation (an object with ray_emulation.StandIn's methods).  Here it is the
library (`Lib`); tests/test_ray_emulation_cpu.py runs the same checkers on the CPU stand-in, faithful and with one
planted defect at a time, so every checker below is known to pass on a correct implementation and to fail on the
defect it is there for.

Bounds: each sits about 10x above the largest value these tests measured on an NVIDIA H100 80GB HBM3 at its 700 W power
limit, written beside it.  The bitwise cases carry no tolerance.

tests/test_gpu_parity.py::test_sample_pdf_known_answers_and_golden allows up to 8 samples a whole bin away from the
reference's fixture.  That fixture was produced with torch's serial cumsum, whose cdf differs from the kernel's
scan-ordered cdf by an ulp at some knots, so against THAT reference a count is the best one can assert.  Here the
reference is the kernel's own order of additions, nothing is allowed to differ, and `check_sample_pdf` adds the
properties that do not depend on the emulation.  The two tests answer different questions and both stay.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import ray_emulation as emu

pytestmark = pytest.mark.gpu

f32 = np.float32
W_TOL = 2e-6        # weights, normalised by 1            (measured 1.2e-7; 3.4e-7 with the degenerate samples)
RGB_TOL = 5e-6      # rgb / its bound                     (measured 4.5e-7)
DEPTH_TOL = 2e-6    # depth / its bound                   (measured 1.3e-7)
GRAW_TOL = 2e-3     # g_raw / its closed-form bound       (measured 1.9e-4; 2.0e-6 when only the losses drive it).  The
#                     bound ignores the 1 / t_i amplification of the rounding of t_i = 1 - alpha_i + 1e-10, which the
#                     scenes keep below e^4
LOSS_TOL = 1e-6     # loss sums / sum of |terms|          (measured 9.7e-8)
PDF_TOL = 300.0       # samples away from cdf knots vs float64, in units of 2^-24 (widest bin + own bin / cdf step): the
#                     cdf is rounded to an ulp of 1 and divided by the bin's cdf step  (measured 30)
FLOOR = 1e-30       # added to every bound: elements whose bound underflows float32 are compared absolutely
MEASURED = {}       # largest error / bound seen per quantity (the first word of `what`), for the figures above

S_ALL = (2, 3, 4, 8, 28, 32, 36, 60, 64, 68, 96, 100, 124, 128, 132, 192, 256)


# ------------------------------------------------------------------------------------------------ the library
class Lib:
    """ray_emulation.StandIn's interface on the C ABI; tensors live on cuda:0."""
    device = "cuda:0"

    def __init__(self):
        from sinnerf_b200 import _lib
        self._lib, self.lib = _lib, _lib.load()
        sm = C.c_int(0)
        assert self.lib.snb_device_check(C.byref(sm), None, None) == 0, self.lib.snb_last_error()
        self.sm_count = sm.value

    def _ok(self, rc):
        assert rc == 0, self.lib.snb_last_error()
        torch.cuda.synchronize()

    def _spec(self, loss):
        p = self._lib.ptr
        return self._lib.SnbLossSpec(p(loss.get("trgb")), p(loss.get("tdepth")), p(loss.get("wr")), p(loss.get("wd")),
                                     float(loss.get("wr0", 0.0)), float(loss.get("wd0", 0.0)))

    def composite_forward(self, raw, raw_channels, z, rays, noise, noise_std, white_back, want_maps=True, w_out=None):
        p, (n, S) = self._lib.ptr, z.shape
        w = torch.empty_like(z) if w_out is None else w_out
        rgb = torch.empty(n, 3, device=z.device) if want_maps else None
        depth = torch.empty(n, device=z.device) if want_maps else None
        self._ok(self.lib.snb_composite_forward(p(raw), raw_channels, p(z), p(rays), p(noise), noise_std, int(white_back),
                                                n, S, p(rgb), p(depth), p(w), None))
        return rgb, depth, w

    def composite_forward_loss(self, raw, z, rays, noise, noise_std, white_back, loss, ws):
        p, (n, S) = self._lib.ptr, z.shape
        w, rgb, depth = torch.empty_like(z), torch.empty(n, 3, device=z.device), torch.empty(n, device=z.device)
        out = torch.full((2,), float("nan"), device=z.device)
        spec = self._spec(loss)
        self._ok(self.lib.snb_composite_forward_loss(p(raw), p(z), p(rays), p(noise), noise_std, int(white_back), n, S,
                                                     C.byref(spec), p(rgb), p(depth), p(w), p(out), p(ws), None))
        return rgb, depth, w, out

    def composite_backward(self, raw, raw_channels, z, rays, noise, noise_std, white_back, g_rgb, g_depth, g_w,
                           loss=None, out_rgb=None, out_depth=None, g_loss=None, amax=None, g_raw_out=None):
        p, (n, S) = self._lib.ptr, z.shape
        g_raw = torch.empty_like(raw) if g_raw_out is None else g_raw_out
        if raw_channels == 1:
            self._ok(self.lib.snb_composite_backward_weights(p(raw), p(z), p(rays), p(noise), noise_std, p(g_w), n, S,
                                                             p(g_raw), p(amax), None))
        elif loss is None and amax is None:
            self._ok(self.lib.snb_composite_backward(p(raw), p(z), p(rays), p(noise), noise_std, int(white_back),
                                                     p(g_rgb), p(g_depth), p(g_w), n, S, p(g_raw), None))
        else:
            spec = None if loss is None else self._spec(loss)
            self._ok(self.lib.snb_composite_backward_loss(
                p(raw), p(z), p(rays), p(noise), noise_std, int(white_back), p(g_rgb), p(g_depth), p(g_w),
                None if spec is None else C.byref(spec), p(out_rgb), p(out_depth), p(g_loss), n, S, p(g_raw), p(amax), None))
        return g_raw

    def sample_pdf(self, bins, weights, u, eps=1e-5):
        p, n, m = self._lib.ptr, weights.shape[0], weights.shape[1]
        assert bins.stride(1) == 1 and weights.stride(1) == 1 and u.is_contiguous()
        out = torch.full((n, u.shape[-1]), float("nan"), device=bins.device)
        self._ok(self.lib.snb_sample_pdf(p(bins), bins.stride(0), p(weights), weights.stride(0), p(u),
                                         0 if u.dim() == 1 else u.shape[1], n, m, u.shape[-1], eps, p(out), None))
        return out

    def importance_merge(self, z, w, u, eps=1e-5, want_new=True, sentinel=-7.0):
        p, (n, S), ni = self._lib.ptr, z.shape, u.shape[-1]
        fine = torch.full((n, S + ni), sentinel, device=z.device)
        new = torch.full((n, ni), sentinel, device=z.device) if want_new else None
        self._ok(self.lib.snb_importance_merge(p(z), p(w), p(u), 0 if u.dim() == 1 else ni, n, S, ni, eps, p(fine), p(new),
                                               None))
        return fine, new


@pytest.fixture(scope="module")
def lib():
    return Lib()


# ------------------------------------------------------------------------------------------------ scenes and measures
def scene(n, S, seed, device, optical_depth=12.0, soft_last=True):
    """Seeded rays with sorted depths in [2, 6], colours in [0, 1] and densities of both signs scaled so that
    sigma_i delta_i stays below min(4, optical_depth / S): no sample but the last saturates, t_i >= e^-4 before it."""
    # soft_last=False keeps the huge density gradients of unsaturated last samples (delta = 1e10 |d|) out of the scene
    g = torch.Generator().manual_seed(seed)
    rays = torch.randn(n, 8, generator=g)
    z = torch.sort(torch.rand(n, S, generator=g) * 4 + 2, -1)[0]
    dn = rays[:, 3:6].norm(dim=1, keepdim=True)
    gaps = z[:, 1:] - z[:, :-1]                                           # the last sample gets an ordinary density, so its
    delta = torch.cat([gaps, gaps.mean(1, keepdim=True)], 1) * dn         # 1e10 delta saturates it as in a real scene;
    if soft_last:                                                         # on odd rays it is faint enough not to
        delta[1::2, -1] = 1e10 * dn[1::2, 0]
    x = torch.rand(n, S, generator=g) * min(4.0, optical_depth / S)
    x = torch.where(torch.rand(n, S, generator=g) < 0.25, -x, x)          # a quarter of the samples are empty space
    raw = torch.cat([torch.rand(n, S, 3, generator=g), (x / delta.clamp_min(1e-6))[..., None]], -1)
    noise = torch.randn(n, S, generator=g)
    mk = lambda *s: torch.randn(*s, generator=g)
    d = dict(rays=rays, z=z, raw=raw, noise=noise, g_rgb=mk(n, 3), g_depth=mk(n), g_w=mk(n, S),
             trgb=torch.rand(n, 3, generator=g), tdepth=torch.rand(n, generator=g) * 4 + 2)
    return {k: v.to(device).contiguous() for k, v in d.items()}


def worst(got, want, bound, tol, what):
    """max over elements of |got - want| / (bound + FLOOR) <= tol, naming the ray and slot of the worst element."""
    err = (got.double() - want).abs() / (bound + FLOOR)
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    flat = int(err.argmax())
    idx = np.unravel_index(flat, tuple(err.shape)) if err.dim() else ()
    m = float(err.reshape(-1)[flat])
    MEASURED[what.split(" S=")[0]] = max(MEASURED.get(what.split(" S=")[0], 0.0), m)
    assert m <= tol, f"{what}: error / bound = {m:.3e} > {tol:.1e} at (ray, slot, ...) = {tuple(int(i) for i in idx)}"
    return m


def noise_args(sc, mode):
    return {"none": (None, 0.0), "zero_std": (sc["noise"], 0.0), "std": (sc["noise"], 0.7)}[mode]


def offset_view(t):
    """The same values one float past a 16-byte boundary (a slice of a larger buffer)."""
    buf = torch.empty(t.numel() + 5, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4
    return v


def ray_counts(impl, S, quad):
    L = 8 if S <= 32 else (16 if S <= 64 else 32)
    rpw = 32 // L if quad else 1
    return sorted({1, max(1, 8 * rpw - 1), 77})


def past_cap(impl, S):
    L = 8 if S <= 32 else (16 if S <= 64 else 32)
    rpw = 32 // L if (S % 4 == 0 and 4 <= S <= 128) else 1
    return 2 * 8 * 8 * impl.sm_count * rpw + 13


# ------------------------------------------------------------------------------------------------ checkers
CONFIGS = (  # raw_channels, white_back, noise, gradient left NULL
    (4, False, "none", None), (4, True, "std", "g_w"), (4, False, "zero_std", "g_rgb"), (4, True, "std", "g_depth"),
    (1, False, "std", None), (1, False, "none", None))


def check_composite(impl, S, n, cfg, seed=0, sc=None, views=()):
    """Forward and backward of one call against float64; `views`: names of tensors passed one float off alignment."""
    ch, wb, nmode, drop = cfg
    sc = scene(n, S, 1000 * S + seed, impl.device) if sc is None else sc
    noise, nstd = noise_args(sc, nmode)
    raw = sc["raw"] if ch == 4 else sc["raw"][..., 3].contiguous()
    z, rays = sc["z"], sc["rays"]
    g_rgb = None if (ch == 1 or drop == "g_rgb") else sc["g_rgb"]
    g_depth = None if (ch == 1 or drop == "g_depth") else sc["g_depth"]
    g_w = None if drop == "g_w" else sc["g_w"]
    w_out = g_raw_out = None
    if "z" in views: z = offset_view(z)
    if "noise" in views and noise is not None: noise = offset_view(noise)
    if "g_w" in views and g_w is not None: g_w = offset_view(g_w)
    if "raw" in views: raw = offset_view(raw); assert ch == 1
    if "w" in views: w_out = offset_view(torch.zeros_like(sc["z"]))
    if "g_raw" in views: g_raw_out = offset_view(torch.zeros_like(raw)); assert ch == 1
    kw = {} if w_out is None else {"w_out": w_out}
    rgb, depth, w = impl.composite_forward(raw, ch, z, rays, noise, nstd, wb, want_maps=(ch == 4), **kw)
    kw = {} if g_raw_out is None else {"g_raw_out": g_raw_out}
    g_raw = impl.composite_backward(raw, ch, z, rays, noise, nstd, wb, g_rgb, g_depth, g_w, **kw)

    raw64 = raw.detach().double().requires_grad_(True)
    c = emu.composite64(raw64, z, rays[:, 3:6].double().norm(dim=1), noise if nstd != 0 else None, nstd, wb)
    zero = lambda t, like: torch.zeros_like(like) if t is None else t.double()
    G = (zero(g_rgb, c["depth"][:, None].expand(-1, 3)), zero(g_depth, c["depth"]), zero(g_w, c["weights"]))
    obj = (G[2] * c["weights"]).sum() + (G[1] * c["depth"]).sum()
    if ch == 4:
        obj = obj + (G[0] * c["rgb"]).sum()
    want_g, = torch.autograd.grad(obj, raw64)
    c = {k: v.detach() for k, v in c.items()}
    res = {"w": worst(w, c["weights"], torch.ones_like(c["weights"]), W_TOL, f"weights S={S} n={n} {cfg}")}
    if ch == 4:
        res["rgb"] = worst(rgb, c["rgb"], c["rgb_bound"], RGB_TOL, f"rgb S={S} n={n} {cfg}")
        res["depth"] = worst(depth, c["depth"], c["depth_bound"], DEPTH_TOL, f"depth S={S} n={n} {cfg}")
    bound = emu.g_raw_bound64(c, raw64.detach(), z, wb, *G)
    res["g_raw"] = worst(g_raw, want_g, bound, GRAW_TOL, f"g_raw S={S} n={n} {cfg}")
    res["out"] = (rgb, depth, w, g_raw)
    return res


def check_offset_views(impl, S=64, n=37):
    """An offset per-sample pointer must select the warp-per-ray kernels: same bounds, and the first sample of every ray
    (T = 1, so w_0 = alpha_0, the element-wise arithmetic the two mappings share) bit for bit as the aligned call."""
    for cfg, names in ((CONFIGS[1], ("z", "noise", "w")), (CONFIGS[3], ("z", "noise", "w")),
                       ((4, False, "std", None), ("g_w",)), (CONFIGS[4], ("z", "noise", "w", "g_w", "raw", "g_raw"))):
        sc = scene(n, S, 77, impl.device)
        base = check_composite(impl, S, n, cfg, sc=sc)["out"]
        for name in names:
            got = check_composite(impl, S, n, cfg, sc=sc, views=(name,))["out"]
            assert torch.equal(got[2][:, 0], base[2][:, 0]), f"{name} offset: w[:, 0] differs in bits ({cfg})"
            assert (got[2] - base[2]).abs().max() <= 2 * W_TOL


def check_degenerate(impl, S=64, n=24):
    """Special samples inside ordinary rays.  Forward against float64 (weights are bounded by 1 whatever happens to
    alpha); backward: finite everywhere and exactly zero wherever sigma + noise <= 0 (the [s > 0] gate)."""
    for quad in (True, False):
        S_ = S if quad else S + 3
        sc = scene(n, S_, 5, impl.device)
        raw, z, rays = sc["raw"].clone(), sc["z"].clone(), sc["rays"].clone()
        z[0, 10] = z[0, 11]; z[0, 4:8] = z[0, 4]                       # coincident depths: delta = 0
        dn1 = float(rays[1, 3:6].norm())
        raw[1, 7, 3] = 20.0 / (dn1 * float(z[1, 8] - z[1, 7]))        # exp(-20) < 2^-25: alpha rounds to 1, t is the bare 1e-10
        raw[2, 3:9, 3] = 1e6                                          # six of them: the carried product underflows
        raw[2, 31:35, 3] = 1e6
        raw[3, :, 3] = 0.0                                            # sigma exactly 0 everywhere
        raw[4, ::2, 3] = -raw[4, ::2, 3].abs() - 1.0                  # negative
        raw[5, :, 3] = -0.7 * sc["noise"][5] + 1e-3 * torch.randn(S_, device=raw.device)   # sigma + noise crosses zero
        rays[6, 3:6] = 0.0                                            # zero direction: dnorm = 0
        raw[7, :, 3] = raw[7, :, 3].abs() * 1e-2
        z[7] = torch.flip(z[7], [0])                                  # descending depths: negative delta, alpha < 0
        for wb in (False, True):
            rgb, depth, w = impl.composite_forward(raw, 4, z, rays, sc["noise"], 0.7, wb)
            c = emu.composite64(raw, z, rays[:, 3:6].double().norm(dim=1), sc["noise"], 0.7, wb)
            # descending depths make alpha negative and T > 1: those weights are bounded by T, not by 1
            worst(w, c["weights"], c["T"].clamp_min(1.0), W_TOL, f"degenerate weights S={S_} wb={wb}")
            worst(rgb, c["rgb"], c["rgb_bound"], RGB_TOL, f"degenerate rgb S={S_} wb={wb}")
            worst(depth, c["depth"], c["depth_bound"], DEPTH_TOL, f"degenerate depth S={S_} wb={wb}")
            assert float(w[6].abs().max()) == 0.0                        # delta = 0 everywhere: nothing absorbs
            g = impl.composite_backward(raw, 4, z, rays, sc["noise"], 0.7, wb, sc["g_rgb"], sc["g_depth"], sc["g_w"])
            assert torch.isfinite(g).all()
            s = raw[..., 3] + sc["noise"] * np.float32(0.7)
            assert float(g[..., 3][s <= 0].abs().max()) == 0.0, "g_sigma is not gated by [sigma + noise > 0]"
            assert float(g[6, :, 3].abs().max()) == 0.0                  # delta = 0: no density gradient
            assert torch.equal(g[..., :3], sc["g_rgb"][:, None, :] * w[..., None])


def loss_spec(sc, mode, n, device):
    """rgb+depth with scalar weights / per-ray weights (zeros and negatives among them) / one term only."""
    g = torch.Generator().manual_seed(n)
    wr = (torch.randn(n, generator=g) * 0.1).to(device)
    wd = (torch.randn(n, generator=g) * 0.1).to(device)
    wr[::5] = 0.0; wd[1::5] = 0.0
    full = dict(trgb=sc["trgb"], tdepth=sc["tdepth"], wr0=1.0 / (3 * n), wd0=1.0 / n)
    return {"scalar": full, "per_ray": dict(full, wr=wr, wd=wd), "rgb_only": dict(trgb=sc["trgb"], wr0=0.25),
            "depth_only": dict(tdepth=sc["tdepth"], wd=wd)}[mode]


def check_losses(impl, S, n, mode, g_loss=None, wb=True):
    """snb_composite_forward_loss / snb_composite_backward_loss: loss values against float64 sums over the call's own
    rgb / depth, g_raw against float64 autograd through composite64 and losses64, twice on one workspace."""
    sc = scene(n, S, 31 * S + n, impl.device)
    ws = torch.zeros(4096, device=impl.device)
    first = impl.composite_forward(sc["raw"], 4, sc["z"], sc["rays"], sc["noise"], 0.7, wb)
    # targets placed so that |depth - target| straddles 1, and equals it on rays 0 and 1 (in float32, both signs)
    k = torch.arange(n, device=impl.device)
    sc["tdepth"] = first[1] + torch.tensor([-1.0, 1.0, 0.5, -0.5, 1.5, -1.5, 0.999999, -1.000001], device=impl.device)[k % 8]
    spec = loss_spec(sc, mode, n, impl.device)
    wr = spec.get("wr", spec.get("wr0", 0.0)); wd = spec.get("wd", spec.get("wd0", 0.0))
    runs = [impl.composite_forward_loss(sc["raw"], sc["z"], sc["rays"], sc["noise"], 0.7, wb, spec, ws) for _ in range(2)]
    rgb, depth, w, loss = runs[0]
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1])), "second call on the same workspace differs"
    assert all(torch.equal(a, b) for a, b in zip(first, runs[0][:3])), "the loss changes the rendered outputs"
    assert int(ws.view(torch.int32)[0]) == 0, "ticket not reset"
    l0, l1 = emu.losses64(rgb, depth, spec.get("trgb"), spec.get("tdepth"), wr, wd)
    a0, a1 = emu.losses64(rgb, depth, spec.get("trgb"), spec.get("tdepth"), torch.as_tensor(wr).abs(), torch.as_tensor(wd).abs())
    m = max(worst(loss[0], l0, a0, LOSS_TOL, f"loss[0] S={S} n={n} {mode}"), worst(loss[1], l1, a1, LOSS_TOL, f"loss[1] S={S} n={n} {mode}"))
    # backward: only the loss drives it, plus an explicit g_depth so both sources are summed
    gl = None if g_loss is None else torch.tensor(g_loss, device=impl.device)
    amax = torch.zeros(1, device=impl.device)
    g_raw = impl.composite_backward(sc["raw"], 4, sc["z"], sc["rays"], sc["noise"], 0.7, wb, None, sc["g_depth"], None,
                                    loss=spec, out_rgb=rgb, out_depth=depth, g_loss=gl, amax=amax)
    raw64 = sc["raw"].double().requires_grad_(True)
    c = emu.composite64(raw64, sc["z"], sc["rays"][:, 3:6].double().norm(dim=1), sc["noise"], 0.7, wb)
    glv = (1.0, 1.0) if g_loss is None else g_loss
    # the derivative is taken at the float32 rgb / depth the forward wrote (that is what the kernel is given)
    rgb_l, dep_l = rgb.double().requires_grad_(True), depth.double().requires_grad_(True)
    q0, q1 = emu.losses64(rgb_l, dep_l, spec.get("trgb"), spec.get("tdepth"), wr, wd)
    gr, gd = torch.autograd.grad(float(f32(glv[0])) * q0 + float(f32(glv[1])) * q1, (rgb_l, dep_l), allow_unused=True)
    gr = torch.zeros_like(rgb_l) if gr is None else gr
    gd = (torch.zeros_like(dep_l) if gd is None else gd) + sc["g_depth"].double()
    want, = torch.autograd.grad((gr * c["rgb"]).sum() + (gd * c["depth"]).sum(), raw64)
    c = {k_: v.detach() for k_, v in c.items()}
    bound = emu.g_raw_bound64(c, sc["raw"], sc["z"], wb, gr, gd, torch.zeros_like(c["weights"]))
    mg = worst(g_raw, want, bound, GRAW_TOL, f"loss g_raw S={S} n={n} {mode}")
    assert amax.view(torch.int32).item() == g_raw.abs().max().view(torch.int32).item(), "g_amax != max |g_raw|"
    return m, mg


def check_amax(impl, S, n):
    """g_amax, rgb form and sigma-only form: the bit pattern of max |g_raw| of what the call wrote; only ever raised;
    zero for a zero gradient; 3.0e38 for an infinite one; a NaN gradient is skipped (fmaxf drops it), so the word holds
    the maximum over the other elements."""
    sc = scene(n, S, 9 * S + n, impl.device, soft_last=False)
    bits = lambda t: int(t.view(torch.int32).item())
    for ch in (4, 1):
        raw = sc["raw"] if ch == 4 else sc["raw"][..., 3].contiguous()
        kw = dict(g_rgb=sc["g_rgb"] * 50, g_depth=None, g_w=sc["g_w"] * 1e-3) if ch == 4 else dict(g_rgb=None, g_depth=None, g_w=sc["g_w"])
        run = lambda amax, **over: impl.composite_backward(raw, ch, sc["z"], sc["rays"], sc["noise"], 0.7, False,
                                                           **{**kw, **over}, amax=amax)
        amax = torch.zeros(1, device=impl.device)
        g = run(amax)
        assert bits(amax) == bits(g.abs().max()), f"g_amax != max |g_raw| (channels {ch}, S={S}, n={n})"
        big = bits(amax)
        g = run(amax, g_w=kw["g_w"] * 1e-3, g_rgb=None)
        assert bits(amax) == big and bits(g.abs().max()) < big, "a smaller gradient lowered g_amax"
        amax.fill_(1e-30)
        run(amax)
        assert bits(amax) == big
        amax.zero_()
        g = run(amax, g_w=torch.zeros_like(sc["g_w"]), g_rgb=None)
        assert float(g.abs().max()) == 0.0 and bits(amax) == 0, "zero gradient must leave g_amax zero"
        s_ = sc["raw"][n // 2, :, 3] + sc["noise"][n // 2] * np.float32(0.7)
        gw = kw["g_w"].clone(); gw[n // 2, int(torch.nonzero(s_ > 0)[1])] = float("inf")    # on the second sample that absorbs: inf * alpha stays
        #                         inf and reaches the first through the suffix sum (at its own sample the warp-per-ray kernel forms inf - inf)
        amax.zero_()
        g = run(amax, g_w=gw)
        assert torch.isinf(g).any() or torch.isnan(g).any()
        assert bits(amax) == int(np.float32(3.0e38).view(np.int32)), "an infinite gradient must saturate g_amax"
    # NaN: a NaN upstream gradient poisons the samples of its ray up to its own and nothing else
    gw = sc["g_w"].clone()
    gw[0, S // 2] = float("nan")
    amax = torch.zeros(1, device=impl.device)
    g = impl.composite_backward(sc["raw"][..., 3].contiguous(), 1, sc["z"], sc["rays"], None, 0.0, False, None, None, gw, amax=amax)
    if n > 1:
        assert torch.isnan(g[0]).any() and torch.isfinite(g[1:]).all()
        assert bits(amax) == bits(g[~torch.isnan(g)].abs().max()), "g_amax must be the maximum over the non-NaN gradients"


def pdf_rows(M, n, seed):
    """Weight rows built to hit the decisions of invert_cdf, then random ones."""
    g = np.random.default_rng(seed)
    w = g.random((n, M)).astype(f32)
    w[0] = 0.0                                                  # all zero: uniform cdf of eps
    w[1 % n] = 0.0; w[1 % n, M // 2] = 1.0                      # one spike
    if n > 2: w[2, :M // 3] = 0.0                               # leading zero run
    if n > 3: w[3, M - M // 3:] = 0.0                           # trailing zero run
    if n > 4: w[4] = 1e-12; w[4, ::3] = 1.0                     # 1e-12 beside 1: bins with denom < eps
    if n > 5: w[5] = np.floor(g.random(M) * 4).astype(f32)      # small integers, zeros among them
    if n > 6: w[6] = (g.random(M) < 0.1).astype(f32) * 100.0
    bins = np.sort(g.random((n, M + 1)).astype(f32) * 4 + 2, 1)
    return bins, w


def check_sample_pdf(impl, M, Ni, shared_u, n=19, strided=False, seed=0):
    bins, w = pdf_rows(M, n, 100 * M + Ni + seed)
    cdf = emu.build_cdf32(w, 1e-5)
    g = np.random.default_rng(M + Ni)
    if shared_u:
        u = np.linspace(0, 1, Ni, dtype=f32) if Ni > 1 else np.array([0.5], f32)
        if Ni >= 5:
            u[1], u[2], u[-2] = cdf[4 % n, min(1, M)], cdf[1 % n, M // 2 + 1], f32(1 - 2.0 ** -24)
    else:
        u = g.random((n, Ni)).astype(f32)
        k = g.integers(0, M + 1, (n, Ni))
        on_knot = g.random((n, Ni)) < 0.4                       # u exactly on knots of the emulated cdf
        u = np.where(on_knot, np.take_along_axis(cdf, k, 1), u).astype(f32)
        u[:, 0] = 0.0
        if Ni > 2: u[:, 1], u[:, 2] = 1.0, f32(1 - 2.0 ** -24)
    tb, tw, tu = (torch.from_numpy(a).to(impl.device) for a in (bins, w, u))
    if strided:                                                 # rows of wider buffers, as render_rays passes weights[:, 1:-1]
        big_b = torch.zeros(n, M + 4, device=impl.device); big_b[:, 2:M + 3] = tb; tb = big_b[:, 2:M + 3]
        big_w = torch.zeros(n, M + 2, device=impl.device); big_w[:, 1:-1] = tw; tw = big_w[:, 1:-1]
    got = impl.sample_pdf(tb, tw, tu).cpu().numpy()
    want = emu.sample_pdf32(bins, w, u)
    diff = got.view(np.uint32) != want.view(np.uint32)
    assert not diff.any(), (f"sample_pdf M={M} Ni={Ni}: {int(diff.sum())} samples differ from the emulation in bits, first at "
                            f"(ray, sample) = {tuple(int(i) for i in np.argwhere(diff)[0])}")
    if n > 1000:
        return 0.0
    # independent of the emulation's inverse: against float64 away from the knots of the float32 cdf
    ref, _, den, binw = emu.sample_pdf64(bins, w, u)
    away = ~emu.knot_samples(w, u, ulps=4)
    uu = np.broadcast_to(u, (n, Ni))
    cd = cdf.astype(np.float64)
    away &= (np.abs(cd[:, None, :] - uu[:, :, None].astype(np.float64)).min(-1) > 1e-5)     # and outside the denom < eps switch
    width = float((bins[:, 1:] - bins[:, :-1]).max())
    unit = 2.0 ** -24 * (width + binw / den)
    m = float((np.abs(got - ref) / unit)[away].max()) if away.any() else 0.0
    MEASURED["sample_pdf"] = max(MEASURED.get("sample_pdf", 0.0), m)
    assert m <= PDF_TOL, f"sample_pdf M={M} Ni={Ni}: {m:.3e} units from float64 away from knots"
    assert (got >= bins[:, :1]).all() and (got <= bins[:, -1:]).all()
    # a bin whose cdf step EQUALS eps keeps its denominator (the test is denom < eps): four zero weights with
    # eps = 0.25 give the cdf 0, .25, .5, .75, 1 exactly
    b4 = torch.from_numpy(bins[:, :5].copy()).to(impl.device) if M >= 4 else torch.arange(5.0, device=impl.device).repeat(n, 1)
    u4 = torch.tensor([0.0, 0.1, 0.25, 0.3, 0.6, 0.75, 0.99, 1.0], device=impl.device)
    got4 = impl.sample_pdf(b4, torch.zeros(n, 4, device=impl.device), u4, eps=0.25).cpu().numpy()
    want4 = emu.sample_pdf32(b4.cpu().numpy(), np.zeros((n, 4), f32), u4.cpu().numpy(), eps=0.25)
    assert np.array_equal(got4.view(np.uint32), want4.view(np.uint32)), "sample_pdf: cdf step == eps"
    for r in range(n):
        k = np.argsort(uu[r][away[r]], kind="stable")
        assert (np.diff(got[r][away[r]][k]) >= -2e-6 * width).all(), f"sample_pdf M={M} Ni={Ni}: samples of ray {r} decrease with increasing u"
    return m


def merge_inputs(S, Ni, kind, n, seed):
    g = np.random.default_rng(seed)
    z = np.sort(g.random((n, S)).astype(f32) * 4 + 2, 1)
    w = g.random((n, S)).astype(f32)
    w[0] = 0.0
    u = np.linspace(0, 1, Ni, dtype=f32) if kind == "linspace" else g.random((n, Ni)).astype(f32)
    if kind == "one_swap" and Ni >= 2:
        u = np.sort(u, 1); j = Ni // 2; u[:, [j - 1, j]] = u[:, [j, j - 1]]
    if kind == "ties" and Ni >= 2:
        u[:, 1::2] = u[:, 0::2][:, :u[:, 1::2].shape[1]]                   # equal new depths, out of order overall
    if kind == "coarse_tie" and S >= 4:
        # a spike at interior weight k puts cdf knots at z_mid; coincident coarse depths make z_mid[k] == z[k] == z[k+1]
        k = S // 2
        z[:, k + 1] = z[:, k]
        z = np.sort(z, 1)
        cdf = emu.build_cdf32(w[:, 1:-1], 1e-5)
        u = g.random((n, Ni)).astype(f32)
        u[:, 0] = cdf[:, min(k, S - 2)]
    if kind == "general" and n >= 4:
        z[1, S // 2] = np.nan; z[2, 0] = np.inf; z[3] = z[3, ::-1]
    return z, w, u


def check_merge(impl, S, Ni, kind, n=13, seed=0):
    z, w, u = merge_inputs(S, Ni, kind, n, 7 * S + Ni + seed)
    tz, tw, tu = (torch.from_numpy(np.ascontiguousarray(a)).to(impl.device) for a in (z, w, u))
    fine, new = impl.importance_merge(tz, tw, tu)
    fine, new = fine.cpu().numpy(), new.cpu().numpy()
    ref_new = impl.sample_pdf(torch.from_numpy(emu.z_mid32(z)).to(impl.device), tw[:, 1:-1], tu).cpu().numpy()
    same = lambda a, b: bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())
    assert same(new, ref_new), f"merge S={S} Ni={Ni} {kind}: z_new is not snb_sample_pdf on z_mid, weights[:, 1:-1]"
    assert same(new, emu.sample_pdf32(emu.z_mid32(z), w[:, 1:-1], u)), f"merge S={S} Ni={Ni} {kind}: z_new differs from the emulation"
    want = emu.sort_like_torch(np.concatenate([z, new], 1))
    ok = (fine.view(np.uint32) == want.view(np.uint32)) | (np.isnan(fine) & np.isnan(want))
    assert ok.all(), (f"merge S={S} Ni={Ni} {kind}: z_fine differs from sort(cat(z, z_new)), first at "
                      f"{tuple(int(i) for i in np.argwhere(~ok)[0])} (a slot holding the -7 sentinel was never written)")
    fine2, none = impl.importance_merge(tz, tw, tu, want_new=False)
    assert none is None and same(fine2.cpu().numpy(), fine)


# ------------------------------------------------------------------------------------------------ the tests
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
@pytest.mark.parametrize("S", S_ALL)
def test_composite_every_kernel_shape(lib, S, cfg):
    quad = S % 4 == 0 and 4 <= S <= 128
    for n in ray_counts(lib, S, quad):
        check_composite(lib, S, n, CONFIGS[cfg])


@pytest.mark.parametrize("S", (64, 132))
def test_composite_past_the_launch_cap(lib, S):
    n = past_cap(lib, S)
    check_composite(lib, S, n, CONFIGS[1])
    check_composite(lib, S, n, CONFIGS[4])


def test_composite_offset_views(lib):
    check_offset_views(lib)


def test_composite_degenerate_samples(lib):
    check_degenerate(lib)


@pytest.mark.parametrize("mode", ("scalar", "per_ray", "rgb_only", "depth_only"))
@pytest.mark.parametrize("S", (8, 30, 64, 128, 132))
def test_fused_losses_every_kernel_shape(lib, S, mode):
    check_losses(lib, S, 77, mode)
    check_losses(lib, S, 5, mode, g_loss=(0.37, -2.5), wb=False)


@pytest.mark.parametrize("S", (64, 132))
def test_fused_losses_past_the_launch_cap(lib, S):
    check_losses(lib, S, past_cap(lib, S), "per_ray", g_loss=(1.7, 0.3))


@pytest.mark.parametrize("S", (8, 64, 128, 30, 132))
def test_g_amax(lib, S):
    for n in (1, 77, past_cap(lib, S) if S in (64, 132) else 300):
        check_amax(lib, S, n)


@pytest.mark.parametrize("Ni", (1, 5, 32, 64, 100))
@pytest.mark.parametrize("M", (1, 2, 31, 32, 33, 62, 126, 254))
def test_sample_pdf_bitwise(lib, M, Ni):
    check_sample_pdf(lib, M, Ni, shared_u=True)
    check_sample_pdf(lib, M, Ni, shared_u=False)
    check_sample_pdf(lib, M, Ni, shared_u=False, strided=True, n=7, seed=1)


def test_sample_pdf_past_the_launch_cap(lib):
    check_sample_pdf(lib, 62, 64, shared_u=False, n=2 * 4 * 16 * lib.sm_count + 13)


# snb_importance_merge refuses S = 2 (it needs one interior weight), so the smallest S is 3
@pytest.mark.parametrize("kind", ("linspace", "random", "one_swap", "ties", "coarse_tie", "general"))
@pytest.mark.parametrize("Ni", (1, 5, 16, 64, 100, 256))
@pytest.mark.parametrize("S", (3, 4, 17, 33, 34, 64, 128))
def test_importance_merge_bitwise(lib, S, Ni, kind):
    check_merge(lib, S, Ni, kind)


def test_importance_merge_past_the_launch_cap(lib):
    """More rays than warps, with NaN / inf / descending rows every 7th ray: ordinary and general-path rows meet in one
    warp's successive trips through its shared-memory slice."""
    n, S, Ni = 2 * 4 * 16 * lib.sm_count + 13, 64, 64
    z, w, u = merge_inputs(S, Ni, "random", n, 3)
    z[::7, 5] = np.nan; z[3::7] = z[3::7, ::-1]; z[5::7, -1] = np.inf
    tz, tw, tu = (torch.from_numpy(np.ascontiguousarray(a)).to(lib.device) for a in (z, w, u))
    fine, new = lib.importance_merge(tz, tw, tu)
    new_np = new.cpu().numpy()
    want_new = emu.sample_pdf32(emu.z_mid32(z), w[:, 1:-1], u)
    assert ((new_np.view(np.uint32) == want_new.view(np.uint32)) | (np.isnan(new_np) & np.isnan(want_new))).all()
    want = torch.sort(torch.cat([tz, new], 1), dim=1, stable=True)[0]
    assert torch.equal(torch.nan_to_num(fine, nan=-1.0), torch.nan_to_num(want, nan=-1.0))


def test_importance_merge_refuses_more_than_256(lib):
    z = torch.zeros(2, 8, device=lib.device)
    fine = torch.zeros(2, 8 + 257, device=lib.device)
    u = torch.zeros(257, device=lib.device)
    p = lib._lib.ptr
    rc = lib.lib.snb_importance_merge(p(z), p(z), p(u), 0, 2, 8, 257, 1e-5, p(fine), None, None)
    assert rc == -3 and b"N_importance > 256" in lib.lib.snb_last_error()


def test_sample_coarse_past_the_cap_one_sample_and_zero_near(lib):
    from oracle import render_oracle as orc
    p = lib._lib.ptr
    g = torch.Generator().manual_seed(2)

    def run(rays, S, use_disp, perturb, u):
        d_rays, d_steps = rays.to(lib.device), torch.linspace(0, 1, S).to(lib.device)
        d_u = None if u is None else u.to(lib.device)
        z = torch.full((rays.shape[0], S), -7.0, device=lib.device)
        rc = lib.lib.snb_sample_coarse(p(d_rays), p(d_steps), p(d_u), perturb, use_disp, rays.shape[0], S, p(z), None)
        assert rc == 0, lib.lib.snb_last_error()
        torch.cuda.synchronize()
        return z.cpu()

    n, S = 8 * lib.sm_count * 256 // 64 * 2 + 13, 64                    # more elements than two trips of the capped grid
    rays = torch.rand(n, 8, generator=g); rays[:, 6] += 0.5; rays[:, 7] = 3 + 4 * rays[:, 7]
    u = torch.rand(n, S, generator=g)
    for use_disp in (0, 1):
        ref = orc.sample_z(rays[:, 6:7], rays[:, 7:8], S, bool(use_disp), 0.37, u)
        assert torch.equal(run(rays, S, use_disp, 0.37, u), ref)
    r1 = rays[:33]
    assert torch.equal(run(r1, 1, 0, 0.0, None), orc.sample_z(r1[:, 6:7], r1[:, 7:8], 1))
    assert torch.equal(run(r1, 1, 0, 1.0, u[:33, :1].contiguous()), orc.sample_z(r1[:, 6:7], r1[:, 7:8], 1, False, 1.0, u[:33, :1]))
    r0 = r1.clone(); r0[:, 6] = 0.0                                      # use_disp with near = 0: 1 / 0 as the oracle's
    got, ref = run(r0, 16, 1, 0.0, None), orc.sample_z(r0[:, 6:7], r0[:, 7:8], 16, True)
    assert torch.equal(torch.isnan(got), torch.isnan(ref)) and torch.equal(torch.nan_to_num(got, nan=-1.0), torch.nan_to_num(ref, nan=-1.0))
