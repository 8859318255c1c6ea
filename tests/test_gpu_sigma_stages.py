"""The sigma-only training forward, stage by stage, and the training backward on poisoned buffers.

snb_field_forward_train_sigma and snb_field_forward_train16_sigma run the coarse pass of render_rays(test_time=True)
and all of eval_points: every sigma-only training step.  Here they are held
  1. layer by layer to float64 from the kernel's own saved inputs, in every precision mode, at the training coarse
     pass (1 M points), a ragged DTU batch and the eval_points shapes (one sample per ray, P = 1, 127, 129, 4097);
  2. bit for bit to the full training pass, of which they are the trunk and the sigma head: sigma, the encoding and
     h1..h8, and in act16 the fp16 cells and ReLU mask bits, with the padded rows zero and the direction encoding and
     direction-layer sections never written;
and the training backward of both passes, in both storage arms, is run on buffers filled with 0xFF bytes (NaN in fp16
and fp32) wherever the library's callers allocate with torch.empty, and with the g_amax statistic the compositing
backward hands it, as production calls it.

The float64 references run on the GPU in blocks of 64 k points; the bars are those of the full pass
(tests/test_gpu_layerwise.py, tests/test_gpu_f16.py), since the arithmetic is the same.
"""
import ctypes as C

import pytest
import torch

from oracle import render_oracle as orc
from tests._common import rel_l2, room_params
from tests.test_gpu_f16 import F16_BOUNDS
from tests.test_gpu_field_schedule import A16_SECTIONS, act16_planes, assert_rows_equal, train_forward
from tests.test_gpu_layerwise import (BLOCK, FWD_BOUNDS, NAMES, ST_AMAX_G, ST_SCALE_H0, ST_SCALE_HG, Stat,
                                      add_trunk_errors, assert_trunk_bounds, bwd16_layout, packed, points32, ray_batch,
                                      report, to_dev, trunk_reference)
from tests.test_gpu_layerwise import P_RAGGED as P_RAGGED_FULL
from tests.test_gpu_sigma_train import P_RAGGED as P_RAGGED_SIGMA
from tests.test_gpu_sigma_train import SIGMA_PASS

DEV = "cuda:0"
MODES = ["fp32", "f16x3", "bf16x3", "bf16", "f16"]


def weights_of(tag):
    return orc.default_init_params(1) if tag == "default" else room_params("coarse")


def point_rays(P, seed):
    """P points in [-1.5, 1.5]^3 staged as eval_points stages them: one sample per ray at z = 0, o = the point, d = 0."""
    g = torch.Generator().manual_seed(seed)
    rays = torch.zeros(P, 8)
    rays[:, :3] = (torch.rand(P, 3, generator=g) * 2 - 1) * 1.5
    return rays.to(DEV).contiguous(), torch.zeros(P, 1, device=DEV)


# (label, rays, z): the training coarse pass (4 x 4096 lego rays x 64 samples), a ragged DTU batch, and eval_points'
# one-sample rays -- S = 1, a single point, a partial last tile, one point past a tile, fewer tiles than CTAs
SHAPES = [("lego 16384x64", lambda: ray_batch("lego", 16384, 64, 61)), ("dtu 333x97", lambda: ray_batch("dtu", 333, 97, 62))] + \
    [(f"points {P}", lambda P=P: point_rays(P, 63 + P)) for P in (1, 127, 129, 4097)]


def lib_prec(precision):
    from sinnerf_b200 import _lib
    return _lib.load(), _lib.precision_id(precision)


# --------------------------------------------------------------------------------------------------------------------
# 1. the float64 sigma-only forward itself (CPU)
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["default", "room"])
def test_fp64_sigma_forward_matches_the_oracle(tag):
    """trunk_reference, the per-layer float64 reference of the GPU checks below, chained on its own outputs with exact
    operands, is oracle.render_oracle.field_mlp(..., sigma_only=True) in float64 to 1e-12."""
    g = torch.Generator().manual_seed(5)
    n = 300
    p = {k: v.double() for k, v in weights_of(tag).items()}
    enc = orc.embed(torch.randn(n, 3, generator=g, dtype=torch.float64) * 1.5, orc.N_XYZ_FREQS)

    def exact(x, nonneg):
        return x.double(), None

    H = [torch.zeros(n, 256, dtype=torch.float64)] * 8
    for _ in range(8):      # layer l reads only h_{l-1}: after eight passes every layer has seen its true input
        layers, _ = trunk_reference(p, enc, H, exact)
        H = [torch.relu(pre) for pre, _ in layers]
    layers, (sigma, norm) = trunk_reference(p, enc, H, exact)
    want = orc.field_mlp(p, enc, None, sigma_only=True)
    assert sigma.shape == want.shape == (n, 1)
    assert torch.allclose(sigma, want, rtol=1e-12, atol=1e-12), float((sigma - want).abs().max())
    assert bool((norm >= sigma.abs()).all())
    for (pre, nrm), h in zip(layers, H):
        assert torch.equal(torch.relu(pre), h) and bool((nrm >= pre.abs()).all())


# --------------------------------------------------------------------------------------------------------------------
# 2. snb_field_forward_train_sigma layer by layer against float64
# --------------------------------------------------------------------------------------------------------------------
# The full pass's bars (FWD_BOUNDS; F16_BOUNDS for f16) hold with the same ~10x margin.  Worst measured over both
# weight sets and all six shapes (NVIDIA H100 80GB HBM3, 700 W):
#              enc      h max    h rms    sigma
#   fp32       8.7e-8   9.4e-7   5.9e-8   4.0e-7
#   f16x3      8.7e-8   2.5e-6   2.8e-7   2.7e-7
#   bf16x3     8.7e-8   2.2e-6   2.3e-7   2.6e-7
#   bf16       4.9e-7   8.0e-7   5.4e-8   2.7e-7
#   f16        4.9e-7   1.0e-6   1.1e-7   2.8e-7
def bounds_of(precision):
    return F16_BOUNDS if precision == "f16" else FWD_BOUNDS[precision]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("weights", ["default", "room"])
def test_sigma_training_forward_layerwise(precision, weights):
    """The saved xyz encoding (padding column zero), h1..h8 (normalised error max and rms, no ReLU flips) and sigma of
    snb_field_forward_train_sigma against float64 from the kernel's own saved inputs, rounded as the training epilogue
    (split_pair<..., kNonNeg>) forms its MMA operands; the full pass's bars."""
    lib, prec = lib_prec(precision)
    pd = to_dev(weights_of(weights))
    _, img = packed(pd, precision)
    bounds = bounds_of(precision)
    for label, make in SHAPES:
        torch.cuda.reset_peak_memory_stats()
        rays, z = make()
        out = train_forward(lib, img, prec, rays, z, True, "fp32")
        sigma = out["raw"]
        P = sigma.shape[0]
        assert torch.isfinite(sigma).all()
        xyz, _ = points32(rays, z)
        st = {k: Stat() for k in ["enc"] + [f"h{l + 1}" for l in range(8)] + ["sigma"]}
        flips = 0
        for p0 in range(0, P, BLOCK):
            sl = slice(p0, min(P, p0 + BLOCK))
            H = [out[f"h{l + 1}"][sl] for l in range(8)]
            flips += add_trunk_errors(st, pd, precision, xyz[sl], out["enc"][sl], H, sigma[sl], bounds[1])
        report(f"sigma-only forward {precision} {weights} {label} (bars: enc {bounds[0]:.1e}, h max {bounds[1]:.1e} "
               f"rms {bounds[2]:.1e}, sigma {bounds[4]:.1e})", st)
        assert_trunk_bounds(st, flips, bounds)
        del out


# --------------------------------------------------------------------------------------------------------------------
# 3. the sigma path is the full pass without the direction layer, bit for bit
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES)
def test_sigma_pass_is_the_full_pass_trunk(precision):
    """sigma_only gates only the direction encoding and the tile's end (field_tc.cu: trunk_epilogue, tile_end; the SIMT
    kernel (field_simt.cu) computes the same encodings, trunk and sigma head and stops before the bottleneck), so on
    the same rays:
      * train_sigma's sigma, enc and h1..h8 are the bits of train's raw[:, 3] and saves;
      * train16_sigma's sigma is train_sigma's; its act16 enc / h cells are the fp32 saves saturated and rounded to
        fp16 and its mask bits their signs; rows [P, Ppad) are zero; the dir and g sections, which the sigma backward
        never reads, still hold the 0xAB the buffer was filled with."""
    lib, prec = lib_prec(precision)
    pd = to_dev(weights_of("room"))
    _, img = packed(pd, precision)
    for label, make in SHAPES[1:]:
        rays, z = make()
        full = train_forward(lib, img, prec, rays, z, False, "fp32")
        sig = train_forward(lib, img, prec, rays, z, True, "fp32")
        P = sig["raw"].shape[0]
        assert torch.isfinite(sig["raw"]).all()
        assert_rows_equal(sig["raw"], full["raw"][:, 3:4].contiguous(), f"{precision} {label} sigma")
        for name in ["enc"] + [f"h{l + 1}" for l in range(8)]:
            assert_rows_equal(sig[name], full[name], f"{precision} {label} {name}")
        del full
        if precision == "fp32":
            continue                       # the 16-bit storage needs a tensor-core mode
        s16 = train_forward(lib, img, prec, rays, z, True, "fp16", fill=0xAB)
        assert_rows_equal(s16["raw"], sig["raw"], f"{precision} {label} train16 sigma")
        planes = act16_planes(s16["act16"], P)
        for name, _ in A16_SECTIONS:
            got = planes[name]
            if name in ("dir", "g"):
                assert bool((got.contiguous().view(torch.uint8) == 0xAB).all()), f"{precision} {label}: {name} was written"
                continue
            assert_rows_equal(got[:P], sig[name].clamp(-65504, 65504).half().view(torch.int16), f"{precision} {label} {name}")
            assert not bool(got[P:].any()), f"{precision} {label} {name}: padded points are not zero"
        bits = planes["mask"]
        for l in range(8):
            assert_rows_equal(bits[l, :P], sig[f"h{l + 1}"] > 0, f"{precision} {label} mask of h{l + 1}")
        assert not bool(bits[:, P:].any()), f"{precision} {label} mask: padded points are not zero"
        print(f"\n{precision} {label}: sigma-only pass = full-pass trunk, bit for bit (P = {P})")


# --------------------------------------------------------------------------------------------------------------------
# 4. the training backward on poisoned buffers, and with the compositing backward's g_amax
# --------------------------------------------------------------------------------------------------------------------
def filled(n, fill, dtype=torch.uint8):
    """n elements of `dtype` whose every byte is `fill`: the library's view of a torch.empty buffer at its worst (0xFF
    is NaN in fp16 and fp32) or at its kindest (0)."""
    nbytes = n * torch.empty(0, dtype=dtype).element_size()
    return torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV).view(dtype)


def grad_arrays(pd, sigma_only):
    grads = {k: torch.zeros_like(v) for k, v in pd.items()}
    parr = (C.c_void_p * 24)(*[pd[k].data_ptr() for k in NAMES])
    garr = (C.c_void_p * 24)(*[grads[k].data_ptr() if (k in SIGMA_PASS or not sigma_only) else None for k in NAMES])
    return grads, parr, garr


class Pass:
    """One field pass through the C ABI, every buffer production takes from torch.empty filled with `fill` bytes:
    forward(rays, z) keeps what the backward reads; backward(g) returns the gradients (and the 16-bit workspace).
    sigma_only: snb_field_forward_train[16]_sigma + snb_field_backward[16]_sigma; else the full pass.
    arm '16': act16 + snb_bwd16_workspace_bytes; arm '32': fp32 saves + ws_a / ws_b / ws_s / ws_w (BWD_WS_FLOATS) / ws_m."""

    def __init__(self, pd, img, precision, sigma_only, arm):
        self.pd, self.img, self.sigma_only, self.arm = pd, img, sigma_only, arm
        self.lib, self.prec = lib_prec(precision)

    def forward(self, rays, z, fill):
        from sinnerf_b200 import _lib
        lib, st = self.lib, _lib.stream_ptr(torch.device(DEV))
        n, S = z.shape
        P = self.P = n * S
        self.rays, self.z = rays, z
        self.raw = self.act16 = self.enc = self.h = self.dir = self.g = None     # free the last pass's buffers first
        self.raw = filled(P * (1 if self.sigma_only else 4), fill, torch.float32).view(P, -1)
        args = (_lib.ptr(self.img), self.prec, _lib.ptr(rays), _lib.ptr(z), n, S, _lib.ptr(self.raw))
        if self.arm == "16":
            self.act16 = filled(lib.snb_act16_bytes(P), fill)
            entry = lib.snb_field_forward_train16_sigma if self.sigma_only else lib.snb_field_forward_train16
            _lib.check(entry(*args, _lib.ptr(self.act16), st), "forward16")
        else:
            self.enc, self.h = filled(P * 64, fill, torch.float32), filled(8 * P * 256, fill, torch.float32)
            if self.sigma_only:
                _lib.check(lib.snb_field_forward_train_sigma(*args, _lib.ptr(self.enc), _lib.ptr(self.h), st), "forward_sigma")
            else:
                self.dir, self.g = filled(P * 32, fill, torch.float32), filled(P * 128, fill, torch.float32)
                _lib.check(lib.snb_field_forward_train(*args, _lib.ptr(self.enc), _lib.ptr(self.dir), _lib.ptr(self.h),
                                                       _lib.ptr(self.g), st), "forward")
        torch.cuda.synchronize()
        return self.raw

    def backward(self, g, fill, g_amax=None):
        from sinnerf_b200 import _lib
        lib, st, P = self.lib, _lib.stream_ptr(torch.device(DEV)), self.P
        grads, parr, garr = grad_arrays(self.pd, self.sigma_only)
        ws = None
        if self.arm == "16":
            ws = filled(lib.snb_bwd16_workspace_bytes(P), fill)
            if self.sigma_only:
                rc = lib.snb_field_backward16_sigma(parr, garr, _lib.ptr(g), _lib.ptr(self.act16), P, _lib.ptr(ws),
                                                    _lib.ptr(g_amax), st)
            else:
                rc = lib.snb_field_backward16(parr, garr, 1, _lib.ptr(g), _lib.ptr(self.raw), _lib.ptr(self.act16), P,
                                              _lib.ptr(ws), _lib.ptr(g_amax), st)
        else:
            assert g_amax is None
            ws_a, ws_b = filled(P * 256, fill, torch.float32), filled(P * 256, fill, torch.float32)
            ws_m = filled(P * 8, fill, torch.int32)
            if self.sigma_only:
                rc = lib.snb_field_backward_sigma(parr, garr, _lib.ptr(g), _lib.ptr(self.enc), _lib.ptr(self.h), P,
                                                  _lib.ptr(ws_a), _lib.ptr(ws_b), _lib.ptr(ws_m), st)
            else:
                ws_s, ws_w = filled(P * 128, fill, torch.float32), filled(_lib.BWD_WS_FLOATS, fill, torch.float32)
                rc = lib.snb_field_backward(parr, garr, 1, _lib.ptr(g), _lib.ptr(self.raw), _lib.ptr(self.enc),
                                            _lib.ptr(self.dir), _lib.ptr(self.h), _lib.ptr(self.g), P, _lib.ptr(ws_a),
                                            _lib.ptr(ws_b), _lib.ptr(ws_s), _lib.ptr(ws_w), _lib.ptr(ws_m), st)
        _lib.check(rc, f"backward arm {self.arm} sigma_only={self.sigma_only}")
        torch.cuda.synchronize()
        return {k: v for k, v in grads.items() if k in SIGMA_PASS or not self.sigma_only}, ws


def check_forward_output(run, fill):
    """What a forward into `fill`-byte buffers leaves for the backward: every saved value finite (no poison left), and
    in act16 the padded rows [P, Ppad) zero in every section the backward reads (the wgrads multiply them by zero
    gradient rows, which a NaN would survive).  -> the saved sections, row-major (act16: fp16 bit patterns)."""
    if run.arm == "32":
        saves = {"enc": run.enc, "h": run.h} if run.sigma_only else {"enc": run.enc, "dir": run.dir, "h": run.h, "g": run.g}
        for name, t in saves.items():
            assert torch.isfinite(t).all(), (name, hex(fill))
        return saves
    planes = act16_planes(run.act16, run.P)
    read = {k: v for k, v in planes.items() if not (run.sigma_only and k in ("dir", "g"))}
    for name, t in read.items():
        rows = t[:, run.P:] if name == "mask" else t[run.P:]
        assert not bool(rows.any()), (name, hex(fill), "padded rows are not zero")
        if name != "mask":
            assert torch.isfinite(t.view(torch.float16)).all(), (name, hex(fill))
    return read


def upstream(P, sigma_only, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(P, device=DEV, generator=gen) if sigma_only else torch.randn(P, 4, device=DEV, generator=gen)


@pytest.mark.gpu
@pytest.mark.parametrize("arm", ["16", "32"])
@pytest.mark.parametrize("sigma_only", [False, True])
def test_backward_on_poisoned_buffers(sigma_only, arm):
    """Forward + backward with every torch.empty buffer (outputs, act16 or the fp32 saves, the workspaces) filled with
    0xFF bytes against the same run on zero-filled buffers: the forward's saves are the same bits with no poison left and
    act16's padded rows zero; on one tile (one ray of 16 samples for the sigma pass, of 32 for the full pass) the
    16-bit arm's gradients are the same bits, since there every gradient element gets one atomic add onto zero; at a
    ragged training size (P_RAGGED of the pass) every gradient is finite and within 4x the run-to-run noise of the
    atomics (max over tensors of the rel-L2 between two clean runs).  The fp32 arm is held to that noise on one tile
    too: its head and wgrad kernels (field_bwd.cu, wgrad_tc.cu) add partial sums with one atomic per warp, so its
    sigma / rgb head and trunk bias gradients change in the last bits between two clean one-tile runs."""
    torch.cuda.reset_peak_memory_stats()
    pd = to_dev(weights_of("room"))
    _, img = packed(pd, "f16x3")
    run = Pass(pd, img, "f16x3", sigma_only, arm)
    # one tile
    rays, z = ray_batch("lego", 1, 16 if sigma_only else 32, 71)
    g = upstream(z.numel(), sigma_only, 72)
    run.forward(rays, z, 0x00)
    saved = {k: v.clone() for k, v in check_forward_output(run, 0x00).items()}
    clean, _ = run.backward(g, 0x00)
    run.forward(rays, z, 0xFF)
    for k, v in check_forward_output(run, 0xFF).items():
        assert torch.equal(v, saved[k]), (k, "the forward's saves depend on what the buffer held")
    dirty, _ = run.backward(g, 0xFF)
    if arm == "32":
        again, _ = run.backward(g, 0x00)
        noise1 = max(rel_l2(again[k], clean[k]) for k in clean)
    for k in clean:
        assert torch.isfinite(dirty[k]).all(), (k, "one tile")
        if arm == "16":
            assert torch.equal(dirty[k].view(torch.int32), clean[k].view(torch.int32)), (k, "one tile")
        else:
            assert rel_l2(dirty[k], clean[k]) <= max(4 * noise1, 1e-6), (k, "one tile", noise1)
    # ragged training size
    P = P_RAGGED_SIGMA if sigma_only else P_RAGGED_FULL
    n = (P + 63) // 64
    rays, z = ray_batch("lego", n, 64, 73)
    rays, z = rays.repeat_interleave(64, 0)[:P].contiguous(), z.reshape(-1, 1)[:P].contiguous()
    g = upstream(P, sigma_only, 74)
    run.forward(rays, z, 0x00)
    clean, _ = run.backward(g, 0x00)
    again, _ = run.backward(g, 0x00)
    noise = max(rel_l2(again[k], clean[k]) for k in clean)
    del again
    run.forward(rays, z, 0xFF)
    check_forward_output(run, 0xFF)
    dirty, _ = run.backward(g, 0xFF)
    worst = 0.0
    for k in clean:
        assert torch.isfinite(dirty[k]).all(), (k, P)
        r = rel_l2(dirty[k], clean[k])
        worst = max(worst, r)
        assert r <= max(4 * noise, 1e-6), (k, r, noise)
    print(f"\npoisoned buffers, {'sigma' if sigma_only else 'full'} pass, arm {arm}, P={P}: worst rel-L2 to the "
          f"clean run {worst:.2e}, atomics noise {noise:.2e}; peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def composite_upstream(run, n, S, seed):
    """The compositing backward production runs before the field backward: (g_raw (P,4) or g_sigma (P,), g_amax)."""
    from sinnerf_b200 import _lib
    lib, st = run.lib, _lib.stream_ptr(torch.device(DEV))
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g_amax = torch.zeros(1, device=DEV)
    g_w = torch.randn(n, S, device=DEV, generator=gen)
    if run.sigma_only:
        g = torch.empty(n, S, device=DEV)
        _lib.check(lib.snb_composite_backward_weights(_lib.ptr(run.raw), _lib.ptr(run.z), _lib.ptr(run.rays), None, 0.0,
                                                      _lib.ptr(g_w), n, S, _lib.ptr(g), _lib.ptr(g_amax), st),
                   "snb_composite_backward_weights")
    else:
        g_rgb, g_depth = torch.randn(n, 3, device=DEV, generator=gen), torch.randn(n, device=DEV, generator=gen)
        g = torch.empty(n, S, 4, device=DEV)
        _lib.check(lib.snb_composite_backward_loss(_lib.ptr(run.raw), _lib.ptr(run.z), _lib.ptr(run.rays), None, 0.0, 0,
                                                   _lib.ptr(g_rgb), _lib.ptr(g_depth), _lib.ptr(g_w), None, None, None,
                                                   None, n, S, _lib.ptr(g), _lib.ptr(g_amax), st),
                   "snb_composite_backward_loss")
    torch.cuda.synchronize()
    return g.reshape(n * S, -1).squeeze(1).contiguous(), g_amax


@pytest.mark.gpu
@pytest.mark.parametrize("sigma_only", [False, True])
def test_backward16_with_the_compositing_g_amax(sigma_only):
    """The 16-bit backward as production calls it: g_amax from snb_composite_backward_loss (full pass) or
    snb_composite_backward_weights (sigma pass) instead of NULL (amax_kernel).  The state block (max |g|, bound
    ingredients, every scale) is the same bits, so are the fp16 gradient planes; on one tile the gradients too.
    Both workspaces start as the same 0xFF bytes, so planes a pass does not write compare equal as well."""
    pd = to_dev(weights_of("room"))
    _, img = packed(pd, "f16x3")
    run = Pass(pd, img, "f16x3", sigma_only, "16")
    for n, S in ((1, 16 if sigma_only else 32), (333, 97)):
        rays, z = ray_batch("lego", n, S, 81)
        run.forward(rays, z, 0xFF)
        g, g_amax = composite_upstream(run, n, S, 82)
        assert float(g_amax.view(torch.float32)) == float(g.abs().max()) > 0
        L = bwd16_layout(n * S)
        with_amax, ws_a = run.backward(g, 0xFF, g_amax)
        null, ws_n = run.backward(g, 0xFF)
        state_a = ws_a[L["state"]:L["state"] + 64 * 4].view(torch.float32)
        state_n = ws_n[L["state"]:L["state"] + 64 * 4].view(torch.float32)
        assert float(state_a[ST_AMAX_G]) == float(g_amax), (n, S)
        assert torch.equal(state_a.view(torch.int32), state_n.view(torch.int32)), \
            (n, S, (state_a != state_n).nonzero().flatten().tolist())
        assert torch.equal(ws_a[:L["fold"]], ws_n[:L["fold"]]), (n, S, "the fp16 gradient planes differ")
        print(f"\ng_amax path, {'sigma' if sigma_only else 'full'} pass, {n}x{S}: scales "
              f"{torch.log2(state_a[ST_SCALE_HG:ST_SCALE_H0 + 8]).tolist()}")
        for k in null:
            assert torch.isfinite(with_amax[k]).all(), k
            if n == 1:
                assert torch.equal(with_amax[k].view(torch.int32), null[k].view(torch.int32)), k
            else:
                assert rel_l2(with_amax[k], null[k]) <= 1e-5, (k, rel_l2(with_amax[k], null[k]))
