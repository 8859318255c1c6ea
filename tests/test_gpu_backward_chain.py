"""The 16-bit training backward hop by hop against float64, one probe point per launch.

snb_field_backward16 and snb_field_backward16_sigma run with the upstream gradient zero except at one point p.  Then
every gradient row is zero except row p, and the backward's arithmetic at p reads back exactly through the C ABI
(tests/bwd16_emulation.py): each layer's fp16 hi plane at p is its bias gradient times its scale, the weight gradients
are rank-1 and bit-exact, dS (hi and residual planes), the hg cell, the fold scratch and the residual planes of g_h6 /
g_h5 stay in the workspace.  The checkers of tests/bwd16_emulation.py (`check_probe`) then hold
  * dS and the hg cell (hi + lo) to float64 from g_raw, raw and the decoded G, within the rounding count of the head;
  * the residual segment (dS -> g_h8 -> ... -> g_h4) chained in float64 from the observed dS, and the hops g_h6 ->
    g_h5 -> g_h4 from their observed hi + lo, to half an fp16 ulp plus the bound B of `hop_chain`;
  * the hi-only hops g_h4 -> g_h3 -> g_h2 -> g_h1 from the kernel's own observed input, likewise;
  * every weight gradient bit for bit, the head rows to one fp32 rounding of (hi + lo) x / s, the head biases and the
    hg cell from them exactly, W' and the unfold to their fp32 fmaf-chain bounds.
A dense backward at the training size then has its final workspace checked at every point (dS, hg, the last hop),
its padding and saturation, and every power-of-two scale recomputed on the host; the fp32-storage backward
(snb_field_backward) gets the same probe method hop by hop and a dense check of its final planes.
Every bar is a derived bound (the accumulation term of B counts one truncated fp32 accumulation per wgmma, 2 U32 of
the running |sum|, which A bounds: kappa = 1), and the exact checks stay exact.  The worst ratio (error / allowance)
measured with correct kernels is written below; each test prints its own.  Each probe is run with g_amax NULL and
with max |g| handed over, as the compositing backward hands it in production.
"""
import ctypes as C

import pytest
import torch

from oracle import render_oracle as orc
from tests import bwd16_emulation as em
from tests.bwd16_emulation import check_probe
from tests.test_gpu_field_schedule import train_forward
from tests.test_gpu_layerwise import (BLOCK, NAMES, P_RAGGED, P_TRAIN, ST_SCALE_DS, ST_SCALE_H0, ST_SCALE_HG, a16_pad,
                                      act16_rows, act16_sections, bwd16_layout, forward_train, forward_train16, packed,
                                      ray_batch, run_backward16, slice_edges, t32_rows, to_dev, training_batch)

DEV = "cuda:0"
TC_MODES = ["f16x3", "bf16x3", "bf16", "f16"]
P_SMALL = 37 * 128 + 77          # ragged: 38 tiles of 128, a partial last tile of 32
SIGMA_PASS = {k for k in NAMES if k.startswith("xyz_encoding_") and not k.startswith("xyz_encoding_final")} | \
    {"sigma.weight", "sigma.bias"}

# Worst ratio (error / allowance; <= 1 passes) measured with correct kernels over every mode, weight set, shape and
# probe, NVIDIA H100 80GB HBM3 (700 W):
#   16-bit probes: head 0.35, head biases 0.30, W' 0.03, unfold 0.08; weight gradients, head rows, hg-from-bias and the
#     sigma head's g_h8 bit-exact.  hg 1.0: g_sigma s_hg is exact, so its allowance is only the half ulp of the
#     residual's own rounding, which a tie reaches.  Residual segment 1.0 and hi-only hops 0.99: the half fp16 ulp of
#     the hi rounding itself; beyond that half ulp an error used at most 0.18 (residual) and 0.08 (hi-only) of B, the
#     bound that carries the wgmma accumulation model ('_B' in the printout) -- a ratio past 1 that needs more than
#     all of B is a defect, not a tie.
#   dense final workspace (P_TRAIN, P_RAGGED): dS 0.30, hg 1.0, g_h2 -> g_h1 0.99 (0.12 of B); scales exact.
#   fp32 storage: dS 0.35, dgrad_tc hops 0.57 at the probes, dense dS 0.26 and g_h2 -> g_h1 0.55.
# The file takes ~3 min.


def weights_of(tag):
    return orc.default_init_params(1) if tag == "default" else room_params_fine()


def room_params_fine():
    from tests._common import room_params
    return room_params("fine")


def forward16(img, precision, rays, z):
    """(raw, act16) of the full training forward with 16-bit saves: forward_train16 in f16x3; the other modes through
    train_forward (forward_train16 is fixed to f16x3)."""
    if precision == "f16x3":
        return forward_train16(img, rays, z)
    from sinnerf_b200 import _lib
    out = train_forward(_lib.load(), img, _lib.precision_id(precision), rays, z, False, "fp16")
    return out["raw"], out["act16"]


def probes(P, sm, slices=False):
    """First and last point, both sides of a 32- and a 128-point tile boundary, the ragged tail; with slices, every
    wgrad slice edge for 1 and 2 blocks per slice."""
    pts = {0, P - 1, 31, 32, 127, 128, (P - 1) // 32 * 32, (P - 1) // 128 * 128 - 1}
    if slices:
        n_tiles = a16_pad(P) // 32
        for blocks in (1, 2):
            pts |= set(slice_edges(n_tiles, 32, blocks, sm))
    return sorted(q for q in pts if 0 <= q < P)


def probe_vec(i):
    """Magnitudes 2^-8 .. 2^8; every fourth probe sigma-only, every fourth + 1 rgb-only."""
    g = torch.Generator().manual_seed(100 + i)
    v = torch.randn(4, generator=g).sign() * torch.exp2(torch.rand(4, generator=g) * 16 - 8)
    if i % 4 == 0:
        v[:3] = 0
    elif i % 4 == 1:
        v[3] = 0
    return v


class Backward16:
    """One backward per probe through the C ABI, outputs decoded at the probe row on the CPU."""

    def __init__(self, pd, raw, act16, P, sigma_only):
        from sinnerf_b200 import _lib
        self.lib, self._lib = _lib.load(), _lib
        self.pd, self.raw, self.act16, self.P, self.sigma_only = pd, raw, act16, P, sigma_only
        self.grads = {k: torch.zeros_like(v) for k, v in pd.items()}
        self.ws = torch.empty(self.lib.snb_bwd16_workspace_bytes(P), device=DEV, dtype=torch.uint8)
        self.parr = (C.c_void_p * 24)(*[pd[k].data_ptr() for k in NAMES])
        self.garr = (C.c_void_p * 24)(*[self.grads[k].data_ptr() if (k in SIGMA_PASS or not sigma_only) else None
                                        for k in NAMES])
        self.secs = act16_sections(act16, P)
        self.L = bwd16_layout(P)

    def run(self, pt, vec, with_amax):
        _lib, P = self._lib, self.P
        for g in self.grads.values():
            g.zero_()
        self.ws.fill_(0xFF)
        g_raw = torch.zeros(P, 4, device=DEV)
        g_raw[pt] = vec.to(DEV)
        # production hands over g_amax from the compositing backward, which raises it to max |g| of its own output
        # (tests/test_gpu_sigma_stages.py holds it bit-equal to g.abs().max()); a probe's g_raw is not a compositing
        # output, so the same value is formed here from the probe's g_raw: max |g| of a finite float tensor is exact
        g_amax = g_raw.abs().max().reshape(1).contiguous() if with_amax else None
        st = _lib.stream_ptr(torch.device(DEV))
        if self.sigma_only:
            gs = g_raw[:, 3].contiguous()
            rc = self.lib.snb_field_backward16_sigma(self.parr, self.garr, _lib.ptr(gs), _lib.ptr(self.act16), P,
                                                     _lib.ptr(self.ws), _lib.ptr(g_amax), st)
        else:
            rc = self.lib.snb_field_backward16(self.parr, self.garr, 1, _lib.ptr(g_raw), _lib.ptr(self.raw),
                                               _lib.ptr(self.act16), P, _lib.ptr(self.ws), _lib.ptr(g_amax), st)
        _lib.check(rc, "backward16")
        torch.cuda.synchronize()
        return self.decode(pt, g_raw)

    def decode(self, pt, g_raw):
        idx = torch.tensor([pt], device=DEV)
        L, ws = self.L, self.ws
        rows = act16_rows(self.secs, idx)
        a = {k: (v.cpu() if torch.is_tensor(v) else [x.cpu() for x in v]) for k, v in rows.items()}
        a["enc"], a["dir"] = a["enc"].float(), a["dir"].float()
        pp = a16_pad(self.P)

        def plane(name, F):
            return t32_rows(ws[L[name]:L[name] + pp * F * 2].view(torch.int16), F, idx).float().cpu()

        state = ws[L["state"]:L["state"] + 64 * 4].view(torch.float32).cpu()
        sc = {l: float(state[ST_SCALE_H0 + l - 1]) for l in range(1, 9)}
        sc.update(hg=float(state[ST_SCALE_HG]), ds=float(state[ST_SCALE_DS]))
        fold = ws[L["fold"]:L["fold"] + (2 * 128 * 256 + 128) * 4].view(torch.float32).cpu()
        w = dict(scale=sc, hg=plane("hg", 8), dya=plane("dya", 256), dyb=plane("dyb", 256),
                 dya_lo=plane("dya_lo", 256), dyb_lo=plane("dyb_lo", 256))
        if not self.sigma_only:
            w.update(ds=plane("ds", 128), ds_lo=plane("ds_lo", 128), fold_W=fold[:128 * 256].view(128, 256),
                     fold_dW=fold[128 * 256:2 * 128 * 256].view(128, 256), fold_db=fold[2 * 128 * 256:])
        grads = {k: v.cpu() for k, v in self.grads.items()}
        return grads, w, a, self.raw[pt:pt + 1].cpu(), g_raw[pt:pt + 1].cpu()


def run_probes(bw, pts, p_cpu, label):
    worst = {}
    for i, pt in enumerate(pts):
        vec = probe_vec(i)
        if bw.sigma_only:
            vec[:3] = 0
            vec[3] = vec[3] if vec[3] != 0 else 2.0 ** (i % 17 - 8)
        for with_amax in (False, True):
            grads, w, a, raw, g_raw = bw.run(pt, vec, with_amax)
            res = check_probe(grads, w, p_cpu, a, raw, g_raw, 0, bw.sigma_only)
            for k, v in res.items():
                worst[k] = max(worst.get(k, 0.0), v)
                assert v <= 1.0, (label, pt, vec.tolist(), with_amax, k, v, res)
    print(f"\n{label}: {len(pts)} probes, worst ratio " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("precision", TC_MODES)
@pytest.mark.parametrize("weights", ["default", "room"])
def test_single_probe_chain_small(precision, weights):
    """Every tensor-core mode's act16 forward at a ragged small P, probes at the tile seams and the tail."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    p = weights_of(weights)
    pd = to_dev(p)
    _, img = packed(pd, precision)
    from sinnerf_b200 import _lib
    rays, z = training_batch(P_SMALL, 91)
    raw, act16 = forward16(img, precision, rays, z)
    bw = Backward16(pd, raw, act16, P_SMALL, False)
    run_probes(bw, probes(P_SMALL, sm), p, f"full pass {precision} {weights} P={P_SMALL}")


@pytest.mark.gpu
@pytest.mark.parametrize("P", [P_TRAIN, P_RAGGED])
def test_single_probe_chain_training_size(P):
    """f16x3 at the training size: probes at every wgrad slice edge for 1 and 2 blocks per slice."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    p = weights_of("default")
    pd = to_dev(p)
    _, img = packed(pd, "f16x3")
    from sinnerf_b200 import _lib
    rays, z = training_batch(P, 93)
    raw, act16 = forward_train16(img, rays, z)
    bw = Backward16(pd, raw, act16, P, False)
    run_probes(bw, probes(P, sm, slices=True), p, f"full pass f16x3 P={P}")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", TC_MODES)
def test_single_probe_chain_sigma_pass(precision):
    """snb_field_backward16_sigma: g_h8 = g_sigma w_sigma mask in fp32, its hi plane bit-exact, then the same chain."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    p = weights_of("room")
    pd = to_dev(p)
    _, img = packed(pd, precision)
    from sinnerf_b200 import _lib
    rays, z = ray_batch("lego", P_SMALL // 64 + 1, 64, 95)
    out = train_forward(_lib.load(), img, _lib.precision_id(precision), rays, z, True, "fp16")
    P = z.numel()
    bw = Backward16(pd, out["raw"], out["act16"], P, True)
    run_probes(bw, probes(P, sm, slices=True), p, f"sigma pass {precision} P={P}")


# --------------------------------------------------------------------------------------------------------------------
# the final workspace of a dense backward at the training size
# --------------------------------------------------------------------------------------------------------------------
def plane_rows(ws, L, name, F, idx, P):
    pp = a16_pad(P)
    return t32_rows(ws[L[name]:L[name] + pp * F * 2].view(torch.int16), F, idx)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [P_TRAIN, P_RAGGED])
def test_dense_final_workspace(P):
    """snb_field_backward16 with a dense seeded g_raw.  trunk_backward16's ping-pong leaves dya = g_h2 hi, dyb = g_h1
    hi, dya_lo = g_h6's residual, dyb_lo = g_h5's (by the same walk the probe tests read).  Checked:
      * every ST_SCALE_* is pow2_scale of its bound recomputed on the host from the state block's own maxima and
        bound ingredients, and those ingredients (column L1 norms, max |w_sigma|, the rgb head's norm, max |g_raw|)
        against the weights; the maxima of dS, g_h2 and g_h1 against the planes;
      * W' (fold scratch) against float64 Wd[:, :256] Wf;
      * dS hi / lo and the hg cell at every point (head_ds / head_hg);
      * the hop g_h2 -> g_h1 at every point, tile and CTA, from the kernel's own g_h2 plane;
      * padded rows [P, Ppad) zero in every plane, no plane element at +-65504 (fp16 bits 0x7BFF / 0xFBFF)."""
    from tests.test_gpu_layerwise import ST_AMAX_DS, ST_AMAX_G, ST_AMAX_H0
    torch.cuda.reset_peak_memory_stats()
    p = weights_of("default")
    pd = to_dev(p)
    _, img = packed(pd, "f16x3")
    rays, z = training_batch(P, 97)
    raw, act16 = forward_train16(img, rays, z)
    gen = torch.Generator(device=DEV).manual_seed(98)
    g_raw = torch.randn(P, 4, device=DEV, generator=gen)
    grads, ws = run_backward16(pd, g_raw, raw, act16, P)
    L = bwd16_layout(P)
    pp = a16_pad(P)
    state = ws[L["state"]:L["state"] + 64 * 4].view(torch.float32).cpu()
    fold = ws[L["fold"]:L["fold"] + (2 * 128 * 256 + 128) * 4].view(torch.float32)
    Wfold = fold[:128 * 256].view(128, 256).cpu()
    ok, ratio = em.fold_w(Wfold, p["dir_encoding.0.weight"], p["xyz_encoding_final.weight"])
    assert bool(ok.all()), ("W'", float(ratio.max()))
    # scales and their ingredients
    assert float(state[ST_AMAX_G]) == float(g_raw.abs().max())
    scales, ing = em.plane_scales(state, Wfold, p)
    got = {"hg": float(state[ST_SCALE_HG]), "ds": float(state[ST_SCALE_DS])}
    got.update({l: float(state[ST_SCALE_H0 + l - 1]) for l in range(1, 9)})
    for k, allowed in scales.items():
        assert got[k] in allowed, (k, got[k], allowed)
    for k, (have, want, allow) in ing.items():
        assert abs(have - want) <= allow, (k, have, want, allow)
    # planes: padding, saturation, maxima
    for name, F in (("ds", 128), ("ds_lo", 128), ("hg", 8), ("dya", 256), ("dyb", 256), ("dya_lo", 256), ("dyb_lo", 256)):
        bits = ws[L[name]:L[name] + pp * F * 2].view(torch.int16)
        assert not bool(((bits == 0x7BFF) | (bits == -1025)).any()), (name, "an element sits at +-65504")
        if pp > P:
            pad = plane_rows(ws, L, name, F, torch.arange(P, pp, device=DEV), P)
            assert not bool(pad.any()), (name, "padded rows are not zero")
    # every point: the head and the last hop
    Wr = pd["rgb.0.weight"]
    secs = act16_sections(act16, P)
    sc = {k: float(state[i]) for k, i in (("hg", ST_SCALE_HG), ("ds", ST_SCALE_DS), (2, ST_SCALE_H0 + 1), (1, ST_SCALE_H0))}
    worst = {"head": 0.0, "hg": 0.0, "hop_2_1": 0.0, "hop_2_1_B": 0.0}
    mx = {"ds": 0.0, 2: 0.0, 1: 0.0}
    for p0 in range(0, P, BLOCK):
        idx = torch.arange(p0, min(P, p0 + BLOCK), device=DEV)
        a = act16_rows(secs, idx)
        dsh, dsl = plane_rows(ws, L, "ds", 128, idx, P), plane_rows(ws, L, "ds_lo", 128, idx, P)
        ok, r = em.head_ds(g_raw[idx], raw[idx], a["G"], Wr, sc["ds"], dsh, dsl)
        bad = (~ok).nonzero()
        assert bool(ok.all()), ("dS", p0, float(r.max()), bad[:4].tolist(),
                                [(float(dsh[i, j]), float(dsl[i, j]), float(r[i, j])) for i, j in bad[:4].tolist()])
        worst["head"] = max(worst["head"], float(r.max()))
        ok, r = em.head_hg(g_raw[idx], raw[idx], sc["hg"], plane_rows(ws, L, "hg", 8, idx, P))
        assert bool(ok.all()), ("hg", p0, float(r.max()))
        worst["hg"] = max(worst["hg"], float(r.max()))
        g2, g1 = plane_rows(ws, L, "dya", 256, idx, P), plane_rows(ws, L, "dyb", 256, idx, P)
        hop = dict(W=pd[em.LAYERS[1] + ".weight"], mask=a["M"][0], s_in=sc[2], s_out=sc[1], lo_in=False, lo_out=False, hi=g1)
        (ok, r, used), = em.hop_chain(g2, torch.zeros_like(g2), [hop])
        assert bool(ok.all()), ("g_h2 -> g_h1", p0, float(r.max()))
        worst["hop_2_1"] = max(worst["hop_2_1"], float(r.max()))
        worst["hop_2_1_B"] = max(worst["hop_2_1_B"], float(used.max()))
        mx["ds"] = max(mx["ds"], float((dsh + dsl).abs().max()))
        mx[2], mx[1] = max(mx[2], float(g2.abs().max())), max(mx[1], float(g1.abs().max()))
    # running maxima: of the fp32 values, whose hi planes are within half an fp16 ulp (dS: hi + lo within 2^-22)
    for k, i, tol in (("ds", ST_AMAX_DS, 2.0 ** -21 * mx["ds"]), (2, ST_AMAX_H0 + 1, 2.0 ** -11 * mx[2]),
                      (1, ST_AMAX_H0, 2.0 ** -11 * mx[1])):
        assert abs(float(state[i]) - mx[k]) <= tol, (k, float(state[i]), mx[k])
    print(f"\ndense final workspace P={P}: worst ratio " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items())
          + f"; scales log2 {[round(__import__('math').log2(v)) for v in got.values()]}")


# --------------------------------------------------------------------------------------------------------------------
# fp32-storage arm: snb_field_backward (dgrad_tc / wgrad_tc)
# --------------------------------------------------------------------------------------------------------------------
def backward32(pd, g_raw, raw, save, P):
    from sinnerf_b200 import _lib
    lib = _lib.load()
    grads = {k: torch.zeros_like(v) for k, v in pd.items()}
    ws = dict(a=torch.empty(P, 256, device=DEV), b=torch.empty(P, 256, device=DEV), s=torch.empty(P, 128, device=DEV),
              w=torch.empty(_lib.BWD_WS_FLOATS, device=DEV), m=torch.empty(P, 8, device=DEV, dtype=torch.int32))
    parr = (C.c_void_p * 24)(*[pd[k].data_ptr() for k in NAMES])
    garr = (C.c_void_p * 24)(*[grads[k].data_ptr() for k in NAMES])
    _lib.check(lib.snb_field_backward(parr, garr, 1, _lib.ptr(g_raw), _lib.ptr(raw), _lib.ptr(save["enc"]),
                                      _lib.ptr(save["dir"]), _lib.ptr(save["h"]), _lib.ptr(save["g"]), P,
                                      *[_lib.ptr(ws[k]) for k in "abswm"], _lib.stream_ptr(torch.device(DEV))),
               "snb_field_backward")
    torch.cuda.synchronize()
    return grads, ws


@pytest.mark.gpu
def test_fp32_storage_probes_and_final_workspace():
    """snb_field_backward on 131 072 - 77 points.  Single probes (first / last point, tile seams, every wgrad slice
    edge): its bias sums are fp32 sums of fp32 rows (wgrad_tc.cu), so db_l is g_h_l at the probe exactly, and every
    dgrad_tc hop (dS -> g_h8 through W' with the sigma term, then g_h8 -> ... -> g_h1) is held from its own input to the
    bf16x3 bound of hop_bf16x3; dS at the probe to head_ds.  Then a dense g_raw: after the call ws_s = dS, ws_b = g_h2,
    ws_a = g_h1 (trunk_backward_fp32's ping-pong), checked at every point (dS, and the hop g_h2 -> g_h1)."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    P = 1024 * 128 - 77
    p = weights_of("room")
    pd = to_dev(p)
    _, img = packed(pd, "f16x3")
    rays, z = training_batch(P, 99)
    raw, save = forward_train(img, "f16x3", rays, z)
    Wp = None
    worst = {"head": 0.0, "hop": 0.0}
    pts = probes(P, sm, slices=True)
    for i, pt in enumerate(pts):
        g_raw = torch.zeros(P, 4, device=DEV)
        g_raw[pt] = probe_vec(i).to(DEV)
        grads, ws = backward32(pd, g_raw, raw, save, P)
        Wp = ws["w"][:128 * 256].view(128, 256)
        db = {l: grads[em.LAYERS[l - 1] + ".bias"] for l in range(1, 9)}
        ok, r = em.head_ds(g_raw[pt:pt + 1], raw[pt:pt + 1], save["g"][pt:pt + 1], pd["rgb.0.weight"], 1.0,
                           ws["s"][pt:pt + 1].double(), torch.zeros(1, 128, device=DEV, dtype=torch.float64))
        assert bool(ok.all()), ("dS", pt, float(r.max()))
        worst["head"] = max(worst["head"], float(r.max()))
        H = save["h"][:, pt]
        hops = [(ws["s"][pt], Wp, H[7] > 0, db[8], g_raw[pt, 3] * pd["sigma.weight"][0])]
        for l in range(8, 1, -1):
            W = pd[em.LAYERS[l - 1] + ".weight"]
            hops.append((db[l], W[:, 63:] if l == 5 else W, H[l - 2] > 0, db[l - 1], None))
        for k, (y, W, m, out, ex) in enumerate(hops):
            ok, r = em.hop_bf16x3(y[None], W, m[None], out[None], None if ex is None else ex[None])
            assert bool(ok.all()), ("hop", k, pt, float(r.max()))
            worst["hop"] = max(worst["hop"], float(r.max()))
    ok, r = em.fold_w(Wp, pd["dir_encoding.0.weight"], pd["xyz_encoding_final.weight"])
    assert bool(ok.all()), ("W'", float(r.max()))
    # dense
    gen = torch.Generator(device=DEV).manual_seed(100)
    g_raw = torch.randn(P, 4, device=DEV, generator=gen)
    grads, ws = backward32(pd, g_raw, raw, save, P)
    for name in NAMES:
        assert torch.isfinite(grads[name]).all(), name
    dense = {"head": 0.0, "hop_2_1": 0.0}
    for p0 in range(0, P, BLOCK):
        sl = slice(p0, min(P, p0 + BLOCK))
        ok, r = em.head_ds(g_raw[sl], raw[sl], save["g"][sl], pd["rgb.0.weight"], 1.0, ws["s"][sl].double(),
                           torch.zeros_like(ws["s"][sl], dtype=torch.float64))
        assert bool(ok.all()), ("dense dS", p0, float(r.max()))
        dense["head"] = max(dense["head"], float(r.max()))
        ok, r = em.hop_bf16x3(ws["b"][sl], pd[em.LAYERS[1] + ".weight"], save["h"][0, sl] > 0, ws["a"][sl])
        assert bool(ok.all()), ("dense g_h2 -> g_h1", p0, float(r.max()))
        dense["hop_2_1"] = max(dense["hop_2_1"], float(r.max()))
    print(f"\nfp32 storage P={P}: {len(pts)} probes, worst ratio head {worst['head']:.3g}, hops {worst['hop']:.3g}; "
          f"dense: head {dense['head']:.3g}, g_h2 -> g_h1 {dense['hop_2_1']:.3g}")
