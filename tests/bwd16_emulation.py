"""References for the 16-bit training backward (sinnerf_b200/csrc/bwd16.cu, dgrad16.cu, wgrad16.cu) at one probe point,
and a CPU stand-in for it.

With the upstream gradient zero everywhere except at one point p, every gradient row the backward forms is zero except
row p, so the backward's arithmetic at p can be read back exactly through the C ABI:
  * wgrad16 forms db[n] = (1 / s) sum_q dY[q][n] from the fp16 hi plane with fp32 adds; one nonzero term, a power-of-
    two scale: db_l * s_l IS the fp16 hi plane of the layer's gradient at p, bit for bit;
  * dW_l = hi(g_l) (x) x_{l-1} / s_l: fp16 x fp16 products are exact in fp32 and every other term is zero, so each
    element is bit-exact (`wgrad_rank1`); the head rows add the hi and residual rows of the hg cell once in fp32
    (`head_rows`);
  * dS (hi and residual planes), the hg cell and the fold scratch stay in the workspace (`make_bwd16_layout`).

Checkers (all in float64, on whatever device the tensors live; each returns (ok, ratio) per element, ratio = error /
allowance, an element passes at ratio <= 1):
  * `head_ds` / `head_hg`: the head kernel's dS and hg cells, hi + lo, against float64 from g_raw, raw and G;
  * `hop_chain`: hops of dgrad16 chained in float64 from an exact start, with the absolute-value chain A and the
    bound B that follow from counting the roundings (see `hop_chain`); used from the observed dS down to g_h4 (the
    residual segment, where lo is never observable) and for each hi-only hop from the kernel's own observed input;
  * `wgrad_rank1` / `head_rows`: the bit-exact rank-1 weight gradients;
  * `unfold`: unfold_grads_kernel (field_bwd.cu) from the observed dW' / db'.

`StandIn` restates field_backward16 (and field_backward16_sigma) for small P in torch float32 / float16, with the
operand splits, the power-of-two scales and the wgrad slicing written out, so that `StandIn(defect=n)` plants one of
the defects in DEFECTS.  tests/test_bwd16_chain_cpu.py shows every checker passing on the faithful stand-in and
failing on the defect aimed at it, and which defects the aggregate per-tensor bars let through.
"""
from __future__ import annotations

import numpy as np
import torch

U32 = 2.0 ** -24                 # unit roundoff of fp32
MIN32 = 2.0 ** -126              # fp32's smallest normal
A16_TARGET = 16384.0             # kA16Target
SM_H100 = 132                    # SMs of the H100 SXM, which sets the wgrad slicing of the stand-in

DEFECTS = {
    1: "dgrad16 ignores dY_lo at every hop",
    2: "trunk_backward16 ends the residual chain one hop early (lo_out = l - 1 >= 5)",
    3: "a hi-only hop reads the stale residual plane (lo_in = l >= 3)",
    4: "head_bwd16_kernel writes the hg residual features 4..7 as zero",
    5: "dgrad16 drops the W-lo product",
    6: "ds_lo is written with the wrong sign",
    7: "wgrad16 skips the bias sum of the last 128-column block",
    8: "wgrad16 skips the last tile of one slice",
}

# the wgmma accumulations of one dgrad16 output: 3 products (2 without dY_lo) per K16 step of the reduction.  Each is
# one fp32 accumulation into a running sum bounded by A (truncation: up to one fp32 ulp, 2 U32 relative)
def wgmma_steps(N, lo_in):
    return (3 if lo_in else 2) * (N // 16)


# --------------------------------------------------------------------------------------------------------------------
# rounding helpers
# --------------------------------------------------------------------------------------------------------------------
def rn16(x):
    """float -> float64 value of its round-to-nearest fp16 form, saturated at +-65504 (cvt.rn.satfinite.f16)."""
    return x.float().clamp(-65504.0, 65504.0).half().double()


def ulp16(v):
    """Spacing of fp16 at |v| (v >= 0, float64): 2^(floor(log2 v) - 10) in the normal range, 2^-24 below 2^-14.
    The exponent comes from frexp, which is exact; log2 on CUDA can return 5.999... for 64."""
    e = torch.frexp(v.double().clamp_min(2.0 ** -14)).exponent         # v = m 2^e, m in [0.5, 1)
    return torch.exp2((e - 11).double())


def split16(W):
    """(Wh, Wl) float64: the fp16 hi + lo split of an fp32 weight matrix (f16_split_pair in dgrad16.cu)."""
    Wh = rn16(W)
    return Wh, rn16(W.double() - Wh)


def pow2_scale(bound, target=A16_TARGET):
    """act16.cuh pow2_scale: the largest power of two s with s * bound <= target, from float32 target / bound."""
    b = np.float32(bound)
    if not (b > 0) or not (b < np.float32(3.0e38)):
        return 1.0
    _, e = np.frexp(np.float32(target) / b)
    return float(2.0 ** min(max(int(e) - 1, -100), 100))


def dgrad_scale(amax_in, s_in, l1, amax_g=None, evec_max=None):
    """s_out of dgrad16_kernel, its bound formed in float32 as the kernel forms it."""
    f = np.float32
    bound = f(f(amax_in) / f(s_in)) * f(l1)
    if amax_g is not None:
        bound = f(bound + f(amax_g) * f(evec_max))
    return pow2_scale(bound)


def head_scales(amax_g, wr_l1):
    """(s_hg, s_ds) of head_bwd16_kernel."""
    f = np.float32
    return pow2_scale(amax_g), pow2_scale(f(f(0.2505) * f(wr_l1)) * f(amax_g))


def col_l1(W):
    """max column L1 norm of an fp32 matrix, summed in fp32 over rows (bwd16_prepare_kernel)."""
    return float(W.float().abs().sum(0).max())


# --------------------------------------------------------------------------------------------------------------------
# checkers
# --------------------------------------------------------------------------------------------------------------------
def _verdict(err, allow):
    ratio = err / allow.clamp_min(1e-300)
    return ratio <= 1.0, ratio


def g_pre_rgb64(g_raw, raw):
    """float64 [g_pre_rgb (3), g_sigma] of the head from g_raw and raw (n, 4), and the bound on |fp32 - float64| of the
    kernel's g_pre_rgb: 0.2505 (1 - t^2) with t = (2 out - 1) / 1.002 takes ~6 fp32 roundings, and 1 - t^2 loses
    its relative accuracy as t -> 1, so the bound is absolute: 8 U32 of 0.2505 |g|, plus 4 U32 relative."""
    g_raw, raw = g_raw.double(), raw.double()
    t = (2.0 * raw[:, :3] - 1.0) / 1.002
    gp = g_raw[:, :3] * 0.2505 * (1.0 - t * t)
    egp = 8 * U32 * 0.2505 * g_raw[:, :3].abs() + 4 * U32 * gp.abs()
    return torch.cat([gp, g_raw[:, 3:4]], 1), torch.cat([egp, torch.zeros_like(egp[:, :1])], 1)


def head_ds(g_raw, raw, G, Wr, s_ds, hi, lo):
    """dS planes (hi, lo: (n,128) decoded, scaled by s_ds) against float64 (W_rgb^T g_pre) act'(G) s_ds.
    Kernel: dg = 3 products and 2 adds in fp32 (3 U32 of sum |W_rgb g_pre|); der = 1 - __expf(-G): __expf is off by at
    most (2 + 1.173 |G|) ulp (CUDA C Programming Guide, intrinsic functions), the subtraction one U32; dg der s_ds two
    more roundings; hi + lo stands for that fp32 value within half an fp16 ulp of lo."""
    gp, egp = g_pre_rgb64(g_raw, raw)
    gp, egp = gp[:, :3], egp[:, :3]
    Wr = Wr.double()
    G = G.double()
    dg = gp @ Wr
    edg = egp @ Wr.abs() + 3 * U32 * (gp.abs() @ Wr.abs())
    e = torch.exp(-G)
    der = -torch.expm1(-G)
    eder = (2.0 + 1.173 * G) * 2 * U32 * e + U32 * der
    want = dg * der * s_ds
    allow = s_ds * (edg * der + (dg.abs() + edg) * eder) + 2 * U32 * want.abs()
    allow = allow * (1 + 1e-6) + 0.5 * ulp16(lo.abs())
    ok, ratio = _verdict((hi + lo - want).abs(), allow)
    structural = lo.abs() <= 0.5 * ulp16(hi.abs())                      # hi is the nearest fp16 of hi + lo
    return ok & structural, torch.where(structural, ratio, torch.full_like(ratio, float("inf")))


def head_hg(g_raw, raw, s_hg, cell):
    """The head-gradient cell (n, 8) decoded: features 0..3 the fp16 hi of [g_pre_rgb, g_sigma] s_hg, 4..7 their
    residuals.  g_sigma s_hg is exact (power of two), so its hi + lo is within half an fp16 ulp of lo."""
    gp, egp = g_pre_rgb64(g_raw, raw)
    hi, lo = cell[:, :4], cell[:, 4:]
    want = gp * s_hg
    allow = egp * s_hg * (1 + 1e-6) + 0.5 * ulp16(lo.abs())
    ok, ratio = _verdict((hi + lo - want).abs(), allow)
    structural = lo.abs() <= 0.5 * ulp16(hi.abs())
    return ok & structural, torch.where(structural, ratio, torch.full_like(ratio, float("inf")))


def hop_chain(r0, B0, hops, kappa=1.0):
    """Hops of dgrad16 chained in float64.  r0 (N0,): the exact start (true gradient x s_in, float64); B0 (N0,): the
    bound on |kernel's input - r0| (0 when the start is observed).  hops: dicts with
        W (N, K) fp32 weight block the hop multiplies by, mask (K,) bool, s_in, s_out, lo_in (dY has its residual
        plane), lo_out (dX gets one), extra (K,) float64 or None (the sigma-head term, true units x s_out), hi (K,)
        the observed fp16 hi plane of the output (scaled by s_out).
    Per hop, with We = Wh + Wl the kernel's split weights and ratio = s_out / s_in:
        r' = (r @ We) ratio + extra,  masked;   A' = (A @ |We|) ratio + |extra|
        B' = ratio [B @ |We| + (2^-22 [lo_in: the missing lo Wl product, |lo| <= 2^-11 |y|, |Wl| <= 2^-11 |W|]
                               + 2 U32 kappa wgmma_steps [one truncated fp32 accumulation per wgmma]) (A @ |We|)]
             + U32 |r'| [the fmaf of the sigma term]
    and the output passes at |hi - r'| <= ulp16(|r'| + B') / 2 + B' (masked outputs exactly 0).  When the output
    keeps its residual plane, the next hop's input is hi + lo, within 2^-22 |x| + 2^-25 of the kernel's fp32 x (half
    an fp16 ulp of lo, subnormal below 2^-14): B'' = B' + 2^-22 (|r'| + B') + 2^-25.
    -> [(ok, ratio, used_B)] per hop, used_B = max(0, |hi - r'| - half ulp) / B'."""
    r, B = r0.double(), B0.double()
    A = r.abs() + B
    out = []
    for h in hops:
        Wh, Wl = split16(h["W"])
        We = Wh + Wl
        Wa = We.abs()
        ratio = h["s_out"] / h["s_in"]
        m = h["mask"].double()
        ex = torch.zeros_like(m) if h.get("extra") is None else h["extra"].double()
        AW = A @ Wa
        r = ((r @ We) * ratio + ex) * m
        local = ((2.0 ** -22 if h["lo_in"] else 0.0) + 2 * U32 * kappa * wgmma_steps(Wa.shape[0], h["lo_in"])) * AW
        B = ((B @ Wa + local) * ratio + U32 * r.abs()) * m
        A = (AW * ratio + ex.abs()) * m
        hi = h["hi"].double()
        half = 0.5 * ulp16(r.abs() + B)
        err = (hi - r).abs()
        ok, ratio_ = _verdict(err, torch.where(m > 0, half + B, torch.zeros_like(B)))
        ok = torch.where(m > 0, ok, hi == 0)
        ratio_ = torch.where(m > 0, ratio_, torch.where(hi == 0, torch.zeros_like(ratio_), torch.full_like(ratio_, float("inf"))))
        # the share of B an error uses beyond the half ulp of the hi rounding: ~0 means a ratio near 1 is that half ulp
        # (a rounding tie), not the accumulation model
        used_B = ((err - half).clamp_min(0) / B.clamp_min(1e-300)) * m
        out.append((ok, ratio_, used_B))
        if h["lo_out"]:
            B = B + 2.0 ** -22 * (r.abs() + B) + 2.0 ** -25 * m
    return out


def wgrad_rank1(hi, x, s, dW, db=None, hi_plane=None):
    """dW (N, K) fp32 of a single-probe wgrad16 against hi (N,) (x) x (K,) / s: bit-exact -- a product of two fp16 values
    is exact in fp32 and the power-of-two scale only moves the exponent -- except where the value falls below fp32's
    normal range, where the division may round (or flush) by less than 2^-126.  db (N,), if given: hi / s exactly.
    hi_plane (N,), if given: the hi plane observed in the workspace, which hi (decoded from db) must equal.
    -> (ok (N, K), n_bad)"""
    want = hi.double()[:, None] * x.double()[None, :] / s
    got = dW.double()
    ok = (got == want.float().double()) | ((want.abs() < MIN32) & ((got - want).abs() < MIN32))
    if db is not None:
        ok = ok & (db.double() == (hi.double() / s).float().double())[:, None]
    if hi_plane is not None:
        ok = ok & (hi.double() == hi_plane.double())[:, None]
    return ok, int((~ok).sum())


def head_rows(hi, lo, x, s, dW):
    """A head row of wgrad16 (dW_sigma or one row of dW_rgb) at one probe: fp32(hi x + lo x) / s -- the two exact
    products added once in fp32 (row r + row r + 4 of the hg operand), then the power-of-two scale."""
    want = (float(hi) * x.double() + float(lo) * x.double()).float().double() / s
    got = dW.double()
    ok = (got == want.float().double()) | ((want.abs() < MIN32) & ((got - want).abs() < MIN32))
    return ok, int((~ok).sum())


def unfold(dWp, dbp, Wd, Wf, bf, dWd, dbd, dWf, dbf):
    """unfold_grads_kernel from its observed inputs dW' (128, 256) and db' (128): sequential fmaf chains of n terms in
    fp32 onto one more term, each fmaf one rounding of a partial sum bounded by the sum of |terms|: n U32 sum |terms|
    (n = 257 for dWd, 128 for dWf and dbf); dbd = db' exactly.  dWd is Wd's gradient columns [0, 256).
    -> {name: (ok, ratio)}"""
    dWp, dbp = dWp.double(), dbp.double()
    Wd0, Wf, bf = Wd[:, :256].double(), Wf.double(), bf.double()
    res = {}
    for name, want, absw, n, got in (
            ("dWd", dWp @ Wf.t() + dbp[:, None] * bf[None, :], dWp.abs() @ Wf.abs().t() + dbp.abs()[:, None] * bf.abs()[None, :], 257, dWd),
            ("dWf", Wd0.t() @ dWp, Wd0.abs().t() @ dWp.abs(), 128, dWf),
            ("dbf", Wd0.t() @ dbp, Wd0.abs().t() @ dbp.abs(), 128, dbf)):
        res[name] = _verdict((got.double() - want).abs(), (n + 1) * U32 * absw + 2.0 ** -149)
    ok = dbd.double() == dbp
    res["dbd"] = (ok, torch.where(ok, torch.zeros_like(dbp), torch.full_like(dbp, float("inf"))))
    return res


# --------------------------------------------------------------------------------------------------------------------
# CPU stand-in
# --------------------------------------------------------------------------------------------------------------------
LAYERS = [f"xyz_encoding_{i + 1}.0" for i in range(8)]


def slice_tiles(n_tiles, blocks, sm=SM_H100):
    """[(t_begin, t_end)] of the split-P slices of a wgrad16 launch with `blocks` CTAs per slice (launch_wgrad16)."""
    ctas = min((sm + blocks - 1) // blocks, n_tiles)
    tpc = (n_tiles + ctas - 1) // ctas
    ctas = (n_tiles + tpc - 1) // tpc
    return [(x * tpc, min((x + 1) * tpc, n_tiles)) for x in range(ctas)]


class StandIn:
    """field_backward16 / field_backward16_sigma on small P, in torch float32 / float16 on the CPU, with one planted
    defect (DEFECTS) or none.  Inputs as the library takes them: p {name: fp32}, the act16 tensors decoded row-major
    (enc (P,63), dir (P,27), H[0..7] (P,256), G (P,128) fp16 values; M[0..7] (P,256) bool ReLU masks).
    backward() returns (grads {name: fp32}, ws) where ws holds what the library's workspace holds afterwards: 'ds',
    'ds_lo', 'hg' (P, 8), 'dya', 'dyb', 'dya_lo', 'dyb_lo', 'fold_W', 'fold_dW', 'fold_db', 'scale' {name: float}
    and, for the checks, 'planes' {l: (hi, lo)} of every gradient the chain formed (l = 1..8 for g_h_l)."""

    def __init__(self, defect=None, sm=SM_H100):
        assert defect is None or defect in DEFECTS
        self.defect, self.sm = defect, sm

    # ---- wgrad16: dW += dY^T X / s, db += colsum(dY) / s over the slices of the launch
    def wgrad(self, dY, X, s, blocks, with_bias):
        P = dY.shape[0]
        n_tiles = (P + 127) // 128 * 128 // 32
        keep = torch.ones(P, dtype=torch.bool)
        if self.defect == 8:
            sl = slice_tiles(n_tiles, blocks, self.sm)
            if len(sl) > 1 and sl[1][1] - sl[1][0] > 1:
                t = sl[1][1] - 1
                keep[t * 32:(t + 1) * 32] = False
        dY = dY.double() * keep[:, None]
        dW = (dY.t() @ X.double() / s).float()
        db = (dY.sum(0) / s).float() if with_bias else None
        if with_bias and self.defect == 7 and dY.shape[1] == 256:
            db[128:] = 0
        return dW, db

    # ---- dgrad16: one hop
    def hop(self, hi, lo, W, mask, s_in, amax_in, l1, extra=None, evec=None, amax_g=None, evec_max=None, lo_out=True):
        s_out = dgrad_scale(amax_in, s_in, l1, amax_g if extra is not None else None, evec_max)
        Wh, Wl = split16(W)
        Wh, Wl = Wh.float(), Wl.float()
        if self.defect == 5:
            Wl = torch.zeros_like(Wl)
        use_lo = lo is not None and self.defect != 1
        acc = (hi.float() + lo.float()) @ Wh if use_lo else hi.float() @ Wh
        acc = acc + hi.float() @ Wl
        x = acc * np.float32(s_out / s_in)
        if extra is not None:
            x = x + (extra.float() * np.float32(s_out))[:, None] * evec.float()[None, :]
        x = torch.where(mask, x, torch.zeros_like(x))
        h = x.clamp(-65504, 65504).half().float()
        lo_o = (x - h).half().float() if lo_out else None
        return h, lo_o, s_out, float(x.abs().max())

    def backward(self, p, a, g_raw, raw, sigma_only=False, g_sigma=None):
        f = np.float32
        p = {k: v.float() for k, v in p.items()}
        grads = {k: torch.zeros_like(v) for k, v in p.items()}
        sc, planes = {}, {}
        P = a["H"][0].shape[0]
        Wfold = (p["dir_encoding.0.weight"][:, :256].double() @ p["xyz_encoding_final.weight"].double()).float()
        l1 = {l: col_l1(p[LAYERS[l - 1] + ".weight"][:, 63:] if l == 5 else p[LAYERS[l - 1] + ".weight"]) for l in range(2, 9)}
        ws_ = p["sigma.weight"][0]
        evec_max = float(ws_.abs().max())
        ws = {}
        if not sigma_only:
            amax_g = float(g_raw.abs().max())
            Wr = p["rgb.0.weight"]
            wr_l1 = float(Wr.abs().sum(0).max())
            s_hg, s_ds = head_scales(amax_g, wr_l1)
            t = (f(2) * raw[:, :3].float() - 1) * f(1 / 1.002)
            gp = g_raw[:, :3].float() * f(0.2505) * (1 - t * t)
            hv = torch.cat([gp, g_raw[:, 3:4].float()], 1) * f(s_hg)
            hgh = hv.half().float()
            hgl = torch.zeros_like(hgh) if self.defect == 4 else (hv - hgh).half().float()
            der = 1 - torch.exp(-a["G"].float())
            ds = (gp @ Wr) * der * f(s_ds)
            dsh = ds.half().float()
            dsl = ((dsh - ds) if self.defect == 6 else (ds - dsh)).half().float()
            ws.update(ds=dsh, ds_lo=dsl, hg=torch.cat([hgh, hgl], 1))
            grads["rgb.0.bias"] += gp.sum(0)
            grads["sigma.bias"] += g_raw[:, 3].float().sum()
            # direction layer: dW', db' and dWd[:, 256:] from the dS hi plane; the head rows from hg (hi + lo)
            dWp, dbp = self.wgrad(dsh, a["H"][7], s_ds, 2, True)
            dWdir, _ = self.wgrad(dsh, a["dir"], s_ds, 1, False)
            hgs = (hgh + hgl).double()
            grads["sigma.weight"] += ((hgs[:, 3:4].t() @ a["H"][7].double()) / s_hg).float()
            grads["rgb.0.weight"] += ((hgs[:, :3].t() @ a["G"].double()) / s_hg).float()
            Wd, Wf, bf = p["dir_encoding.0.weight"], p["xyz_encoding_final.weight"], p["xyz_encoding_final.bias"]
            grads["dir_encoding.0.weight"][:, 256:] += dWdir
            grads["dir_encoding.0.weight"][:, :256] += (dWp.double() @ Wf.double().t() + dbp.double()[:, None] * bf.double()[None, :]).float()
            grads["xyz_encoding_final.weight"] += (Wd[:, :256].double().t() @ dWp.double()).float()
            grads["xyz_encoding_final.bias"] += (Wd[:, :256].double().t() @ dbp.double()).float()
            grads["dir_encoding.0.bias"] += dbp
            ws.update(fold_W=Wfold, fold_dW=dWp, fold_db=dbp)
            sc.update(hg=s_hg, ds=s_ds)
            h, lo, s8, amax = self.hop(dsh, dsl, Wfold, a["M"][7], s_ds, float(ds.abs().max()), col_l1(Wfold),
                                       extra=g_raw[:, 3], evec=ws_, amax_g=amax_g, evec_max=evec_max)
        else:
            amax_g = float(g_sigma.abs().max())
            s_hg = pow2_scale(amax_g)
            s8 = pow2_scale(f(amax_g) * f(evec_max))
            hv = g_sigma.float() * f(s_hg)
            hgh = hv.half().float()
            hgl = (hv - hgh).half().float()
            z = torch.zeros(P, 2)
            ws["hg"] = torch.cat([z, torch.zeros(P, 1), hgh[:, None], z, torch.zeros(P, 1), hgl[:, None]], 1)
            grads["sigma.bias"] += g_sigma.float().sum()
            grads["sigma.weight"] += (((hgh + hgl).double()[:, None].t() @ a["H"][7].double()) / s_hg).float()
            x = (g_sigma.float() * f(s8))[:, None] * ws_[None, :]
            x = torch.where(a["M"][7], x, torch.zeros_like(x))
            h = x.half().float()
            lo = (x - h).half().float()
            amax = float(x.abs().max())
            sc["hg"] = s_hg
        # trunk: the same ping-pong as trunk_backward16
        sc[8] = s8
        planes[8] = (h, lo)
        cur, cur_lo = "dya", "dya_lo"
        nxt, nxt_lo = "dyb", "dyb_lo"
        ws[cur], ws[cur_lo] = h, lo
        ws.setdefault(nxt, torch.zeros_like(h))
        ws.setdefault(nxt_lo, torch.zeros_like(h))
        for l in range(8, 1, -1):                         # g_h_l -> g_h_{l-1}; wgrad of layer l
            s = sc[l]
            hi = ws[cur]
            x = torch.cat([a["enc"], a["H"][3]], 1) if l == 5 else a["H"][l - 2]
            dW, db = self.wgrad(hi, x, s, 2, True)
            grads[LAYERS[l - 1] + ".weight"] += dW
            grads[LAYERS[l - 1] + ".bias"] += db
            lo_in = l - 1 >= (3 if self.defect == 3 else 4)          # the library's l - 1 >= 4 (0-based l)
            lo_out = l - 2 >= (5 if self.defect == 2 else 4)
            W = p[LAYERS[l - 1] + ".weight"]
            W = W[:, 63:] if l == 5 else W
            h, lo, s_o, amax = self.hop(hi, ws[cur_lo] if lo_in else None, W, a["M"][l - 2], s, amax, l1[l], lo_out=lo_out)
            sc[l - 1] = s_o
            planes[l - 1] = (h, lo)
            ws[nxt] = h
            if lo_out:
                ws[nxt_lo] = lo
            cur, nxt, cur_lo, nxt_lo = nxt, cur, nxt_lo, cur_lo
        dW, db = self.wgrad(ws[cur], a["enc"], sc[1], 2, True)
        grads[LAYERS[0] + ".weight"] += dW
        grads[LAYERS[0] + ".bias"] += db
        ws["scale"], ws["planes"] = sc, planes
        return grads, ws


def head_bias(g_row, raw_row, s_hg, cell, db_rgb, db_sigma):
    """The head biases at one probe: one nonzero term each, so db_sigma is g_sigma exactly and db_rgb is the kernel's
    fp32 g_pre_rgb (within g_pre_rgb64's bound of float64); the hg cell's hi and residual features are that fp32 value
    times s_hg rounded to fp16 and its residual rounded to fp16, bit for bit.  raw_row / db_rgb None: a sigma-only pass
    (rgb features of hg zero).  -> (ok (4,), ratio (4,))"""
    ok = torch.ones(4, dtype=torch.bool)
    ratio = torch.zeros(4, dtype=torch.float64)
    v = torch.zeros(4, dtype=torch.float32)
    v[3] = g_row[3].float()
    ok[3] = float(db_sigma.reshape(-1)[0]) == float(g_row[3])
    if raw_row is not None:
        gp, egp = g_pre_rgb64(g_row[None].double(), raw_row[None].double())
        e = (db_rgb.double() - gp[0, :3]).abs()
        ratio[:3] = e / egp[0, :3].clamp_min(1e-300)
        ok[:3] = ratio[:3] <= 1
        v[:3] = db_rgb.float()
    hv = v * float(s_hg)
    hi = hv.half().float()
    lo = (hv - hi).half().float()
    exact = (cell[:4].float() == hi) & (cell[4:].float() == lo)
    ok = ok & exact
    return ok, torch.where(ok, ratio, torch.full_like(ratio, float("inf")))


def fold_w(Wp, Wd, Wf):
    """W' = Wd[:, :256] Wf as fold_weights_kernel forms it: a chain of 256 fmaf, each one rounding of a partial sum
    bounded by sum |Wd||Wf|: |W' - float64| <= 257 U32 sum |Wd||Wf|.  -> (ok, ratio)"""
    want = Wd[:, :256].double() @ Wf.double()
    allow = 257 * U32 * (Wd[:, :256].double().abs() @ Wf.double().abs()) + 2.0 ** -149
    return _verdict((Wp.double() - want).abs(), allow)


def check_probe(grads, ws, p, a, raw, g_raw, pt, sigma_only=False, kappa=1.0):
    """Every single-probe checker on one backward of the 16-bit arm: {checker: worst ratio (inf = a structural or
    exact check failed)}; for the hop checkers also '<name>_B', the largest share of the bound B an error needed beyond
    the half ulp of its hi rounding.  grads / ws / a / raw / g_raw as StandIn.backward returns and takes them, rows
    indexed by pt.  Used identically on the stand-in and on the library's outputs."""
    sc = ws["scale"]
    row = lambda t: t[pt]
    worst = {}

    def note(name, res):
        r = max([float(x[1].max()) if x[1].numel() else 0.0 for x in res])
        worst[name] = max(worst.get(name, 0.0), r)
        if len(res[0]) == 3:
            worst[name + "_B"] = max(worst.get(name + "_B", 0.0), max(float(x[2].max()) for x in res))

    hi = {l: grads[LAYERS[l - 1] + ".bias"].double() * sc[l] for l in range(1, 9)}
    if not sigma_only:
        note("head", [head_ds(row(g_raw)[None], row(raw)[None], row(a["G"])[None], p["rgb.0.weight"], sc["ds"],
                                 row(ws["ds"]).double()[None], row(ws["ds_lo"]).double()[None])])
    note("hg", [head_hg_of(g_raw, raw, ws, sc, pt, sigma_only)])
    note("bias", [head_bias(row(g_raw), None if sigma_only else row(raw), sc["hg"], row(ws["hg"]),
                            None if sigma_only else grads["rgb.0.bias"], grads["sigma.bias"])])
    # residual segment: from the observed dS (hi + lo) or the sigma head's exact g_h8, down to g_h4
    hops = []
    if not sigma_only:
        ds = (row(ws["ds"]) + row(ws["ds_lo"])).double()
        r0, B0 = ds, torch.zeros_like(ds)
        note("fold", [fold_w(ws["fold_W"], p["dir_encoding.0.weight"], p["xyz_encoding_final.weight"])])
        hops.append(dict(W=ws["fold_W"], mask=row(a["M"][7]), s_in=sc["ds"], s_out=sc[8], lo_in=True, lo_out=True,
                         extra=float(row(g_raw)[3]) * sc[8] * p["sigma.weight"][0].double(), hi=hi[8]))
    else:
        gs = float(row(g_raw)[3])
        x = torch.where(row(a["M"][7]), (torch.tensor(gs).float() * float(sc[8])) * p["sigma.weight"][0].float(),
                        torch.zeros(256))
        worst["sigma_head"] = 0.0 if torch.equal(hi[8], x.half().double()) else float("inf")
        r0 = x.double()
        B0 = U32 * r0.abs() + 2.0 ** -22 * r0.abs() + 2.0 ** -25
    for l in (8, 7, 6, 5):
        W = p[LAYERS[l - 1] + ".weight"]
        hops.append(dict(W=W[:, 63:] if l == 5 else W, mask=row(a["M"][l - 2]), s_in=sc[l], s_out=sc[l - 1], lo_in=True,
                         lo_out=l - 1 >= 5, hi=hi[l - 1]))
    note("residual", hop_chain(r0, B0, hops, kappa))
    # after the call dya_lo / dyb_lo still hold the residuals of g_h6 / g_h5 (trunk_backward16's ping-pong): at the
    # probe they must be residuals of those hi planes, and the hops g_h6 -> g_h5 -> g_h4 run from them exactly
    for l, plane in ((6, "dya_lo"), (5, "dyb_lo")):
        lo = row(ws[plane]).double()
        if not bool((lo.abs() <= 0.5 * ulp16(hi[l].abs())).all()):
            worst["residual"] = float("inf")
        W = p[LAYERS[l - 1] + ".weight"]
        hop = dict(W=W[:, 63:] if l == 5 else W, mask=row(a["M"][l - 2]), s_in=sc[l], s_out=sc[l - 1], lo_in=True,
                   lo_out=False, hi=hi[l - 1])
        note("residual", hop_chain(hi[l] + lo, torch.zeros(256, dtype=torch.float64), [hop], kappa))
    # hi-only hops, each from the kernel's own observed input
    for l in (4, 3, 2):
        W = p[LAYERS[l - 1] + ".weight"]
        hop = dict(W=W, mask=row(a["M"][l - 2]), s_in=sc[l], s_out=sc[l - 1], lo_in=False, lo_out=False, hi=hi[l - 1])
        note("hi_only", hop_chain(hi[l], torch.zeros(256, dtype=torch.float64), [hop], kappa))
    # weight gradients, bit-exact rank-1
    bad = 0
    for l in range(1, 9):
        x = row(a["enc"]) if l == 1 else (torch.cat([row(a["enc"]), row(a["H"][3])]) if l == 5 else row(a["H"][l - 2]))
        plane = {1: ws["dyb"], 2: ws["dya"]}.get(l)
        bad += wgrad_rank1(hi[l], x, sc[l], grads[LAYERS[l - 1] + ".weight"], grads[LAYERS[l - 1] + ".bias"],
                              None if plane is None else row(plane))[1]
    hg = row(ws["hg"]).double()
    bad += head_rows(hg[3], hg[7], row(a["H"][7]), sc["hg"], grads["sigma.weight"][0])[1]
    if not sigma_only:
        dsh = row(ws["ds"]).double()
        bad += wgrad_rank1(dsh, row(a["H"][7]), sc["ds"], ws["fold_dW"], ws["fold_db"])[1]
        bad += wgrad_rank1(dsh, row(a["dir"]), sc["ds"], grads["dir_encoding.0.weight"][:, 256:])[1]
        for c in range(3):
            bad += head_rows(hg[c], hg[4 + c], row(a["G"]), sc["hg"], grads["rgb.0.weight"][c])[1]
        res = unfold(ws["fold_dW"], ws["fold_db"], p["dir_encoding.0.weight"], p["xyz_encoding_final.weight"],
                        p["xyz_encoding_final.bias"], grads["dir_encoding.0.weight"][:, :256], grads["dir_encoding.0.bias"],
                        grads["xyz_encoding_final.weight"], grads["xyz_encoding_final.bias"])
        note("unfold", list(res.values()))
    worst["wgrad"] = float("inf") if bad else 0.0
    return worst


def head_hg_of(g_raw, raw, ws, sc, pt, sigma_only):
    cell = ws["hg"][pt].double()[None]
    if sigma_only:
        g = torch.zeros(1, 4, dtype=torch.float64)
        g[0, 3] = g_raw[pt, 3]
        return head_hg(g, torch.full((1, 4), 0.5, dtype=torch.float64), sc["hg"], cell)
    return head_hg(g_raw[pt][None], raw[pt][None], sc["hg"], cell)



BF16_SPLIT = 3 * 2.0 ** -18      # dgrad_tc's bf16 split: |y - yh - yl|, |W - Wh - Wl| and the missing yl Wl, each <= 2^-18


def hop_bf16x3(y, W, mask, got, extra=None, kappa=1.0):
    """One hop of dgrad_tc (fp32 storage) from its own exact fp32 input y (n, N): dY and W split into bf16 hi + lo,
    products yh Wh + yl Wh + yh Wl, fp32 accumulation (one truncated accumulation per wgmma, 3 per K16 step), the
    sigma term added in fp32, output stored in fp32:
        |got - r| <= (3 2^-18 + 2 U32 kappa wgmma_steps) (|y| @ |W|) + U32 |r|,   masked outputs exactly 0.
    -> (ok, ratio)"""
    y, Wd = y.double(), W.double()
    m = mask.double()
    ex = torch.zeros_like(m) if extra is None else extra.double()
    r = (y @ Wd + ex) * m
    A = y.abs() @ Wd.abs() + ex.abs()
    allow = ((BF16_SPLIT + 2 * U32 * kappa * wgmma_steps(W.shape[0], True)) * A + U32 * r.abs()) * m
    err = (got.double() - r).abs()
    ok, ratio = _verdict(err, allow)
    ok = torch.where(m > 0, ok, got == 0)
    ratio = torch.where(m > 0, ratio, torch.where(got == 0, torch.zeros_like(ratio), torch.full_like(ratio, float("inf"))))
    return ok, ratio


def plane_scales(state, Wfold, params, sigma_only=False):
    """Every ST_SCALE_* of the 16-bit backward recomputed on the host from the state block's own maxima and bound
    ingredients, as the kernels form them in fp32 (state: the 64 floats of the workspace's state block).  The sigma
    term of the first dgrad bound is added either rounded once or as one fmaf (the compiler may contract it).
    Also returns the ingredients recomputed from the weights: {name: (state value, host value, allowance)}.
    -> (scales {name: [allowed values]}, ingredients)"""
    st = state.float()
    amax = lambda i: float(st[i])      # the maxima are raised as uint32 bit patterns of non-negative floats
    f = np.float32
    amax_g, evec_max, wr_l1 = amax(0), float(st[29]), float(st[30])
    sc = {}
    if not sigma_only:
        s_hg, s_ds = head_scales(amax_g, wr_l1)
        sc["hg"], sc["ds"] = [s_hg], [s_ds]
        base = f(f(amax(1)) / f(float(st[11]))) * f(float(st[20]))
        two = [pow2_scale(f(base + f(amax_g) * f(evec_max))),
               pow2_scale(float(np.float32(np.float64(base) + np.float64(f(amax_g)) * np.float64(f(evec_max)))))]
        sc[8] = two
    else:
        sc["hg"] = [pow2_scale(amax_g)]
        sc[8] = [pow2_scale(f(amax_g) * f(evec_max))]
    for l in range(8, 1, -1):
        sc[l - 1] = [dgrad_scale(amax(2 + l - 1), float(st[12 + l - 1]), float(st[21 + l - 1]))]
    ing = {"evec_max": (evec_max, float(params["sigma.weight"].abs().max()), 0.0)}
    for l in range(2, 9):
        W = params[LAYERS[l - 1] + ".weight"]
        W = W[:, 63:] if l == 5 else W
        ing[f"l1_{l}"] = (float(st[21 + l - 1]), float(W.double().abs().sum(0).max()), 256 * U32 * float(W.double().abs().sum(0).max()))
    if not sigma_only:
        ing["l1_fold"] = (float(st[20]), float(Wfold.double().abs().sum(0).max()), 128 * U32 * float(Wfold.double().abs().sum(0).max()))
        Wr = params["rgb.0.weight"].double()
        ing["wr_l1"] = (wr_l1, float(Wr.abs().sum(0).max()), 3 * U32 * float(Wr.abs().sum(0).max()))
    return sc, ing
