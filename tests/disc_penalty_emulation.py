"""What the discriminator's gradient-penalty kernels (csrc/disc.cu, snb_disc_penalty_*) compute, restated in float64
for the stage-by-stage tests (tests/test_gpu_disc_penalty_stages.py, tests/test_disc_penalty_stages_cpu.py).

- Layout: `disc_ws(..., save=1, pen=1)` as named float offsets, on top of tests/disc_emulation.py's first-order layout.
- Stage references, each from the kernel's own inputs: the penalty direction v = 2 d_reg g with its exponent, the
  tangent DiffAugment words, the tangent gathers, the InstanceNorm tangent, the second-order fold of both adjoint
  streams (`fold2_ref`, and `in_lrelu_adjoint`, its closed form on one row), the weight-gradient combine.  The GEMMs
  reuse disc_emulation's `gemm_fwd_ref` / `dgrad_ref` / `wgrad_ref` (operands rounded as tc_gemm.cuh rounds them).
- `emulate_penalty_backward`: the whole penalty backward chained from those stages, fp32 wherever the kernel stores,
  with switches that plant the defects the CPU test holds the bars to.
- PEN_BARS: the per-stage bars, about 4x the largest error measured on the H100 (DESIGN.md section 2).
"""
import math

import torch
import torch.nn.functional as F

from tests import disc_emulation as de

SLOPE = de.SLOPE


# --------------------------------------------------------------------------------------------------------------------
# workspace layout
# --------------------------------------------------------------------------------------------------------------------
def workspace_layout(imsize, n, h, w):
    """disc_ws(save = 1, pen = 1): ({name: (float offset, shape)}, total floats).  On top of the first-order buffers:
    'g' 'vt' (n, 3, h, w), 'ones' (n P_last), 'taug' (n, 16), 'dreg' (n), 'dp0' 'dp1' 'dcolp', the int32 exponent
    blocks 'ev' 'gt' 'gp' 'gu' 'gw' (6 each), and per layer 'tcol{i}' (n P, K), 'ty{i}' (cout, n, P) when an
    activation follows, 'tmean{i}' 'tq{i}' (cout, n) when an InstanceNorm does, 'dwt{i}' 'dwp{i}' (cout, K)."""
    bufs, off = de.workspace_layout(imsize, n, h, w, 1)
    layers = de.net(imsize, n, h, w)
    dy_max = max(n * y["P"] * y["cout"] for y in layers)
    dcol_max = max(n * y["P"] * y["K"] for y in layers)

    def take(name, *shape):
        nonlocal off
        bufs[name] = (off, shape)
        off = de._al(off + math.prod(shape))

    take("g", n, 3, h, w)
    take("vt", n, 3, h, w)
    take("ones", n * layers[-1]["P"])
    take("taug", n, de.AUG_FLOATS)
    take("dreg", n)
    take("dp0", dy_max)
    take("dp1", dy_max)
    take("dcolp", dcol_max)
    e0 = off
    take("exps", 5 * de.MAX_LAYERS)
    del bufs["exps"]
    for j, k in enumerate(("ev", "gt", "gp", "gu", "gw")):
        bufs[k] = (e0 + j * de.MAX_LAYERS, (de.MAX_LAYERS,))
    for i, y in enumerate(layers):
        rows = n * y["P"]
        take(f"tcol{i}", rows, y["K"])
        if y["act"]:
            take(f"ty{i}", y["cout"], n, y["P"])
        if y["in_norm"]:
            take(f"tmean{i}", y["cout"], n)
            take(f"tq{i}", y["cout"], n)
        take(f"dwt{i}", y["cout"], y["K"])
        take(f"dwp{i}", y["cout"], y["K"])
    return bufs, off


INT_BUFS = ("gexp", "ev", "gt", "gp", "gu", "gw")


def workspace_views(ws, imsize, n, h, w):
    """{name: view} of a float32 penalty workspace tensor (the exponent blocks as int32)"""
    bufs, total = workspace_layout(imsize, n, h, w)
    assert ws.dtype == torch.float32 and ws.numel() >= total
    v = {k: ws[o:o + math.prod(s)].view(*s) for k, (o, s) in bufs.items()}
    for k in INT_BUFS:
        v[k] = v[k].view(torch.int32)
    return v


def t_buffer(L, i):
    """the scratch holding layer i's scaled tangent adjoint ('dy0' for the last layer, then alternating); the primal
    adjoint is in the matching 'dp0' / 'dp1'"""
    return de.dy_buffer(L, i)


def p_buffer(L, i):
    return "dp0" if de.dy_buffer(L, i) == "dy0" else "dp1"


# --------------------------------------------------------------------------------------------------------------------
# stage references
# --------------------------------------------------------------------------------------------------------------------
def reg_ref(g):
    """reg[b] = sum g[b]^2 from the kernel's fp32 g: (ref, scale) -- every term is positive, so scale = ref"""
    r = g.double().flatten(1).square().sum(1)
    return r, r


def pen_dir_ref(g, d_reg):
    """(dreg, v, ev0), bit for bit: d_reg scaled by the power of two that puts its largest element in [2^14, 2^15),
    v = 2 dreg g in fp32 rescaled the same way, and the exponent that undoes both"""
    kd = de.pow2_exponent(d_reg.abs().max())
    dreg = de.ldexp32(d_reg.float(), kd)
    v = 2.0 * dreg.view(-1, 1, 1, 1) * g.float()
    kv = de.pow2_exponent(v.abs().max())
    return dreg, de.ldexp32(v, kv), -kd - kv


def taug_words(aug_ws, defect=None):
    """the exact words of the tangent's DiffAugment parameters from the forward's (n, 16): the call's own with the
    brightness shift 0 -> (n, 4) [enabled, 0, sat, con] and the (n, 4) box.  defect 'shift': the shift kept"""
    f = aug_ws[:, :4].clone()
    if defect != "shift":
        f[:, 1] = 0.0
    return f, aug_ws[:, 5:9]


def taug_mean_ref(vt, sat, defect=None):
    """float64 contrast mean of the tangent: over its saturation (shift 0).  defects: 'unsat' (over the unsaturated
    tangent, equal in exact arithmetic: saturation keeps every pixel's channel mean), 'shift' (the brightness shift
    kept; pass shift), 'primal' is planted by the caller (the forward's mean copied)"""
    return de.aug_mean_ref(vt, torch.zeros_like(sat), sat if defect != "unsat" else torch.ones_like(sat))


def source_index(y, device):
    """(n P, K) int64: the flat (n, cin, hin, win) index of the element each col entry of layer y copies, -1 in the
    padding"""
    n, C, H, W = y["n"], y["cin"], y["hin"], y["win"]
    idx = torch.arange(1, n * C * H * W + 1, device=device, dtype=torch.float64).view(n, C, H, W)
    return de.unfold(idx, y).round().long() - 1


def zdot_ref(ty, y, mean, rstd, tmean, tq):
    """float64 InstanceNorm tangent zd = rstd (yd - mean(yd) - z q) of the kernel's yd (ty), y, mean / rstd and its own
    mean(yd) / q, as (C, n, P), with the scale |rstd| (|yd| + |m| + |z q|)"""
    yd, y64 = ty.double(), y.double()
    mu, rs = mean.double().unsqueeze(-1), rstd.double().unsqueeze(-1)
    m, q = tmean.double().unsqueeze(-1), tq.double().unsqueeze(-1)
    z = (y64 - mu) * rs
    return rs * (yd - m - z * q), rs.abs() * (yd.abs() + m.abs() + (z * q).abs())


def in_tangent_ref(ty, y, mean, rstd, tmean):
    """float64 (tmean, tq) per row: mean(yd) and q = mean(z (yd - m)) with the kernel's m; scales mean |yd| and
    mean |z (yd - m)|"""
    yd = ty.double()
    z = (y.double() - mean.double().unsqueeze(-1)) * rstd.double().unsqueeze(-1)
    c = yd - tmean.double().unsqueeze(-1)
    return yd.mean(-1), (z * c).mean(-1), yd.abs().mean(-1), (z * c).abs().mean(-1)


def tangent_gather(layers, i, zs, yprev, mean, rstd):
    """layer i >= 1's tangent col in fp32, bit for bit, from the scaled tangent zs (C, n, P) the previous layer left:
    zs with the slope the primal value (y - mean) rstd took, zero padding"""
    y, p = layers[i], layers[i - 1]
    nv = de.normalized(yprev, mean, rstd)
    v = zs.float().transpose(0, 1)
    v = torch.where(nv > 0, v, v * SLOPE)
    return de.unfold(v.reshape(y["n"], p["cout"], y["hin"], y["win"]).contiguous(), y)


# the four sub-terms of InstanceNorm's second-order cross term rstd^2 (-a z + 3 q c z - c yc - q (gt - mean gt))
CROSS_TERMS = ("a_z", "3qcz", "c_yc", "q_gt")


def in_lrelu_adjoint(gt, gp, y, mean, rstd, yd, tmean, tq, eg=0, ex=0, drop=None, flip=None, gt_abs=None,
                     gp_abs=None):
    """the second-order fold's InstanceNorm part on (C, n, P) rows, float64: gt / gp the slope-masked folded tangent /
    primal adjoints (exponents ex - ev and eg), y the pre-norm primal, yd its tangent (exponent ev).  mean None: no
    InstanceNorm (out_p = gp, at eg).  -> (out_t, out_p, e_out, scale_t, scale_p).  drop / flip: a CROSS_TERMS name,
    that sub-term left out / with its sign flipped (planted defects).  gt_abs / gp_abs: the magnitudes of the terms
    summed into gt / gp (default |gt|, |gp|), for the error scales."""
    gt, gp = gt.double(), gp.double()
    ga = gt.abs() if gt_abs is None else gt_abs.double()
    gpa = gp.abs() if gp_abs is None else gp_abs.double()
    if mean is None:
        return gt, gp, eg, ga, gpa
    mu, rs = mean.double().unsqueeze(-1), rstd.double().unsqueeze(-1)
    z = (y.double() - mu) * rs
    yc = yd.double() - tmean.double().unsqueeze(-1)
    q = tq.double().unsqueeze(-1)
    mt, c = gt.mean(-1, keepdim=True), (gt * z).mean(-1, keepdim=True)
    mp, cp = gp.mean(-1, keepdim=True), (gp * z).mean(-1, keepdim=True)
    a = (gt * yc).mean(-1, keepdim=True)
    terms = {"a_z": -a * z, "3qcz": 3 * q * c * z, "c_yc": -c * yc, "q_gt": -q * (gt - mt)}
    cross = 0.0
    for k, t in terms.items():
        if k != drop:
            cross = cross + (-t if k == flip else t)
    cross = rs * rs * cross
    f = 2.0 ** (eg - ex)
    out_t = rs * (gt - mt - z * c)
    out_p = f * rs * (gp - mp - z * cp) + cross
    sc_t = rs * (ga + ga.mean(-1, keepdim=True) + z.abs() * (ga * z.abs()).mean(-1, keepdim=True))
    sc_p = f * rs * (gpa + gpa.mean(-1, keepdim=True) + z.abs() * (gpa * z.abs()).mean(-1, keepdim=True)) + rs * rs * (
        (ga * yc.abs()).mean(-1, keepdim=True) * z.abs() + 3 * q.abs() * (ga * z.abs()).mean(-1, keepdim=True) * z.abs()
        + (ga * z.abs()).mean(-1, keepdim=True) * yc.abs() + q.abs() * (ga + ga.mean(-1, keepdim=True)))
    return out_t, out_p, ex, sc_t, sc_p


def masked_fold(layers, i, dcol, yprev, mean, rstd):
    """layer i's col2im sum of dcol times the LeakyReLU slope of layer i - 1's fp32 normalised output (mean None: of
    its pre-norm output), as disc_fold2_kernel forms it before the InstanceNorm part: (C, n, P) float64 and |.|"""
    y = layers[i]
    n = y["n"]

    def fold(c):
        c = c.view(n, y["P"], y["K"]).transpose(1, 2)
        return F.fold(c, (y["hin"], y["win"]), 4, padding=y["pad"], stride=y["stride"]).reshape(n, y["cin"], -1)
    g, ga = fold(dcol.double()), fold(dcol.double().abs())
    mask = de.normalized(yprev, mean, rstd) > 0
    g, ga = torch.where(mask, g, g * SLOPE), torch.where(mask, ga, ga * SLOPE)
    return g.transpose(0, 1), ga.transpose(0, 1)


def fold2_ref(layers, i, dcol_t, dcol_p, yprev, mean, rstd, yd, tmean, tq, gt_in, gp_in, ev, **defect):
    """disc_fold2_kernel at layer i (into layer i - 1's output), float64 from the kernel's dcols (dcol_p None: a zero
    primal adjoint) and exponents: (out_t, out_p, e_out, scale_t, scale_p), each (C, n, P), before the rescales"""
    gt, gta = masked_fold(layers, i, dcol_t, yprev, mean, rstd)
    gp, gpa = (torch.zeros_like(gt),) * 2 if dcol_p is None else masked_fold(layers, i, dcol_p, yprev, mean, rstd)
    eg = 0 if gp_in is None else gp_in
    return in_lrelu_adjoint(gt, gp, yprev, mean, rstd, yd, tmean, tq, eg, gt_in + ev, gt_abs=gta, gp_abs=gpa,
                            **defect)


def combine_ref(dwt, dwp, et, ep, smaller=False):
    """disc_pen_combine_kernel in fp32, bit for bit: dwt 2^et + dwp 2^ep written at the larger exponent (dwp None: dwt
    alone).  -> (values, exponent).  smaller: planted defect (the smaller exponent)"""
    if dwp is None:
        return dwt.float().clone(), et
    e = min(et, ep) if smaller else max(et, ep)
    return de.ldexp32(dwt, et - e) + de.ldexp32(dwp, ep - e), e


# --------------------------------------------------------------------------------------------------------------------
# the whole penalty, chained from the stages
# --------------------------------------------------------------------------------------------------------------------
def emulate_penalty_forward(imsize, Ws, us, vs, x, training, aug, mode):
    """emulate_forward's buffers plus 'g' (grad_x sum out, as the plain backward from ones gives it) and 'reg'"""
    b = de.emulate_forward(imsize, Ws, us, vs, x, training, aug, mode)
    ones = torch.ones_like(b["out"])
    g = de.emulate_backward(dict(b), Ws, ones, mode)["d_input"]
    b["g"] = g
    b["reg"] = reg_ref(g)[0].float()
    return b


def emulate_penalty_backward(b, Ws, d_reg, mode, defect=None):
    """the gradients of sum(d_reg reg) from the penalty forward's buffers, every stage as the kernels chain them
    (fp32 where they store).  Adds 'dreg', 'vt', 'taug_f', 'taug_mean', 'tcol{i}', 'ty{i}', 'tmean{i}', 'tq{i}', 'ev',
    'gt', 'gp', 'gu' (lists), 'pt{i}' / 'pp{i}' (layer i's scaled adjoints), 'dwt{i}', 'dwp{i}', 'pdW{i}', 'pd_input'.
    defect: None or (name, arg) -- 'cross_drop' / 'cross_flip' (a CROSS_TERMS name), 'taug_mean' ('unsat' / 'primal'),
    'taug_shift', 'ev_off' (layer), 'combine_smaller', 'alpha_p' (the primal z slice at alpha^2), 'dwp_no_cs',
    'p_start_one'."""
    name, arg = defect if defect is not None else (None, None)
    layers = b["layers"]
    L, n = len(layers), layers[0]["n"]
    h, w = layers[0]["hin"], layers[0]["win"]
    dreg, vt, ev0 = pen_dir_ref(b["g"], d_reg.float())
    ev = [0] * L
    ev[0] = ev0
    b["dreg"], b["vt"] = dreg, vt
    # DiffAugment's linear part along vt
    if b["aug_f"] is None:
        tf = None
        tcol = de.unfold(vt, layers[0])
    else:
        aug_ws = torch.zeros(n, de.AUG_FLOATS, dtype=torch.float32)
        aug_ws[:, :4], aug_ws[:, 4], aug_ws[:, 5:9] = b["aug_f"], b["aug_mean"], b["box"].float()
        tf, box = taug_words(aug_ws, "shift" if name == "taug_shift" else None)
        if name == "taug_mean" and arg == "primal":
            tm = b["aug_mean"].clone()
        elif name == "taug_shift":
            tm = de.aug_mean_ref(vt, tf[:, 1], tf[:, 2])[0].float()
        else:
            tm = taug_mean_ref(vt, tf[:, 2], arg if name == "taug_mean" else None)[0].float()
        b["taug_mean"] = tm
        tcol = de.gather0_ref(layers, vt, tf, tm, box)[0].float()
    b["taug_f"] = tf
    # the tangent forward
    for i, y in enumerate(layers):
        b[f"tcol{i}"] = tcol
        if i == L - 1:
            break
        ty = de.gemm_fwd_ref(b[f"ws{i}"], tcol, b["alpha"][i], 1.0, mode)[0].float().view(y["cout"], n, y["P"])
        b[f"ty{i}"] = ty
        zsrc = ty
        if y["in_norm"]:
            tmean = ty.double().mean(-1).float()
            tq = in_tangent_ref(ty, b[f"y{i}"], b[f"mean{i}"], b[f"rstd{i}"], tmean)[1].float()
            b[f"tmean{i}"], b[f"tq{i}"] = tmean, tq
            zsrc = zdot_ref(ty, b[f"y{i}"], b[f"mean{i}"], b[f"rstd{i}"], tmean, tq)[0].float()
        k = de.pow2_exponent(zsrc.abs().max())
        ev[i + 1] = ev[i] - k + (1 if name == "ev_off" and arg == i + 1 else 0)
        tcol = tangent_gather(layers, i + 1, de.ldexp32(zsrc, k), b[f"y{i}"], b.get(f"mean{i}"), b.get(f"rstd{i}"))
    # the reverse pass over both adjoint streams
    gt, gp, gu = [0] * L, [0] * L, [0] * L
    t = torch.full((1, n * layers[-1]["P"]), 2.0 ** 14)
    gt[L - 1] = -14
    p = t.clone() if name == "p_start_one" else None
    gp[L - 1] = -14 if p is not None else 0
    dwt, dwp = [None] * L, [None] * L
    for i in range(L - 1, -1, -1):
        y = layers[i]
        b[f"pt{i}"], b[f"pp{i}"] = t, p
        dwt[i] = de.wgrad_ref(t, b[f"tcol{i}"], 1.0, mode)[0].float()
        if p is not None:
            cs = 1.0 if name == "dwp_no_cs" else de.col_scale(layers, i)
            dwp[i] = de.wgrad_ref(p, b[f"col{i}"], cs, mode)[0].float()
        alpha = b["alpha"][i]
        dcol_p = None if p is None else de.dgrad_ref(p, b[f"ws{i}"], alpha, mode,
                                                     alpha_times=2 if name == "alpha_p" else 1)[0].float()
        if i == 0:
            dx = de.fold_ref(layers, 0, dcol_p, None, None, None)[0].float()
            b["pdx"] = dx
            b["pd_input"] = de.aug_bwd_ref(dx, b["aug_f"], b["box"], gp[0], h, w)[0].float()
            break
        dcol_t = de.dgrad_ref(t, b[f"ws{i}"], alpha, mode)[0].float()
        q = i - 1
        drop = arg if name == "cross_drop" else None
        flip = arg if name == "cross_flip" else None
        ot, op, eo, _, _ = fold2_ref(layers, i, dcol_t, dcol_p, b[f"y{q}"], b.get(f"mean{q}"), b.get(f"rstd{q}"),
                                     b[f"ty{q}"], b.get(f"tmean{q}"), b.get(f"tq{q}"), gt[i],
                                     gp[i] if p is not None else None, ev[q], drop=drop, flip=flip)
        ot, op = ot.float().reshape(y["cin"], -1), op.float().reshape(y["cin"], -1)
        gu[q] = eo
        kt, kp = de.pow2_exponent(ot.abs().max()), de.pow2_exponent(op.abs().max())
        t, p = de.ldexp32(ot, kt), de.ldexp32(op, kp)
        gt[q], gp[q] = gt[i] - kt, gu[q] - kp
    b["ev"], b["gt"], b["gp"], b["gu"] = ev, gt, gp, gu
    # the weight gradients: combine, the spectral-norm correction
    for i, y in enumerate(layers):
        comb, e = combine_ref(dwt[i], dwp[i], gt[i] + ev[i], gp[i], smaller=name == "combine_smaller")
        b[f"dwt{i}"], b[f"dwp{i}"], b[f"comb{i}"], b[f"gw{i}"] = dwt[i], dwp[i], comb, e
        Wm = Ws[i].reshape(y["cout"], -1)
        part = (comb.double() * Wm.double()).sum(1).float()
        b[f"ppart{i}"] = part
        raw = comb.double()
        b[f"pdW{i}"] = de.sn_fix_ref(raw, raw.abs(), part, b["inv_sigma"][i], b[f"u{i}"], b[f"v{i}"],
                                     e)[0].float().view_as(Ws[i])
    return b


# --------------------------------------------------------------------------------------------------------------------
# bars
# --------------------------------------------------------------------------------------------------------------------
# (worst, rms) of the per-element error against the float64 reference, per stage and mode, about 4x the largest value
# measured on an H100 SXM (80 GB, 700 W) over the cases of tests/test_gpu_disc_penalty_stages.py; DESIGN.md section 2
# lists the measurements.  Units: |y - ref| / scale as each reference states it; 'tgather0' in units of 2^-24 of its
# terms' magnitude.  'ty', 'dgrad_t', 'dgrad_p', 'wgrad_p', 'wgrad_t' (the combined, corrected weight gradient) and
# 'part' (its row sums against W) come from the GEMMs; the other stages share one bar, 4x their largest over the modes.
_PEN_COMMON = {
    "reg": (7.6e-7, 3.5e-7), "taug_mean": (3.1e-7, 3.1e-7), "tgather0": (61.0, 1.7), "tmean": (4.0e-7, 6.6e-8),
    "tq": (6.2e-7, 1.2e-7), "zdot": (8.5e-7, 1.8e-7), "fold2_t": (8.3e-7, 1.1e-7), "fold2_p": (1.0e-6, 1.2e-7),
    "fold": (6.1e-7, 1.1e-7), "aug_bwd": (6.0e-7, 1.0e-7),
}
PEN_BARS = {
    "split": dict(_PEN_COMMON, ty=(1.2e-5, 2.2e-6), dgrad_t=(4.2e-6, 5.4e-7), dgrad_p=(4.4e-6, 6.5e-7),
                  wgrad_p=(8.2e-6, 2.6e-6), wgrad_t=(3.3e-5, 6.7e-6), part=(6.2e-6, 3.5e-6)),
    "f16": dict(_PEN_COMMON, ty=(4.3e-6, 7.4e-7), dgrad_t=(1.7e-6, 1.9e-7), dgrad_p=(1.8e-6, 2.3e-7),
                wgrad_p=(3.8e-6, 8.6e-7), wgrad_t=(1.9e-5, 2.8e-6), part=(2.7e-6, 1.4e-6)),
    "bf16": dict(_PEN_COMMON, ty=(3.9e-6, 6.8e-7), dgrad_t=(1.3e-6, 1.5e-7), dgrad_p=(1.5e-6, 1.9e-7),
                 wgrad_p=(2.4e-6, 8.0e-7), wgrad_t=(9.6e-6, 2.0e-6), part=(1.9e-6, 1.1e-6)),
}
