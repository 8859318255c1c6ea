"""What the discriminator kernels (csrc/disc.cu) compute, restated in float64 for the stage-by-stage tests.

- Layout: the workspace (`disc_ws`) as float offsets per buffer, so a test can read every intermediate the kernels
  leave in a workspace it allocated itself.  tests/test_disc_stages_cpu.py holds the restated totals equal to the
  library's byte counts.
- Operands: vit_emulation's `operand` / `Prod` (the same cvt2 of tc_gemm.cuh).
- Stage references in float64, one per stage the workspace brackets, each from the kernel's own inputs: the power
  iteration, the exact words derived from sigma, the DiffAugment parameter words, the im2col gather, the convolution
  GEMMs (forward, dgrad, wgrad), the InstanceNorm statistics, the col2im fold with the LeakyReLU / InstanceNorm
  backward, the spectral-norm weight-gradient correction and the DiffAugment backward.  The GEMM error measure is
  |y - y_ref| / (|alpha| sum_k |a_k||b_k|), alpha the product of the GEMM's scales (2^-e / sigma, and 1 / col_scale for
  layers >= 1); the other stages say what they divide by.
- `emulate_forward` / `emulate_backward`: the whole call chained from those stages, every buffer rounded to fp32 where
  the kernel stores it.  The CPU tests take their stage inputs from it at kernel shapes and plant defects in it.
- BARS: the per-stage bars of tests/test_gpu_disc_stages.py, shared with the CPU test that plants defects under them.
"""
import math

import torch
import torch.nn.functional as F

from sinnerf_b200.discriminator import layer_schedule, output_sizes
from tests.vit_emulation import MODES, Prod, operand, stats  # noqa: F401  (re-exported for the tests)

MAX_LAYERS = 6          # SNB_DISC_MAX_LAYERS
AUG_FLOATS = 16         # per image: enabled, shift, saturation, contrast, mean, cutout box y0 y1 x0 x1
SN_EPS, IN_EPS, SLOPE = 1e-12, 1e-5, 0.2


def _al(x):
    return (x + 63) // 64 * 64


# --------------------------------------------------------------------------------------------------------------------
# layer schedule and workspace layout
# --------------------------------------------------------------------------------------------------------------------
def net(imsize, n, h, w):
    """[dict(cin, cout, K, stride, pad, in_norm, act, hin, win, hout, wout, P)] of the branch at this shape"""
    spec, sizes = layer_schedule(imsize), output_sizes(imsize, h, w)
    L, out = len(spec), []
    for i, ((cin, cout, inorm), (ho, wo)) in enumerate(zip(spec, sizes)):
        last = i == L - 1
        out.append(dict(cin=cin, cout=cout, K=16 * cin, stride=1 if last else 2, pad=0 if last else 1,
                        in_norm=bool(inorm), act=not last, hin=h, win=w, hout=ho, wout=wo, P=ho * wo, n=n))
        h, w = ho, wo
    return out


def col_scale(layers, i):
    """the power of two layer i's im2col values carry (csrc/disc.cu col_scale)"""
    if i == 0 or not layers[i - 1]["in_norm"]:
        return 1.0
    return 2.0 ** math.floor(math.log2(32768.0 / math.sqrt(layers[i - 1]["P"])))


def workspace_layout(imsize, n, h, w, save):
    """disc_ws: ({name: (float offset, shape)}, total floats).  Every buffer starts 64-float aligned.  Per layer i:
    'u{i}' 'v{i}' 't{i}' 's{i}' 'part{i}' 'rmax{i}' 'ws{i}' (cout, K) 'col{i}' (n P, K), 'y{i}' (cout, n, P) when an
    activation follows, 'mean{i}' 'rstd{i}' (cout, n) when an InstanceNorm does.  'gexp' holds int32 exponents."""
    layers = net(imsize, n, h, w)
    bufs, off = {}, 0

    def take(name, *shape):
        nonlocal off
        bufs[name] = (off, shape)
        off = _al(off + math.prod(shape))

    for k in ("sigma", "inv_sigma", "alpha", "wscale", "dot", "gexp"):
        take(k, MAX_LAYERS)
    take("aug", n, AUG_FLOATS)
    dy_max = dcol_max = 0
    for i, y in enumerate(layers):
        rows = n * y["P"]
        take(f"u{i}", y["cout"])
        take(f"v{i}", y["K"])
        take(f"t{i}", y["K"])
        take(f"s{i}", y["cout"])
        take(f"part{i}", y["cout"])
        take(f"rmax{i}", y["cout"])
        take(f"ws{i}", y["cout"], y["K"])
        take(f"col{i}", rows, y["K"])
        if y["act"]:
            take(f"y{i}", y["cout"], n, y["P"])
        if y["in_norm"]:
            take(f"mean{i}", y["cout"], n)
            take(f"rstd{i}", y["cout"], n)
        dy_max, dcol_max = max(dy_max, rows * y["cout"]), max(dcol_max, rows * y["K"])
    if save:
        take("dy0", dy_max)
        take("dy1", dy_max)
        take("dcol", dcol_max)
        take("dx", 3, n, h * w)
    return bufs, off


def workspace_views(ws, imsize, n, h, w, save=1):
    """{name: view} of a float32 workspace tensor ('gexp' as int32)"""
    bufs, total = workspace_layout(imsize, n, h, w, save)
    assert ws.dtype == torch.float32 and ws.numel() >= total
    v = {k: ws[o:o + math.prod(s)].view(*s) for k, (o, s) in bufs.items()}
    v["gexp"] = v["gexp"].view(torch.int32)
    return v


def dy_buffer(L, i):
    """the backward scratch holding layer i's scaled output gradient: 'dy0' for the last layer, then alternating"""
    return "dy0" if (L - 1 - i) % 2 == 0 else "dy1"


# --------------------------------------------------------------------------------------------------------------------
# exact words
# --------------------------------------------------------------------------------------------------------------------
def frexp_exp(m):
    """e with m = f 2^e, f in [0.5, 1) (m > 0 finite)"""
    return math.frexp(float(m))[1]


def pow2_exponent(m):
    """k with m 2^k in [2^14, 2^15); 0 for m = 0 or non-finite (csrc/disc.cu pow2_exponent)"""
    m = float(m)
    return 15 - frexp_exp(m) if m > 0 and math.isfinite(m) else 0


def ldexp32(x, e):
    """fp32 x 2^e rounded once to fp32 (ldexpf)"""
    return (x.double() * 2.0 ** e).float()


def sn_words(sigma, rmax):
    """(inv_sigma, alpha, wscale) the kernel derives from its fp32 sigma and the rows' max |W|, as fp32 scalars"""
    sigma = sigma.float().reshape(())
    inv = torch.ones((), dtype=torch.float32, device=sigma.device) / sigma
    e = pow2_exponent(rmax.float().max())
    return inv, ldexp32(inv, -e), torch.tensor(2.0 ** e, dtype=torch.float32, device=sigma.device)


def aug_words(aug, h, w):
    """the exact words of the (n, 16) DiffAugment parameters but the mean: [enabled, shift, sat, con] (fp32) and the
    clamped cutout box [y0, y1, x0, x1] (int64)"""
    rb, rs, rc, oy, ox = aug
    ch, cw = int(h * 0.5 + 0.5), int(w * 0.5 + 0.5)
    f = torch.stack([torch.ones_like(rb), rb - 0.5, rs * 2, rc + 0.5], 1)
    y0, x0 = oy - ch // 2, ox - cw // 2
    box = torch.stack([y0.clamp(0, h - 1), (y0 + ch - 1).clamp(0, h - 1), x0.clamp(0, w - 1),
                       (x0 + cw - 1).clamp(0, w - 1)], 1)
    return f, box


def cut_mask(box, h, w):
    """(n, h, w) bool: the pixels the cutout zeroes, from an (n, 4) box"""
    box = box.long()
    r = torch.arange(h, device=box.device).view(1, h, 1)
    c = torch.arange(w, device=box.device).view(1, 1, w)
    b = box.view(-1, 4, 1, 1)
    return (r >= b[:, 0]) & (r <= b[:, 1]) & (c >= b[:, 2]) & (c <= b[:, 3])


# --------------------------------------------------------------------------------------------------------------------
# stage references
# --------------------------------------------------------------------------------------------------------------------
def sn_ref(W, u_old, v_old, training, t, s, u):
    """float64 references of the power iteration, each from the kernel's previous output: {name: (ref, scale)}.
    W (cout, K) fp32; t = W^T u_old, v = t / |t|, s = W v, u = s / |s|, sigma = u . s.  Eval: v = v_old, u = u_old
    (copies, scale 0)."""
    W64 = W.double()
    out = {}
    if training:
        out["t"] = (W64.t() @ u_old.double(), W64.abs().t() @ u_old.double().abs())
        t64 = t.double()
        out["v"] = (t64 / t64.norm().clamp_min(SN_EPS), torch.ones_like(t64))
    else:
        out["v"] = (v_old.double(), torch.zeros_like(v_old.double()))
    out["s"] = (W64 @ out["v"][0], W64.abs() @ out["v"][0].abs())
    s64 = s.double()
    if training:
        out["u"] = (s64 / s64.norm().clamp_min(SN_EPS), torch.ones_like(s64))
    else:
        out["u"] = (u_old.double(), torch.zeros_like(s64))
    out["sigma"] = ((u.double() * s64).sum().reshape(1), (u.double() * s64).abs().sum().reshape(1))
    return out


def aug_mean_ref(x, shift, sat):
    """float64 per-image mean of the saturated image (rand_contrast's x_mean) from fp32 x (n, 3, h, w) and the
    kernel's shift / sat words; scale: the mean of |terms|"""
    x = x.double() + shift.double().view(-1, 1, 1, 1)
    m = x.mean(1, keepdim=True)
    v = (x - m) * sat.double().view(-1, 1, 1, 1) + m
    return v.mean((1, 2, 3)), v.abs().mean((1, 2, 3))


def unfold(src, y):
    """(n, C, hin, win) -> col (n P, 16 C): col[(b, oy, ox)][(ci, ky, kx)], zero padding"""
    n = src.shape[0]
    c = F.unfold(src, 4, padding=y["pad"], stride=y["stride"])
    return c.transpose(1, 2).reshape(n * y["P"], y["K"])


def pad_mask(y, device):
    """(n P, K) bool: the col entries that fall in the padding"""
    ones = torch.ones(1, y["cin"], y["hin"], y["win"], device=device)
    return (unfold(ones, dict(y, n=1)) == 0).repeat(y["n"], 1)


def normalized(yprev, mean, rstd):
    """(C, n, P) pre-norm y -> (n, C, P) fp32 nv = (y - mean) rstd as the kernels form it (mean None: nv = y)"""
    if mean is None:
        return yprev.transpose(0, 1)
    v = yprev - mean.unsqueeze(-1)
    v = v * rstd.unsqueeze(-1)
    return v.transpose(0, 1)


def gather_ref(layers, i, yprev, mean, rstd, row_index=None):
    """layer i >= 1's col in fp32, bit for bit: lrelu((y - mean) rstd) col_scale on load, zero padding.
    row_index: planted defect, the (channel, image) statistics row map (default c n + b)"""
    y = layers[i]
    p = layers[i - 1]
    if row_index is not None and mean is not None:
        mean, rstd = (t.reshape(-1)[row_index].view(t.shape) for t in (mean, rstd))
    v = normalized(yprev, mean, rstd)
    v = torch.where(v > 0, v, v * SLOPE)
    v = v * col_scale(layers, i)
    return unfold(v.reshape(y["n"], p["cout"], y["hin"], y["win"]).contiguous(), y)


def gather0_ref(layers, x, aug_f, aug_mean, box):
    """layer 0's col: x itself (aug_f None), else float64 of the DiffAugment maps from fp32 x and the kernel's words,
    with an error scale for the fp32 evaluation (|terms| of each multiply-add): (col, scale, cut entries)"""
    y = layers[0]
    if aug_f is None:
        return unfold(x.float(), y), None, None
    n, _, h, w = x.shape
    shift, sat, con = (aug_f[:, j].double().view(n, 1, 1, 1) for j in (1, 2, 3))
    mu = aug_mean.double().view(n, 1, 1, 1)
    xs = x.double() + shift
    m = xs.mean(1, keepdim=True)
    s = (xs - m) * sat + m
    v = (s - mu) * con + mu
    mag = ((xs.abs() + m.abs()) * sat.abs() + m.abs() + mu.abs()) * con.abs() + mu.abs() + xs.abs()
    cut = cut_mask(box, h, w).unsqueeze(1).expand(n, 3, h, w)
    v = torch.where(cut, torch.zeros_like(v), v)
    return unfold(v, y), unfold(mag, y), unfold(cut.double(), y) > 0


def gemm_fwd_ref(ws, col, alpha, cs, mode, **defect):
    """y (cout, n P) = alpha / cs sum_k ws col: (emu, exact, scale)"""
    p = Prod(ws, col, mode, **defect)
    a = float(alpha) / cs
    return p.emu * a, p.exact * a, p.abs * abs(a)


def in_stats_ref(y):
    """float64 (mean, rstd) per (channel, image) row of the kernel's pre-norm y (C, n, P), and their error scales:
    mean |y| for the mean, rstd for rstd (a relative error)"""
    y64 = y.double()
    m = y64.mean(-1)
    var = (y64 - m.unsqueeze(-1)).square().mean(-1)
    r = 1.0 / torch.sqrt(var + IN_EPS)
    return m, r, y64.abs().mean(-1), r


def scaled_upstream(d_out):
    """(dy, k): the upstream gradient times 2^k, its largest element in [2^14, 2^15), bit for bit"""
    k = pow2_exponent(d_out.abs().nan_to_num(0.0).max())
    return ldexp32(d_out.float(), k), k


def dgrad_ref(dy, ws, alpha, mode, alpha_times=1):
    """dcol (n P, K) = alpha sum_co dy[co][j] ws[co][k]: (emu, exact, scale).  alpha_times: planted defect"""
    p = Prod(dy.t(), ws.t(), mode)
    a = float(alpha) ** alpha_times
    return p.emu * a, p.exact * a, p.abs * abs(a)


def wgrad_ref(dy, col, cs, mode):
    """dW_raw (cout, K) = (1 / cs) sum_j dy[co][j] col[j][k]: (emu, exact, scale)"""
    p = Prod(dy, col.t(), mode)
    return p.emu / cs, p.exact / cs, p.abs / cs


def fold_ref(layers, i, dcol, yprev, mean, rstd, mask_on_y=False, drop_gn=False, row_index=None):
    """float64 gradient at layer i's input (cin, n, hin win), before its rescale, from the kernel's dcol and layer
    i - 1's saved y / mean / rstd: the col2im sum, then the LeakyReLU backward with the mask nv > 0 of fp32 nv, then
    the InstanceNorm backward rstd (g - mean g - nv mean(g nv)).  i = 0: the col2im sum alone (scaled input gradient).
    -> (ref, scale, mask).  Planted defects: mask_on_y (the mask taken on pre-norm y), drop_gn (no nv mean(g nv)
    term), row_index (the statistics row map)."""
    y = layers[i]
    n, H, W = y["n"], y["hin"], y["win"]

    def fold(c):
        c = c.double().view(n, y["P"], y["K"]).transpose(1, 2)
        return F.fold(c, (H, W), 4, padding=y["pad"], stride=y["stride"]).reshape(n, y["cin"], H * W)
    g, ga = fold(dcol), fold(dcol.abs())
    if i == 0:
        return g.transpose(0, 1), ga.transpose(0, 1), None
    if row_index is not None and mean is not None:
        mean, rstd = (t.reshape(-1)[row_index].view(t.shape) for t in (mean, rstd))
    nv = normalized(yprev, mean, rstd)                    # (n, C, P) fp32
    mask = (yprev.transpose(0, 1) if mask_on_y else nv) > 0
    g, ga = torch.where(mask, g, g * SLOPE), torch.where(mask, ga, ga * SLOPE)
    if mean is None:
        return g.transpose(0, 1), ga.transpose(0, 1), mask.transpose(0, 1)
    nv = nv.double()
    rs = rstd.double().transpose(0, 1).unsqueeze(-1)
    gn = 0.0 if drop_gn else (g * nv).mean(-1, keepdim=True)
    ref = rs * (g - g.mean(-1, keepdim=True) - nv * gn)
    scale = rs * (ga + ga.mean(-1, keepdim=True) + nv.abs() * (ga * nv.abs()).mean(-1, keepdim=True))
    return ref.transpose(0, 1), scale.transpose(0, 1), mask.transpose(0, 1)


def part_ref(dw_raw, dw_abs, W):
    """part[r] = <dW_raw[r], W[r]>: (ref, scale)"""
    return (dw_raw * W.double()).sum(1), (dw_abs * W.double().abs()).sum(1)


def sn_fix_ref(dw_raw, dw_abs, part, inv_sigma, u, v, gexp, sigma_power=2):
    """dW_orig = 2^gexp (dW_raw / sigma - (sum part / sigma^2) u v^T) from the kernel's part, inv_sigma, u, v:
    (ref, scale).  sigma_power: planted defect (1: the correction divides by sigma once)"""
    is64 = float(inv_sigma)
    c = part.double().sum() * is64 ** sigma_power
    uv = torch.outer(u.double(), v.double())
    f = 2.0 ** int(gexp)
    return f * (dw_raw * is64 - c * uv), f * (dw_abs * abs(is64) + (c * uv).abs())


def aug_bwd_ref(dx, aug_f, box, gexp, h, w, cut_in_mean=False):
    """input gradient (n, 3, h, w) from the kernel's dx (3, n, h w) (the scaled col2im sum at layer 0): the contrast
    backward con g + (1 - con) S, S the mean of g over the pixels the cutout keeps, then the saturation backward
    sat g + (1 - sat) mean_c g, times 2^gexp.  -> (ref, scale).  cut_in_mean: planted defect (S over every pixel)."""
    n = dx.shape[1]
    g = dx.double().transpose(0, 1).reshape(n, 3, h, w)
    f = 2.0 ** int(gexp)
    if aug_f is None:
        return f * g, f * g.abs()
    sat, con = (aug_f[:, j].double().view(n, 1, 1, 1) for j in (2, 3))
    keep = (~cut_mask(box, h, w)).unsqueeze(1).double()
    gk = g * keep
    S = (g if cut_in_mean else gk).sum((1, 2, 3), keepdim=True) / (3 * h * w)
    Sa = (g.abs() if cut_in_mean else gk.abs()).sum((1, 2, 3), keepdim=True) / (3 * h * w)
    g1 = con * gk + (1 - con) * S
    a1 = con.abs() * gk.abs() + (1 - con).abs() * Sa
    g2 = sat * g1 + (1 - sat) * g1.mean(1, keepdim=True)
    a2 = sat.abs() * a1 + (1 - sat).abs() * a1.mean(1, keepdim=True)
    return f * g2, f * a2


def err(y, ref, scale):
    """per-element |y - ref| / scale (scale 0 only where both are 0)"""
    return (y.double() - ref).abs() / scale.clamp_min(1e-300)


# --------------------------------------------------------------------------------------------------------------------
# the whole call, chained from the stages (fp32 where the kernel stores)
# --------------------------------------------------------------------------------------------------------------------
def emulate_forward(imsize, Ws, us, vs, x, training, aug, mode):
    """the buffers of snb_disc_forward as workspace_views names them (fp32), plus 'out' and 'layers'.  Ws: fp32
    weight_orig tensors, us / vs the stored u / v, x (n, 3, h, w) fp32, aug None or the five draws."""
    n, _, h, w = x.shape
    layers = net(imsize, n, h, w)
    b = {"layers": layers}
    sig, inv, alp, wsc = [], [], [], []
    for i, (Wt, u0, v0) in enumerate(zip(Ws, us, vs)):
        W = Wt.float().reshape(layers[i]["cout"], -1)
        if training:
            t = (W.double().t() @ u0.double()).float()
            v = (t.double() / t.double().norm().clamp_min(SN_EPS)).float()
        else:
            t, v = torch.full_like(v0, float("nan")), v0.float().clone()
        s = (W.double() @ v.double()).float()
        u = (s.double() / s.double().norm().clamp_min(SN_EPS)).float() if training else u0.float().clone()
        sigma = (u.double() * s.double()).sum().float()
        rmax = W.abs().amax(1)
        iv, a, ws_ = sn_words(sigma, rmax)
        b.update({f"t{i}": t, f"v{i}": v, f"s{i}": s, f"u{i}": u, f"rmax{i}": rmax, f"ws{i}": W * ws_})
        sig.append(sigma)
        inv.append(iv)
        alp.append(a)
        wsc.append(ws_)
    b["sigma"], b["inv_sigma"], b["alpha"], b["wscale"] = (torch.stack(t) for t in (sig, inv, alp, wsc))
    aug_f = box = mean_aug = None
    if aug is not None:
        aug_f, box = aug_words(aug, h, w)
        mean_aug = aug_mean_ref(x, aug_f[:, 1], aug_f[:, 2])[0].float()
    b["aug_f"], b["box"], b["aug_mean"] = aug_f, box, mean_aug
    for i, y in enumerate(layers):
        if i == 0:
            col = gather0_ref(layers, x, aug_f, mean_aug, box)[0].float()
        else:
            col = gather_ref(layers, i, b[f"y{i - 1}"], b.get(f"mean{i - 1}"), b.get(f"rstd{i - 1}"))
        b[f"col{i}"] = col
        out = gemm_fwd_ref(b[f"ws{i}"], col, b["alpha"][i], col_scale(layers, i), mode)[0].float()
        if y["act"]:
            b[f"y{i}"] = out.view(y["cout"], n, y["P"])
        else:
            b["out"] = out.view(n, 1, y["hout"], y["wout"])
        if y["in_norm"]:
            m, r, _, _ = in_stats_ref(b[f"y{i}"])
            b[f"mean{i}"], b[f"rstd{i}"] = m.float(), r.float()
    return b


def emulate_backward(b, Ws, d_out, mode):
    """adds to the forward's buffers: 'dy{i}' (layer i's scaled output gradient), 'k{i}' (its exponent), 'dcol{i}',
    'fold{i}' (layer i's input gradient before the rescale), 'dwraw{i}', 'part{i}', 'dW{i}', 'gexp' (list), 'dx',
    'd_input'"""
    layers = b["layers"]
    L, n = len(layers), layers[0]["n"]
    h, w = layers[0]["hin"], layers[0]["win"]
    dy, k = scaled_upstream(d_out.reshape(1, -1))
    gexp = [0] * L
    gexp[L - 1] = -k
    for i in range(L - 1, -1, -1):
        y = layers[i]
        b[f"dy{i}"] = dy
        cs = col_scale(layers, i)
        raw = wgrad_ref(dy, b[f"col{i}"], cs, mode)[0].float()
        b[f"dwraw{i}"] = raw
        b[f"part{i}"] = (raw.double() * Ws[i].reshape(y["cout"], -1).double()).sum(1).float()
        dcol = dgrad_ref(dy, b[f"ws{i}"], b["alpha"][i], mode)[0].float()
        b[f"dcol{i}"] = dcol
        g = fold_ref(layers, i, dcol, b.get(f"y{i - 1}"), b.get(f"mean{i - 1}"), b.get(f"rstd{i - 1}"))[0].float()
        b[f"fold{i}"] = g
        if i > 0:
            k = pow2_exponent(g.abs().max())
            dy = ldexp32(g, k).reshape(layers[i - 1]["cout"], -1)
            gexp[i - 1] = gexp[i] - k
    b["gexp"] = gexp
    b["dx"] = b["fold0"]
    b["d_input"] = aug_bwd_ref(b["dx"], b["aug_f"], b["box"], gexp[0], h, w)[0].float()
    for i, y in enumerate(layers):
        raw = b[f"dwraw{i}"].double()
        b[f"dW{i}"] = sn_fix_ref(raw, raw.abs(), b[f"part{i}"], b["inv_sigma"][i], b[f"u{i}"], b[f"v{i}"],
                                 gexp[i])[0].float().view_as(Ws[i])
    return b


# --------------------------------------------------------------------------------------------------------------------
# bars
# --------------------------------------------------------------------------------------------------------------------
# (worst, rms) of the per-element error against the float64 reference, per stage and mode, about 4x the largest value
# measured on an H100 SXM (80 GB, 700 W) over the branches, shapes, batch sizes and augmentation edges of
# tests/test_gpu_disc_stages.py.  DESIGN.md section 2 lists the measurements.  The stages around the GEMMs do not
# depend on the mode.  Units: |y - ref| / scale as each reference states it; 'gather0' in units of 2^-24 of the
# magnitude of its terms; 'v' and 'u' absolute (unit vectors).
_COMMON = {
    "t": (1.0e-6, 1.1e-7), "v": (1.0e-7, 3.1e-8), "s": (4.2e-7, 4.2e-7), "u": (1.0e-7, 2.9e-8),
    "sigma": (4.0e-7, 4.0e-7), "aug_mean": (3.5e-7, 3.1e-7), "gather0": (6.1, 0.87), "in_mean": (8.0e-7, 2.0e-7),
    "in_rstd": (7.2e-7, 2.2e-7), "fold": (8.2e-7, 1.1e-7), "aug_bwd": (5.9e-7, 1.1e-7), "part": (8.3e-7, 3.1e-7),
}
BARS = {
    "split": dict(_COMMON, fwd=(1.2e-5, 2.6e-6), dgrad=(4.3e-6, 5.6e-7), wgrad=(1.25e-5, 2.4e-6)),
    "f16": dict(_COMMON, fwd=(4.0e-6, 1.0e-6), dgrad=(1.7e-6, 2.0e-7), wgrad=(3.9e-6, 8.0e-7)),
    "bf16": dict(_COMMON, fwd=(3.5e-6, 8.2e-7), dgrad=(1.4e-6, 1.6e-7), wgrad=(4.0e-6, 7.7e-7)),
}
