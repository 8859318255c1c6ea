"""References for the ray kernels (sinnerf_b200/csrc/ray_kernels.cu) and a CPU stand-in for them.

Three things, none of which imports the library or reads anything outside the tree:

* float64 truth of each stage, written from the mathematics (`composite64`, `sample_pdf64`, `losses64`,
  `g_raw_bound64`); the compositing backward is float64 autograd through `composite64`.
* fp32 emulation, operation for operation, of the stages whose result holds a discrete decision: the cdf
  (`build_cdf32`: per-lane strided sum, xor butterfly, 32-wide Hillis-Steele scan with a carried total), the
  inverse cdf (`invert_cdf32`: the binary search itself, both clamps, `denom < eps -> 1`, each operation rounded on
  its own) and the sorted union (`merge32`).  Those kernels use only explicitly rounded adds, subtracts, multiplies
  and divides, so numpy float32 reproduces them bit for bit.
* `StandIn`: the entry points of include/sinnerf_b200.h that the stage tests drive, on CPU tensors, with the two
  compositing mappings (warp per ray; four samples per thread in lane groups of 8 / 16 / 32) written out in float32 in
  the kernels' order of operations.  numpy's exp is not CUDA's expf, so the compositing half is not bitwise; it
  exists so that the checkers of tests/test_gpu_ray_stages.py can be exercised, and shown to catch planted defects,
  without a GPU.  `StandIn(defect=...)` plants one defect (names in DEFECTS).
"""
import numpy as np
import torch

f32 = np.float32
EPS_T = float(f32(1e-10))        # the 1e-10f the kernels add to 1 - alpha
SATURATED = float(f32(3.0e38))   # g_amax value for an infinite gradient

DEFECTS = (
    "search_lt",            # invert_cdf: cdf[mid] <= u  ->  <
    "above_clamp",          # invert_cdf: above clamped to M - 1
    "denom_le",             # invert_cdf: denom < eps  ->  <=
    "merge_lt",             # merge: zs[mid] <= v  ->  <   (ties no longer coarse first)
    "rank_no_tiebreak",     # rank sort of the new depths without  k < j
    "last_delta_no_dnorm",  # last sample's 1e10 not multiplied by |d|
    "quad_scan_gt",         # four-per-thread product scan: sl >= off  ->  sl > off
    "quad_tail_kept",       # four-per-thread backward: tail not zeroed for the group's last lane
    "warp_no_carry_step2",  # warp-per-ray: carried product not applied on the second 32-sample step
    "warp_suffix_late",     # warp-per-ray backward: suffix scan starts one 32-sample group late
    "warp_mse_no_2",        # warp-per-ray backward: 2 * missing from the MSE derivative
    "amax_no_gw",           # g_amax without the g * w terms
    "ticket_not_reset",     # the loss workspace's ticket is left at gridDim.x
    "second_trip_cdf",      # a warp's second ray reuses its first ray's cdf
)


# ------------------------------------------------------------------------------------------------ float64 truth
def composite64(raw, z, dnorm, noise, noise_std, white_back):
    """models/rendering.py:215-248 in float64 on whatever device the inputs live on.  raw (N,S,4) or sigma (N,S);
    dnorm (N,); noise (N,S) or None.  Differentiable in raw."""
    raw, z, dnorm = raw.double(), z.double(), dnorm.double()
    sigma = raw[..., 3] if raw.dim() == 3 else raw
    s = sigma if noise is None else sigma + noise.double() * float(f32(noise_std))
    delta = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], 1) * dnorm[:, None]
    e = torch.exp(-delta * torch.relu(s))
    alpha = 1 - e
    t = 1 - alpha + EPS_T
    T = torch.cat([torch.ones_like(t[:, :1]), torch.cumprod(t, 1)[:, :-1]], 1)
    w = alpha * T
    out = {"weights": w, "alpha": alpha, "T": T, "t": t, "delta": delta, "e": e, "s": s}
    if raw.dim() == 3:
        rgb = (w[..., None] * raw[..., :3]).sum(1)
        if white_back:
            rgb = rgb + 1 - w.sum(1, keepdim=True)
        out["rgb"] = rgb
        # bounds with T_i in place of w_i = alpha_i T_i: alpha = 1 - exp(-x) is rounded to an ulp of 1, not of alpha
        out["rgb_bound"] = (T[..., None] * raw[..., :3].abs()).sum(1) + (1 + T.sum(1, keepdim=True) if white_back else 0)
    out["depth"] = (w * z).sum(1)
    out["depth_bound"] = (T * z.abs()).sum(1)
    return out


def losses64(rgb, depth, trgb, tdepth, wr, wd):
    """loss[0] = sum_ray wr sum_c (rgb - t)^2, loss[1] = sum_ray wd smooth_l1(depth - t) (beta 1); wr / wd scalars or
    (N,) tensors; a None target gives 0."""
    l0 = rgb.new_zeros((), dtype=torch.float64)
    l1 = rgb.new_zeros((), dtype=torch.float64)
    if trgb is not None:
        l0 = (torch.as_tensor(wr, device=rgb.device).double() * ((rgb.double() - trgb.double()) ** 2).sum(1)).sum()
    if tdepth is not None:
        x = depth.double() - tdepth.double()
        sl1 = torch.where(x.abs() < 1, 0.5 * x * x, x.abs() - 0.5)
        l1 = (torch.as_tensor(wd, device=rgb.device).double() * sl1).sum()
    return l0, l1


def g_raw_bound64(c64, raw, z, white_back, g_rgb, g_depth, g_w):
    """Per element of g_raw, the float64 sum of absolute values of the terms of its closed form (SURVEY.md 8a-7), with
    every w_k = alpha_k T_k replaced by T_k: alpha = 1 - exp(-x) carries an ABSOLUTE rounding error of an ulp of 1, so
    what bounds the error of w_k is T_k, not w_k.
       g_sigma_i:  |delta_i| e_i ( G_i T_i + sum_{k>i} G_k T_k / t_i ),  G_i = |g_rgb| . |c_i| + |g_depth z_i| + |g_w_i| + [wb] sum |g_rgb|
       g_c_i:      |g_rgb_c| T_i
    c64: composite64's dict; g_rgb (N,3) / g_depth (N,) / g_w (N,S) float64 (zeros where absent)."""
    G = g_depth.abs()[:, None] * z.double().abs() + g_w.abs()
    if raw.dim() == 3:
        G = G + (g_rgb.abs()[:, None, :] * raw[..., :3].double().abs()).sum(-1)
        if white_back:
            G = G + g_rgb.abs().sum(1, keepdim=True)
    v = G * c64["T"].abs()
    suffix = torch.flip(torch.cumsum(torch.flip(v, [1]), 1), [1]) - v
    gs = c64["delta"].abs() * c64["e"] * (G * c64["T"] + suffix / c64["t"])
    if raw.dim() == 2:
        return gs
    return torch.cat([g_rgb.abs()[:, None, :] * c64["T"].abs()[..., None], gs[..., None]], -1)


def g_raw_closed_form64(c64, raw, z, white_back, g_rgb, g_depth, g_w):
    """SURVEY.md 8a-7 written out in float64 (what float64 autograd through composite64 must equal)."""
    gw = g_depth[:, None] * z.double() + g_w
    if raw.dim() == 3:
        gw = gw + (g_rgb[:, None, :] * raw[..., :3].double()).sum(-1)
        if white_back:
            gw = gw - g_rgb.sum(1, keepdim=True)
    v = gw * c64["weights"]
    suffix = torch.flip(torch.cumsum(torch.flip(v, [1]), 1), [1]) - v
    galpha = gw * c64["T"] - suffix / c64["t"]
    gs = torch.where(c64["s"] > 0, galpha * c64["delta"] * c64["e"], torch.zeros_like(galpha))
    if raw.dim() == 2:
        return gs
    return torch.cat([g_rgb[:, None, :] * c64["weights"][..., None], gs[..., None]], -1)


def sample_pdf64(bins, weights, u, eps=1e-5):
    """models/rendering.py:15-61 in float64 (numpy).  u (Ni,) shared or (N,Ni).  Returns samples, cdf, and per sample
    the denominator used and the width of its bin."""
    bins, w = np.asarray(bins, np.float64), np.asarray(weights, np.float64) + float(f32(eps))
    n, m = w.shape
    u = np.broadcast_to(np.asarray(u, np.float64), (n, np.shape(u)[-1]))
    cdf = np.concatenate([np.zeros((n, 1)), np.cumsum(w / w.sum(1, keepdims=True), 1)], 1)
    idx = (cdf[:, None, :] <= u[:, :, None]).sum(-1)
    lo, hi = np.maximum(idx - 1, 0), np.minimum(idx, m)
    c0, c1 = np.take_along_axis(cdf, lo, 1), np.take_along_axis(cdf, hi, 1)
    b0, b1 = np.take_along_axis(bins, lo, 1), np.take_along_axis(bins, hi, 1)
    den = c1 - c0
    den = np.where(den < float(f32(eps)), 1.0, den)
    return b0 + (u - c0) / den * (b1 - b0), cdf, den, b1 - b0


# ------------------------------------------------------------------------------------------------ fp32, bit for bit
def build_cdf32(w, eps):
    """warp_build_cdf on rows w (N,M) float32 -> cdf (N,M+1) float32, in the kernel's order of additions."""
    w = np.ascontiguousarray(w, f32)
    n, m = w.shape
    we = w + f32(eps)
    pad = (-m) % 32
    wl = np.concatenate([we, np.zeros((n, pad), f32)], 1).reshape(n, -1, 32)
    valid = (np.arange(m + pad) < m).reshape(-1, 32)
    lane = np.zeros((n, 32), f32)
    for k in range(wl.shape[1]):                 # lane l: w[l] + w[l + 32] + ... serially (absent elements are skipped)
        lane = np.where(valid[k][None, :], lane + wl[:, k], lane)
    idx = np.arange(32)
    for off in (16, 8, 4, 2, 1):                 # xor butterfly: every lane ends with the same total
        lane = lane + lane[:, idx ^ off]
    total = lane[:, :1]
    cdf = np.zeros((n, m + pad + 1), f32)
    carry = np.zeros(n, f32)
    with np.errstate(all="ignore"):
        for k in range(wl.shape[1]):
            v = np.where(valid[k][None, :], wl[:, k] / total, f32(0))
            for off in (1, 2, 4, 8, 16):         # Hillis-Steele inclusive scan of 32 lanes
                nv = v.copy()
                nv[:, off:] = v[:, off:] + v[:, :-off]
                v = nv
            cdf[:, 1 + 32 * k:33 + 32 * k] = carry[:, None] + v
            carry = carry + v[:, 31]
    return cdf[:, :m + 1]


def invert_cdf32(cdf, bins, u, eps, defect=None):
    """invert_cdf for every (row, u): cdf (N,M+1), bins (N,M+1), u (N,Ni), all float32.  Returns samples, below, above."""
    n, m1 = cdf.shape
    m = m1 - 1
    lo = np.zeros(u.shape, np.int64)
    hi = np.full(u.shape, m + 1, np.int64)
    while True:
        act = lo < hi
        if not act.any():
            break
        mid = (lo + hi) >> 1
        c = np.take_along_axis(cdf, np.minimum(mid, m), 1)
        go = (c < u) if defect == "search_lt" else (c <= u)
        lo = np.where(act & go, mid + 1, lo)
        hi = np.where(act & ~go, mid, hi)
    below = np.maximum(lo - 1, 0)
    above = np.minimum(lo, m - 1 if defect == "above_clamp" and m >= 1 else m)
    c0, c1 = np.take_along_axis(cdf, below, 1), np.take_along_axis(cdf, above, 1)
    b0, b1 = np.take_along_axis(bins, below, 1), np.take_along_axis(bins, above, 1)
    with np.errstate(all="ignore"):
        den = c1 - c0
        den = np.where((den <= f32(eps)) if defect == "denom_le" else (den < f32(eps)), f32(1), den)
        out = b0 + ((u - c0) / den) * (b1 - b0)
    return out.astype(f32), below, above


def sample_pdf32(bins, weights, u, eps=1e-5, defect=None):
    """snb_sample_pdf bit for bit.  u (Ni,) shared or (N,Ni)."""
    bins, weights = np.asarray(bins, f32), np.asarray(weights, f32)
    n = weights.shape[0]
    u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, f32), (n, np.shape(u)[-1])))
    cdf = build_cdf32(weights, eps)
    if defect == "second_trip_cdf" and n > 1:
        cdf = cdf.copy()
        cdf[1::2] = cdf[0::2][:cdf[1::2].shape[0]]
    return invert_cdf32(cdf, bins, u, eps, defect)[0]


def knot_samples(weights, u, eps=1e-5, ulps=2):
    """(N,Ni) mask of the samples whose u lies within `ulps` float32 ulps of a knot of the emulated cdf: the only places
    where an implementation with a differently rounded cdf may land in the neighbouring bin."""
    cdf = build_cdf32(np.asarray(weights, f32), eps).astype(np.float64)
    n = cdf.shape[0]
    u = np.broadcast_to(np.asarray(u, np.float64), (n, np.shape(u)[-1]))
    d = np.abs(cdf[:, None, :] - u[:, :, None]).min(-1)
    return d <= ulps * np.spacing(np.maximum(u, 2.0 ** -126).astype(f32)).astype(np.float64)


def z_mid32(z):
    z = np.asarray(z, f32)
    with np.errstate(all="ignore"):
        return f32(0.5) * (z[:, :-1] + z[:, 1:])


def sort_like_torch(rows):
    """torch.sort's order on float32 rows: ascending, stable, NaN last."""
    rows = np.asarray(rows, f32)
    return np.take_along_axis(rows, np.argsort(rows, 1, kind="stable"), 1)


def merge32(z, z_new, defect=None, sentinel=f32(-7.0)):
    """importance_merge_kernel's sorted union, path by path, on rows z (N,S), z_new (N,Ni): slots the algorithm never
    writes keep `sentinel`."""
    z, z_new = np.asarray(z, f32), np.asarray(z_new, f32)
    n, S = z.shape
    Ni = z_new.shape[1]
    out = np.full((n, S + Ni), sentinel, f32)
    for r in range(n):
        zs, zn = z[r], z_new[r].copy()
        allv = np.concatenate([zs, zn])
        if np.isnan(allv).any() or not (zs[:-1] <= zs[1:]).all():      # general path: all-pairs rank, NaN last
            out[r] = sort_like_torch(allv[None])[0]
            continue
        if not (zn[:-1] <= zn[1:]).all():                              # rank sort of the new depths
            k = np.arange(Ni)
            less = zn[None, :] < zn[:, None]
            tie = (zn[None, :] == zn[:, None]) & (k[None, :] < k[:, None])
            rk = (less | tie).sum(1) if defect != "rank_no_tiebreak" else less.sum(1)
            srt = zn.copy()
            srt[rk] = zn
            zn = srt
        out[r, np.arange(S) + np.searchsorted(zn, zs, "left")] = zs     # coarse: + #{new < z}
        side = "left" if defect == "merge_lt" else "right"
        out[r, np.arange(Ni) + np.searchsorted(zs, zn, side)] = zn      # new: + #{coarse <= z}
    return out


# ------------------------------------------------------------------------------------------------ the stand-in
def _aligned(*ts):
    return all(t is None or t.data_ptr() % 16 == 0 for t in ts)


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def quad_mapping(S, *per_sample):
    """The launcher's choice: four samples per thread when rows are whole 16-byte quads at aligned addresses."""
    return 4 <= S <= 128 and S % 4 == 0 and _aligned(*per_sample)


def _lane_group(S):
    return 8 if S <= 32 else (16 if S <= 64 else 32)


class StandIn:
    """The ray entry points on CPU float32 tensors.  `sm_count` fixes the launch caps as on a 132-SM part."""
    sm_count = 132
    device = "cpu"

    def __init__(self, defect=None):
        assert defect is None or defect in DEFECTS, defect
        self.defect = defect
        self.ticket = 0

    # ---- compositing, forward part shared by both directions
    def _forward_core(self, raw, z, rays, noise, noise_std, quad):
        d = self.defect
        sigma = raw[..., 3] if raw.ndim == 3 else raw
        n, S = z.shape
        dnorm = np.sqrt((rays[:, 3:6] * rays[:, 3:6]).sum(1, dtype=f32)).astype(f32)
        with np.errstate(all="ignore"):
            delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((n, 1), 1e10, f32)], 1)
            scale = np.repeat(dnorm[:, None], S, 1)
            if d == "last_delta_no_dnorm":
                scale[:, -1] = 1
            delta = delta * scale
            sg = sigma if noise is None else sigma + noise * f32(noise_std)
            e = np.exp(-(delta * np.fmax(sg, f32(0)))).astype(f32)    # fmaxf: a NaN density counts as 0
            alpha = f32(1) - e
            t = (f32(1) - alpha) + f32(1e-10)
            T = self._scan_quad(t, _lane_group(S)) if quad else self._scan_warp(t)
        return dict(delta=delta, sg=sg, e=e, alpha=alpha, t=t, T=T, w=alpha * T)

    def _scan_warp(self, t):
        n, S = t.shape
        T = np.empty_like(t)
        carry = np.ones(n, f32)
        for step, base in enumerate(range(0, S, 32)):
            m = min(32, S - base)
            scan = np.ones((n, 32), f32)
            scan[:, :m] = t[:, base:base + m]
            for off in (1, 2, 4, 8, 16):
                nv = scan.copy()
                nv[:, off:] = scan[:, off:] * scan[:, :-off]
                scan = nv
            excl = np.concatenate([np.ones((n, 1), f32), scan[:, :-1]], 1)
            c = np.ones(n, f32) if (self.defect == "warp_no_carry_step2" and step == 1) else carry
            T[:, base:base + m] = (c[:, None] * excl)[:, :m]
            carry = carry * scan[:, 31]
        return T

    def _scan_quad(self, t, L):
        n, S = t.shape
        nq = S // 4
        tq = np.ones((n, L, 4), f32)
        tq[:, :nq] = t.reshape(n, nq, 4)
        p0 = tq[..., 0]
        p1 = p0 * tq[..., 1]
        p2 = p1 * tq[..., 2]
        scan = p2 * tq[..., 3]
        off = 1
        while off < L:
            first = off + 1 if self.defect == "quad_scan_gt" else off
            nv = scan.copy()
            nv[:, first:] = scan[:, first:] * scan[:, first - off:L - off]
            scan = nv
            off <<= 1
        excl = np.concatenate([np.ones((n, 1), f32), scan[:, :-1]], 1)
        return np.stack([excl, excl * p0, excl * p1, excl * p2], -1)[:, :nq].reshape(n, S)

    def composite_forward(self, raw, raw_channels, z, rays, noise, noise_std, white_back, want_maps=True, w_out=None):
        S = z.shape[1]
        noise = noise if noise_std != 0 else None
        w_out = torch.empty_like(z) if w_out is None else w_out
        quad = quad_mapping(S, raw, z, noise, w_out)
        raw_, z_ = _np(raw), _np(z)
        f = self._forward_core(raw_, z_, _np(rays), _np(noise), noise_std, quad)
        w = f["w"]
        w_out.copy_(torch.from_numpy(w))
        if not want_maps:
            return None, None, w_out
        with np.errstate(all="ignore"):
            c = raw_[..., :3] if raw_channels == 4 else np.zeros(z_.shape + (3,), f32)
            rgb = (w[..., None] * c).sum(1, dtype=f32)
            if white_back:
                rgb = (rgb + f32(1)) - w.sum(1, dtype=f32)[:, None]
            depth = (w * z_).sum(1, dtype=f32)
        return torch.from_numpy(rgb), torch.from_numpy(depth), w_out

    def composite_forward_loss(self, raw, z, rays, noise, noise_std, white_back, loss, ws):
        """loss: dict(trgb, tdepth, wr, wd, wr0, wd0); ws: the (LOSS_WS_FLOATS,) workspace, word 0 the ticket."""
        rgb, depth, w = self.composite_forward(raw, 4, z, rays, noise, noise_std, white_back)
        assert int(ws.view(torch.int32)[0]) == 0, "loss workspace ticket was not zero on entry"
        with np.errstate(all="ignore"):
            out = np.zeros(2, f32)
            if loss.get("trgb") is not None:
                wr = _np(loss["wr"]) if loss.get("wr") is not None else f32(loss["wr0"])
                out[0] = (wr * ((_np(rgb) - _np(loss["trgb"])) ** 2).sum(1, dtype=f32)).sum(dtype=f32)
            if loss.get("tdepth") is not None:
                wd = _np(loss["wd"]) if loss.get("wd") is not None else f32(loss["wd0"])
                x = _np(depth) - _np(loss["tdepth"])
                out[1] = (wd * np.where(np.abs(x) < 1, f32(0.5) * x * x, np.abs(x) - f32(0.5))).sum(dtype=f32)
        if self.defect == "ticket_not_reset":
            ws.view(torch.int32)[0] = 1
        return rgb, depth, w, torch.from_numpy(out)

    def composite_backward(self, raw, raw_channels, z, rays, noise, noise_std, white_back, g_rgb, g_depth, g_w,
                           loss=None, out_rgb=None, out_depth=None, g_loss=None, amax=None, g_raw_out=None):
        """-> g_raw like raw.  amax: a (1,) float32 tensor raised in place to the bit pattern of max |g_raw|."""
        d = self.defect
        n, S = z.shape
        noise = noise if noise_std != 0 else None
        g_raw = torch.empty_like(raw) if g_raw_out is None else g_raw_out
        quad = quad_mapping(S, raw, z, noise, g_w, g_raw)
        raw_, z_ = _np(raw), _np(z)
        f = self._forward_core(raw_, z_, _np(rays), _np(noise), noise_std, quad)
        with np.errstate(all="ignore"):
            g = np.zeros((n, 3), f32) if g_rgb is None else _np(g_rgb).copy()
            gd = np.zeros(n, f32) if g_depth is None else _np(g_depth).copy()
            if loss is not None:
                gl = np.ones(2, f32) if g_loss is None else _np(g_loss)
                if loss.get("trgb") is not None:
                    wr = _np(loss["wr"]) if loss.get("wr") is not None else f32(loss["wr0"])
                    k = (f32(1) if (d == "warp_mse_no_2" and not quad) else f32(2)) * wr * gl[0]
                    g = g + (np.asarray(k, f32).reshape(-1, 1) * (_np(out_rgb) - _np(loss["trgb"]))).astype(f32)
                if loss.get("tdepth") is not None:
                    wd = _np(loss["wd"]) if loss.get("wd") is not None else f32(loss["wd0"])
                    x = _np(out_depth) - _np(loss["tdepth"])
                    gd = gd + (wd * gl[1] * np.where(np.abs(x) < 1, x, np.sign(x))).astype(f32)
            c = raw_[..., :3] if raw_channels == 4 else np.zeros(z_.shape + (3,), f32)
            gwb = g.sum(1, dtype=f32) if white_back else np.zeros(n, f32)
            gw = (c * g[:, None, :]).sum(-1, dtype=f32) + gd[:, None] * z_ - gwb[:, None]
            if g_w is not None:
                gw = gw + _np(g_w)
            v = gw * f["alpha"] * f["T"]
            suf = self._suffix_quad(v, _lane_group(S)) if quad else self._suffix_warp(v)
            galpha = gw * f["T"] - suf / f["t"]
            gs = np.where(f["sg"] > 0, galpha * f["delta"] * f["e"], f32(0)).astype(f32)
            gc = (g[:, None, :] * f["w"][..., None]).astype(f32)
        if raw_channels == 4:
            g_raw.copy_(torch.from_numpy(np.concatenate([gc, gs[..., None]], -1)))
        else:
            g_raw.copy_(torch.from_numpy(gs))
        if amax is not None:
            terms = np.abs(gs).ravel() if d == "amax_no_gw" else np.concatenate([np.abs(gs).ravel(), np.abs(gc).ravel()])
            terms = terms[~np.isnan(terms)]                 # fmaxf drops NaN operands
            m = f32(terms.max()) if terms.size else f32(0)
            if m > 0:
                bits = np.minimum(m, f32(3.0e38)).view(np.uint32)
                a = amax.view(torch.int32)
                a[0] = max(int(a[0]), int(bits))
        return g_raw

    def _suffix_warp(self, v):
        n, S = v.shape
        out = np.zeros_like(v)
        tail = np.zeros(n, f32)
        start = ((S - 1) // 32) * 32
        if self.defect == "warp_suffix_late":
            start -= 32
        for base in range(start, -1, -32):
            m = min(32, S - base)
            blk = np.zeros((n, 32), f32)
            blk[:, :m] = v[:, base:base + m]
            scan = blk.copy()
            for off in (1, 2, 4, 8, 16):
                nv = scan.copy()
                nv[:, :32 - off] = scan[:, :32 - off] + scan[:, off:]
                scan = nv
            out[:, base:base + m] = (tail[:, None] + scan - blk)[:, :m]
            tail = tail + scan[:, 0]
        return out

    def _suffix_quad(self, v, L):
        n, S = v.shape
        nq = S // 4
        vq = np.zeros((n, L, 4), f32)
        vq[:, :nq] = v.reshape(n, nq, 4)
        s2 = vq[..., 3]
        s1 = vq[..., 3] + vq[..., 2]
        s0 = s1 + vq[..., 1]
        scan = s0 + vq[..., 0]
        off = 1
        while off < L:
            nv = scan.copy()
            nv[:, :L - off] = scan[:, :L - off] + scan[:, off:]
            scan = nv
            off <<= 1
        last = scan[:, -1:] if self.defect == "quad_tail_kept" else np.zeros((n, 1), f32)   # shfl_down past the group
        tail = np.concatenate([scan[:, 1:], last], 1)                                        # returns the lane's own value
        return np.stack([tail + s0, tail + s1, tail + s2, tail], -1)[:, :nq].reshape(n, S)

    # ---- sampling
    def sample_pdf(self, bins, weights, u, eps=1e-5):
        return torch.from_numpy(sample_pdf32(_np(bins), _np(weights), _np(u), eps, self.defect))

    def importance_merge(self, z, w, u, eps=1e-5, want_new=True, sentinel=-7.0):
        z_, w_ = _np(z), _np(w)
        zn = sample_pdf32(z_mid32(z_), w_[:, 1:-1], _np(u), eps, self.defect)
        fine = merge32(z_, zn, self.defect, f32(sentinel))
        return torch.from_numpy(fine), (torch.from_numpy(zn) if want_new else None)
