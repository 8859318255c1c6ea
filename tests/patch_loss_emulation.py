"""References for the patch-loss kernels (sinnerf_b200/csrc/patch_loss.cu) and a CPU stand-in for them.

Three things, none of which imports the library:

* float64 truth of each stage, on whatever device the inputs live on.  `ssim64`: the five window sums, mu1, mu2, s1, s2,
  s12, u, the loss terms and the three coefficient maps the forward writes (dL/dmu1, dL/df(x^2), dL/df(xy) for a unit
  upstream gradient) in closed form, with the window sums taken by tests/patch_loss_oracle.py's filter2d.
  `adjoint64`: the image gradient from ANY coefficient maps, as float64 autograd of that same reflect-pad + depthwise
  conv2d (it does not restate the kernels' mirror-term weights).  `smooth64`: the smoothness loss and gradients by
  float64 autograd of the oracle, with the per-element sums of |terms| the error bounds use.
* the bounds: every error is divided by the float64 sum of absolute values of the terms that form the element.  For
  the coefficient maps that sum is multiplied by the condition `kappa` of the two variance sums A2 = 2 s12 + C2 and
  B2 = s1 + s2 + C2, which cancel most of their digits on smooth depth patches.
* `StandIn`: the entry points of include/sinnerf_b200.h the stage tests drive, on CPU tensors, written out as the
  kernels compute: SSIM over 16x32 output tiles with a 5-pixel halo staged with the reflection applied at load and two
  separable 11-tap passes, the backward's staged coefficient tiles and its 1-D adjoint weight with the mirror terms,
  the grid-stride walk over tiles under the launch caps, the smoothness edges per pixel, and the loss ticket on the
  shared scratch.  numpy's exp is not CUDA's expf and its sums are not the kernels' order, so the stand-in is not
  bitwise; it exists so that the checkers of tests/test_gpu_patch_loss_stages.py can be exercised, and shown to catch
  planted defects, without a GPU.  `StandIn(defect=...)` plants one defect (names in DEFECTS).
"""
import numpy as np
import torch

from tests import patch_loss_oracle as plo

f32 = np.float32
WIN, PAD = 11, 5
TH, TW = 16, 32                       # SSIM output tile
THREADS = 256
LOSS_WS_FLOATS = 4096                 # SNB_LOSS_WS_FLOATS
MAX_LOSS_BLOCKS = (LOSS_WS_FLOATS - 4) // 2   # block partials that fit in the loss scratch: 2046
U_ROUND = 2.0 ** -48                  # rounding scale of u in fp64, per unit of (1 + |ssim| kappa)

DEFECTS = (
    "mirror_q1",            # SSIM backward: the top / left mirror term dropped at q = 1
    "mirror_n6",            # SSIM backward: the bottom / right mirror term dropped at q = n - 6
    "halo_shift",           # SSIM forward: the left halo of a tile past the first column seam read one column left
    "taps_fp32",            # both SSIM kernels: the Gaussian taps rounded to fp32
    "coef_next_plane",      # SSIM backward: coefficient maps staged from the next plane
    "strict_gate",          # SSIM forward: the clamp passes the gradient only for 0 < u < 1
    "last_tile_skipped",    # SSIM forward: the grid-stride loop stops one tile short when it takes a second trip
    "clamp_swallows_nan",   # SSIM forward: fmin(fmax(u, 0), 1) adds 0 for a NaN u
    "sign0_is_1",           # smoothness backward: sign(0) = 1
    "no_inv_c",             # smoothness backward: the 1/C of the channel mean dropped from the image gradient
    "ticket_not_reset",     # the loss scratch's ticket word is left non-zero
)


# ------------------------------------------------------------------------------------------------ launch geometry
def ssim_tiles(B, C, H, W):
    return B * C * -(-H // TH) * -(-W // TW)


def ssim_fwd_grid(n_tiles):
    return min(n_tiles, MAX_LOSS_BLOCKS)


def ssim_bwd_grid(n_tiles, sm_count):
    return min(n_tiles, 8 * sm_count)


def smooth_fwd_grid(n_pixels):
    return max(1, min(-(-n_pixels // THREADS), MAX_LOSS_BLOCKS))


def smooth_bwd_grid(n_pixels, sm_count):
    return max(1, min(-(-n_pixels // THREADS), 16 * sm_count))


# ------------------------------------------------------------------------------------------------ float64 truth
def _filter(t):
    return plo.filter2d(t, plo.gaussian_2d(WIN, 1.5, torch.float64, t.device))


def ssim_constants(max_val):
    return (0.01 * max_val) ** 2, (0.03 * max_val) ** 2


def ssim64(x, y, max_val=1.0, eps=1e-12):
    """Every per-pixel quantity of ssim_loss(x, y, 11, max_val, eps) in float64, from the float32 inputs as given.
    Pass max_val and eps as the kernel receives them (rounded to float32) to compare with the kernel."""
    X, Y = x.double(), y.double()
    n = X.shape[0]
    f = _filter(torch.cat([X, Y, X * X, Y * Y, X * Y, X.abs(), Y.abs(), (X * Y).abs()], 0))
    mu1, mu2, fxx, fyy, fxy, fax, fay, faxy = f.split(n, 0)
    c1, c2 = ssim_constants(max_val)
    s1, s2, s12 = fxx - mu1 * mu1, fyy - mu2 * mu2, fxy - mu1 * mu2
    A1, A2 = 2.0 * mu1 * mu2 + c1, 2.0 * s12 + c2
    B1, B2 = mu1 * mu1 + mu2 * mu2 + c1, s1 + s2 + c2
    den = B1 * B2 + eps
    ssim = A1 * A2 / den
    u = (1.0 - ssim) * 0.5
    inv_n = 1.0 / X.numel()
    terms = torch.clamp(u, 0, 1)

    def coefs(gs):
        dA1, dA2 = gs * A2 / den, gs * A1 / den
        dB1, dB2 = -gs * ssim * B2 / den, -gs * ssim * B1 / den
        c = torch.stack([2.0 * mu2 * (dA1 - dA2) + 2.0 * mu1 * (dB1 - dB2), dB2, 2.0 * dA2])
        t = torch.stack([2.0 * mu2.abs() * (dA1.abs() + dA2.abs()) + 2.0 * mu1.abs() * (dB1.abs() + dB2.abs()),
                         dB2.abs(), 2.0 * dA2.abs()])
        return c, t

    gate = (u >= 0) & (u <= 1)
    coef, cterms = coefs(gate.double() * (-0.5 * inv_n))
    coef_open, cterms_open = coefs(torch.full_like(u, -0.5 * inv_n))
    kappa = (1.0 + (2.0 * (faxy + (mu1 * mu2).abs()) + c2) / A2.abs() + (fxx + mu1 * mu1 + fyy + mu2 * mu2 + c2) / B2.abs()
             + (2.0 * (mu1 * mu2).abs() + c1) / A1.abs())
    du = U_ROUND * (1.0 + ssim.abs() * kappa)
    return dict(mu1=mu1, mu2=mu2, fxx=fxx, fyy=fyy, fxy=fxy, s1=s1, s2=s2, s12=s12, A1=A1, A2=A2, B1=B1, B2=B2,
                den=den, ssim=ssim, u=u, terms=terms, loss=terms.mean(), loss_bound=(terms.abs() + du).mean(),
                coef=coef, coef_bound=cterms_open * kappa, coef_open=coef_open, gate=gate, kappa=kappa, du=du,
                exact=(fax == 0) & (fay == 0), inv_n=inv_n)


def adjoint64(coef, x, y):
    """(g, bound) for a unit upstream gradient: g = F^T c0 + 2 x F^T c1 + y F^T c2, F = reflect-pad by 5 then correlate
    with the 11x11 Gaussian, F^T by float64 autograd through plo.filter2d; bound the same with |c|, |x|, |y|.
    coef (3, B, C, H, W); x, y (B, C, H, W)."""
    B = x.shape[0]
    c = coef.double()
    z = torch.zeros((6 * B,) + tuple(x.shape[1:]), dtype=torch.float64, device=x.device, requires_grad=True)
    (a,) = torch.autograd.grad(_filter(z), z, grad_outputs=torch.cat([c[0], c[1], c[2], c[0].abs(), c[1].abs(),
                                                                       c[2].abs()], 0))
    a = a.split(B, 0)
    X, Y = x.double(), y.double()
    return a[0] + 2.0 * X * a[1] + Y * a[2], a[3] + 2.0 * X.abs() * a[4] + Y.abs() * a[5]


def smooth64(d, img):
    """Loss and gradients of inverse_depth_smoothness_loss in float64 autograd of the oracle, and the bounds: the loss
    sum itself (its terms are |.|), per pixel inv_n * sum of incident-edge weights for g_d, inv_n / C * sum of
    |d(p) - d(q)| w over incident edges for g_img."""
    D, I = d.double().requires_grad_(True), img.double().requires_grad_(True)
    loss = plo.inverse_depth_smoothness_loss(D, I)
    gd, gi = torch.autograd.grad(loss, (D, I))
    D, I = D.detach(), I.detach()
    B, C, H, W = I.shape
    inv_nx, inv_ny = 1.0 / (B * H * (W - 1)), 1.0 / (B * (H - 1) * W)
    wx = torch.exp(-(I[..., :-1] - I[..., 1:]).abs().mean(1, keepdim=True))
    wy = torch.exp(-(I[..., :-1, :] - I[..., 1:, :]).abs().mean(1, keepdim=True))
    tx, ty = ((D[..., :-1] - D[..., 1:]) * wx).abs(), ((D[..., :-1, :] - D[..., 1:, :]) * wy).abs()

    def incident(ex, ey):   # per pixel: the sum over its (up to four) incident edges
        s = torch.zeros(B, 1, H, W, dtype=torch.float64, device=d.device)
        s[..., :-1] += ex; s[..., 1:] += ex; s[..., :-1, :] += ey; s[..., 1:, :] += ey
        return s
    return dict(loss=loss.detach(), loss_bound=tx.mean() + ty.mean(), g_d=gd, g_img=gi,
                g_d_bound=incident(inv_nx * wx, inv_ny * wy), g_img_bound=incident(inv_nx * tx, inv_ny * ty) / C)


# ------------------------------------------------------------------------------------------------ the stand-in
def _taps(fp32=False):
    x = np.arange(WIN, dtype=np.float64) - PAD
    g = np.exp(-x * x / (2.0 * 1.5 * 1.5))
    g = g / g.sum()
    return g.astype(f32).astype(np.float64) if fp32 else g


def _reflect(k, n):
    k = np.where(k < 0, -k, np.where(k >= n, 2 * (n - 1) - k, k))
    return np.clip(k, 0, n - 1)


def _adj_weight(g, p, q, n, defect):
    """The kernels' 1-D adjoint weight, vectorised over p and q."""
    def tap(k):
        return np.where((k >= -PAD) & (k <= PAD), g[np.clip(k + PAD, 0, WIN - 1)], 0.0)
    lo = (q >= 1) & (q <= PAD) & ~((q == 1) & (defect == "mirror_q1"))
    hi = (q >= n - 1 - PAD) & (q <= n - 2) & ~((q == n - 6) & (defect == "mirror_n6"))
    return tap(q - p) + np.where(lo, tap(-q - p), 0.0) + np.where(hi, tap(2 * (n - 1) - q - p), 0.0)


def _planes(t):
    B, C, H, W = t.shape
    return t.detach().cpu().numpy().reshape(B * C, H, W)


def _sgn(v, defect):
    s = np.where(np.isnan(v), 0, np.sign(v))          # torch.sign: sign(0) = sign(NaN) = 0
    if defect == "sign0_is_1":
        s = np.where(v == 0, 1, s)
    return s.astype(f32)


class StandIn:
    """The patch-loss entry points on CPU float32 tensors.  `sm_count` fixes the backward launch caps as on a 132-SM
    part.  Outputs are written into caller-owned tensors, through their strides, as the C ABI does."""
    sm_count = 132
    device = "cpu"

    def __init__(self, defect=None):
        assert defect is None or defect in DEFECTS, defect
        self.defect = defect

    def _ticket(self, ws):
        assert int(ws.view(torch.int32)[0]) == 0, "loss scratch ticket was not zero on entry"
        if self.defect == "ticket_not_reset":
            ws.view(torch.int32)[0] = 1

    # ---- SSIM
    def _tiles(self, B, C, H, W):
        th, tw = -(-H // TH), -(-W // TW)
        t = np.arange(B * C * th * tw)
        return t % tw * TW, (t // tw) % th * TH, t // (tw * th)

    def ssim_forward(self, x, y, max_val, eps, loss, coef, ws):
        d = self.defect
        B, C, H, W = x.shape
        X, Y = _planes(x), _planes(y)
        c0, r0, plane = self._tiles(B, C, H, W)
        n_tiles = len(plane)
        if d == "last_tile_skipped" and n_tiles > ssim_fwd_grid(n_tiles):
            c0, r0, plane = c0[:-1], r0[:-1], plane[:-1]
        rr, cc = np.arange(TH + 2 * PAD), np.arange(TW + 2 * PAD)
        gi = _reflect(r0[:, None] + rr[None, :] - PAD, H)
        cols = c0[:, None] + cc[None, :] - PAD
        if d == "halo_shift":
            cols = np.where((c0[:, None] > 0) & (cc[None, :] < PAD), cols - 1, cols)
        gj = _reflect(cols, W)
        sx = X[plane[:, None, None], gi[:, :, None], gj[:, None, :]].astype(np.float64)
        sy = Y[plane[:, None, None], gi[:, :, None], gj[:, None, :]].astype(np.float64)
        g = _taps(d == "taps_fp32")
        maps = (sx, sy, sx * sx, sy * sy, sx * sy)
        hs = [sum(g[k] * m[:, :, k:k + TW] for k in range(WIN)) for m in maps]
        mu1, mu2, fxx, fyy, fxy = (sum(g[k] * h[:, k:k + TH, :] for k in range(WIN)) for h in hs)
        mv = float(f32(max_val))
        c1, c2 = (0.01 * mv) * (0.01 * mv), (0.03 * mv) * (0.03 * mv)
        inv_n = 1.0 / (B * C * H * W)
        with np.errstate(all="ignore"):
            s1, s2, s12 = fxx - mu1 * mu1, fyy - mu2 * mu2, fxy - mu1 * mu2
            A1, A2 = 2.0 * mu1 * mu2 + c1, 2.0 * s12 + c2
            B1, B2 = mu1 * mu1 + mu2 * mu2 + c1, s1 + s2 + c2
            den = B1 * B2 + float(f32(eps))
            ssim = A1 * A2 / den
            u = (1.0 - ssim) * 0.5
            clamped = np.fmin(np.fmax(u, 0.0), 1.0)
            if d != "clamp_swallows_nan":
                clamped = np.where(np.isnan(u), u, clamped)
            gate = ((u > 0) & (u < 1)) if d == "strict_gate" else ((u >= 0) & (u <= 1))
            gs = np.where(gate, -0.5 * inv_n, 0.0)
            dA1, dA2 = gs * A2 / den, gs * A1 / den
            dB1, dB2 = -gs * ssim * B2 / den, -gs * ssim * B1 / den
            maps = (2.0 * mu2 * (dA1 - dA2) + 2.0 * mu1 * (dB1 - dB2), dB2, 2.0 * dA2)
        i = r0[:, None, None] + np.arange(TH)[None, :, None]
        j = c0[:, None, None] + np.arange(TW)[None, None, :]
        valid = (i < H) & (j < W)
        i, j = np.broadcast_to(i, valid.shape), np.broadcast_to(j, valid.shape)
        pl = np.broadcast_to(plane[:, None, None], valid.shape)
        lsum = clamped[valid].astype(f32).sum(dtype=f32)
        self._ticket(ws)
        loss.copy_(torch.tensor(f32(inv_n) * lsum))
        if coef is not None:
            total = B * C * H * W
            o = pl[valid] * H * W + i[valid] * W + j[valid]
            cf = coef.numpy()
            for m in range(3):
                cf[m * total + o] = maps[m][valid]

    def ssim_backward(self, x, y, coef, g_loss, g_x):
        d = self.defect
        B, C, H, W = x.shape
        P, total = B * C, B * C * H * W
        X, Y = _planes(x), _planes(y)
        cf = coef.detach().cpu().numpy().reshape(3, P, H, W)
        c0, r0, plane = self._tiles(B, C, H, W)
        src = np.minimum(plane + 1, P - 1) if d == "coef_next_plane" else plane
        pi = r0[:, None] + np.arange(TH + 2 * PAD)[None, :] - PAD
        pj = c0[:, None] + np.arange(TW + 2 * PAD)[None, :] - PAD
        inside = ((pi >= 0) & (pi < H))[:, :, None] & ((pj >= 0) & (pj < W))[:, None, :]
        pic, pjc = np.clip(pi, 0, H - 1), np.clip(pj, 0, W - 1)
        sv = [np.where(inside, cf[m][src[:, None, None], pic[:, :, None], pjc[:, None, :]], 0.0) for m in range(3)]
        g = _taps(d == "taps_fp32")
        q = c0[:, None] + np.arange(TW)[None, :]                                    # (n, 32) columns
        wq = [np.where(q < W, _adj_weight(g, q + k - PAD, q, W, d), 0.0) for k in range(WIN)]
        su = [sum(wq[k][:, None, :] * s[:, :, k:k + TW] for k in range(WIN)) for s in sv]
        qr = r0[:, None] + np.arange(TH)[None, :]                                   # (n, 16) rows
        wr = [_adj_weight(g, qr + k - PAD, qr, H, d) for k in range(WIN)]
        s0, s1, s2 = (sum(wr[k][:, :, None] * s[:, k:k + TH, :] for k in range(WIN)) for s in su)
        i = np.broadcast_to(qr[:, :, None], s0.shape)
        j = np.broadcast_to(q[:, None, :], s0.shape)
        valid = (i < H) & (j < W)
        pl = np.broadcast_to(plane[:, None, None], s0.shape)[valid]
        iv, jv = i[valid], j[valid]
        xv, yv = X[pl, iv, jv].astype(np.float64), Y[pl, iv, jv].astype(np.float64)
        with np.errstate(all="ignore"):
            v = (s0[valid] + 2.0 * xv * s1[valid] + yv * s2[valid]).astype(f32) * f32(g_loss.cpu().numpy()[0])
        out = g_x.numpy()
        out[pl // C, pl % C, iv, jv] = v

    # ---- smoothness
    def _smooth_edges(self, d, img):
        D, I = d.detach().cpu().numpy(), img.detach().cpu().numpy()
        C = I.shape[1]
        with np.errstate(all="ignore"):
            mx = np.zeros(D[..., :-1].shape, f32)
            my = np.zeros(D[..., :-1, :].shape, f32)
            for c in range(C):
                mx = mx + np.abs(I[:, c:c + 1, :, :-1] - I[:, c:c + 1, :, 1:])
                my = my + np.abs(I[:, c:c + 1, :-1, :] - I[:, c:c + 1, 1:, :])
            wx, wy = np.exp(-(mx / f32(C))).astype(f32), np.exp(-(my / f32(C))).astype(f32)
            ddx, ddy = D[..., :-1] - D[..., 1:], D[..., :-1, :] - D[..., 1:, :]
        return D, I, wx, wy, ddx, ddy

    def smooth_forward(self, d, img, loss, ws):
        B, C, H, W = img.shape
        D, I, wx, wy, ddx, ddy = self._smooth_edges(d, img)
        with np.errstate(all="ignore"):
            sx = np.abs(ddx * wx).sum(dtype=f32)
            sy = np.abs(ddy * wy).sum(dtype=f32)
            inv_nx, inv_ny = f32(1.0 / (B * H * (W - 1))), f32(1.0 / (B * (H - 1) * W))
            v = inv_nx * sx + inv_ny * sy
        self._ticket(ws)
        loss.copy_(torch.tensor(v))

    def smooth_backward(self, d, img, g_loss, g_d, g_img):
        dfc = self.defect
        if g_d is None and g_img is None:
            return
        B, C, H, W = img.shape
        D, I, wx, wy, ddx, ddy = self._smooth_edges(d, img)
        g = f32(g_loss.cpu().numpy()[0])
        inv_nx, inv_ny = f32(1.0 / (B * H * (W - 1))), f32(1.0 / (B * (H - 1) * W))
        with np.errstate(all="ignore"):
            tx, ty = _sgn(ddx * wx, dfc) * inv_nx, _sgn(ddy * wy, dfc) * inv_ny
            gdx, gdy = tx * wx, ty * wy
            gmx, gmy = -(tx * ddx) * wx, -(ty * ddy) * wy
            if g_d is not None:
                z = np.zeros((B, 1, H, W), f32)
                a, b = z.copy(), z.copy()
                a[..., :-1] += gdx; a[..., :-1, :] += gdy          # (gd0 + gd1): right and lower edges
                b[..., 1:] += gdx; b[..., 1:, :] += gdy            # (gd2 + gd3): left and upper edges
                g_d.numpy()[...] = (a - b) * g
            if g_img is not None:
                acc = np.zeros((B, C, H, W), f32)
                sx_ = _sgn(I[..., :-1] - I[..., 1:], dfc)          # sgn(v - right) at p; sgn(left - v) at p + 1
                sy_ = _sgn(I[..., :-1, :] - I[..., 1:, :], dfc)
                acc[..., :-1] += gmx * sx_
                acc[..., :-1, :] += gmy * sy_
                acc[..., 1:] -= gmx * sx_
                acc[..., 1:, :] -= gmy * sy_
                inv_c = f32(1) if dfc == "no_inv_c" else f32(1.0) / f32(C)
                g_img.numpy()[...] = acc * inv_c * g
