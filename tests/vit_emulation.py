"""What the semantic-loss kernels (csrc/vit.cu) compute, restated in float64 for the layer-by-layer ViT tests.

- Layouts: the weight image (`vit_layout`) and the workspace (`vit_ws`) as float offsets, so a test can read every
  intermediate the kernels leave in buffers it allocated itself.  tests/test_vit_layerwise_cpu.py holds the restated
  totals equal to the library's byte counts.
- Operands: what each wgmma multiplies.  Split mode (fp32 / f16x3 / bf16x3): hi = fp16_rn(clamp(x, +-65504)),
  lo = fp16_rn(x_clamped - hi) with fp16 subnormals kept, products lo.hi + hi.lo + hi.hi; f16: the hi word alone;
  bf16: bf16_rn(x).
- Stage references in float64 with the kernels' epilogues (alpha, bias, residual, exact-erf GELU, its derivative,
  pos_embed), and the per-element error measure |y - y_ref| / (sum_k |a_k||b_k| + |bias| + |residual|).
- BARS: the per-stage bars of tests/test_gpu_vit_layerwise.py, shared with the CPU test that plants defects under them.
"""
import math

import torch

DIM, HEADS, HD, TOK, PATCHES, GRID, MLP, QKV, PATCHK, BLOCKS, RES = 384, 6, 64, 197, 196, 14, 1536, 1152, 768, 12, 224
LDS = 200                    # row stride of the 197 x 197 score tiles
TILE_S = TOK * LDS
ALPHA = 0.125                # 64 ** -0.5
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
# operand mode -> SNB_PREC_* id that runs it ('fp32', 'f16x3' and 'bf16x3' all run the split)
MODES = {"split": 1, "f16": 4, "bf16": 3}


def _al(x, a):
    return (x + a - 1) // a * a


# --------------------------------------------------------------------------------------------------------------------
# layouts
# --------------------------------------------------------------------------------------------------------------------
def pack_layout(mode):
    """vit_layout: {'cls','pos','pe_b': float offsets, 'pe': 16-bit element offset, 'blk': [12 dicts], 'n_floats',
    'n_halfs', 'planes'}.  fp32 vectors 64-float aligned, then 16-bit planes 128-element aligned (hi then lo)."""
    planes = 2 if mode == "split" else 1
    f = h = 0

    def vec(n):
        nonlocal f
        o, f = f, _al(f + n, 64)
        return o

    def mat(n):
        nonlocal h
        o, h = h, _al(h + planes * n, 128)
        return o

    L = {"planes": planes, "cls": vec(DIM), "pos": vec(TOK * DIM), "pe_b": vec(DIM), "pe": mat(DIM * PATCHK), "blk": []}
    for _ in range(BLOCKS):
        B = {k: vec(n) for k, n in (("n1w", DIM), ("n1b", DIM), ("qkv_b", QKV), ("proj_b", DIM), ("n2w", DIM),
                                    ("n2b", DIM), ("fc1_b", MLP), ("fc2_b", DIM))}
        B.update({k: mat(n) for k, n in (("qkv", QKV * DIM), ("proj", DIM * DIM), ("fc1", MLP * DIM),
                                         ("fc2", DIM * MLP))})
        L["blk"].append(B)
    L["n_floats"], L["n_halfs"] = f, h
    return L


def pack_bytes(mode):
    L = pack_layout(mode)
    return L["n_floats"] * 4 + L["n_halfs"] * 2


def workspace_layout(n, save):
    """vit_ws: ({name: (float offset, shape)}, total floats).  Every buffer starts 64-float aligned; the per-block saved
    state is 'blk{l}.x_in', 'blk{l}.x_mid', 'blk{l}.qkv', 'blk{l}.O', 'blk{l}.pre', 'blk{l}.lse'."""
    bufs, off = {}, 0

    def take(name, *shape):
        nonlocal off
        bufs[name] = (off, shape)
        off = _al(off + math.prod(shape), 64)

    take("col", n, PATCHES, PATCHK)
    for k in ("X0", "X1", "ln"):
        take(k, n, TOK, DIM)
    take("qkv", n, TOK, QKV)
    take("O", n, TOK, DIM)
    take("h", n, TOK, MLP)
    take("S", n, HEADS, TOK, LDS)
    take("dP", n, HEADS, TOK, LDS)
    take("lse", n, HEADS, TOK)
    for k, w in (("xmid_c", DIM), ("ln_c", DIM), ("O_c", DIM), ("h_c", MLP), ("pre_c", MLP), ("lse_c", HEADS)):
        take(k, n, w)
    if save:
        for k in ("dx", "dx2", "dln"):
            take(k, n, TOK, DIM)
        take("dqkv", n, TOK, QKV)
        take("dO", n, TOK, DIM)
        take("dh", n, TOK, MLP)
        for k, w in (("c0", DIM), ("c1", DIM), ("c2", DIM), ("ch", MLP)):
            take(k, n, w)
        take("inv", n)
        for l in range(BLOCKS):
            for k, w in (("x_in", DIM), ("x_mid", DIM), ("qkv", QKV), ("O", DIM), ("pre", MLP)):
                take(f"blk{l}.{k}", n, TOK, w)
            take(f"blk{l}.lse", n, HEADS, TOK)
    return bufs, off


def workspace_views(ws, n, save):
    """{name: view} of a float32 workspace tensor, shaped as workspace_layout says."""
    bufs, total = workspace_layout(n, save)
    assert ws.dtype == torch.float32 and ws.numel() >= total
    return {k: ws[o:o + math.prod(s)].view(*s) for k, (o, s) in bufs.items()}


# --------------------------------------------------------------------------------------------------------------------
# operands and products
# --------------------------------------------------------------------------------------------------------------------
def operand(x, mode):
    """fp32 x -> (hi, lo) as the fp32 values the kernel's wgmmas multiply (lo None: one product)."""
    x = x.float()
    if mode == "bf16":
        return x.bfloat16().float(), None
    x = x.clamp(-65504.0, 65504.0)
    hi = x.half().float()
    if mode == "f16":
        return hi, None
    return hi, (x - hi).half().float()


def packed_planes(w, mode):
    """The int16 plane(s) vit_pack_kernel writes for an fp32 weight: [hi] or [hi, lo]."""
    w = w.float()
    if mode == "bf16":
        return [w.bfloat16().view(torch.int16)]
    w = w.clamp(-65504.0, 65504.0)
    hi = w.half()
    if mode == "f16":
        return [hi.view(torch.int16)]
    return [hi.view(torch.int16), (w - hi.float()).half().view(torch.int16)]


class Prod:
    """float64 sum_k a[..., m, k] b[..., n, k]: `emu` over the operands the kernel multiplies, `exact` over the
    unrounded fp32 values, `abs` = sum_k |a||b| (the error scale)."""

    def __init__(self, a, b, mode, k_chunks_without_lo_hi=()):
        a, b = a.float(), b.float()
        ah, al = operand(a, mode)
        bh, bl = operand(b, mode)
        d = torch.float64
        bt = bh.to(d).transpose(-1, -2)
        self.emu = ah.to(d) @ bt
        if al is not None:
            self.emu += al.to(d) @ bt + ah.to(d) @ bl.to(d).transpose(-1, -2)
            for c in k_chunks_without_lo_hi:       # planted defect: one 64-deep chunk missing its lo.hi product
                ks = slice(64 * c, 64 * (c + 1))
                self.emu -= al[..., ks].to(d) @ bt[..., ks, :]
        self.exact = a.to(d) @ b.to(d).transpose(-1, -2)
        self.abs = a.to(d).abs() @ b.to(d).abs().transpose(-1, -2)


def gelu64(x):
    x = x.double()
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x, magnitude=False):
    """GELU'(x) = cdf(x) + x pdf(x); magnitude: cdf + |x| pdf, the error scale of the fp32 sum, which cancels to 0
    near x = -0.75"""
    x = x.double()
    cdf, xpdf = 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))), x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    return cdf + xpdf.abs() if magnitude else cdf + xpdf


def ln64(x, g, b):
    return torch.nn.functional.layer_norm(x.double(), (DIM,), g.double(), b.double(), 1e-6)


def ln_bwd64(x, g, dy, dy_abs=None):
    """(dx, scale) of LayerNorm's input gradient (no residual).  scale bounds how errors of size |dy| (dy_abs: a bound
    on dy's own error scale, default |dy|) propagate: rstd (|g dy| + mean |g dy| + |xh| mean |g dy xh|)."""
    x, g, dy = x.double(), g.double(), dy.double()
    mu = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt((x - mu).square().mean(-1, keepdim=True) + 1e-6)
    xh = (x - mu) * rstd
    gd = dy * g
    dx = rstd * (gd - gd.mean(-1, keepdim=True) - xh * (gd * xh).mean(-1, keepdim=True))
    ga = (dy.abs() if dy_abs is None else dy_abs) * g.abs()
    scale = rstd * (ga + ga.mean(-1, keepdim=True) + xh.abs() * (ga * xh.abs()).mean(-1, keepdim=True))
    return dx, scale


def linear_ref(x, w, b, mode, resid=None, k_chunks_without_lo_hi=()):
    """y = x w^T + b (+ resid), the GEMM epilogue EPI_STORE / EPI_RESID / EPI_EMBED: (emu, exact, scale)"""
    p = Prod(x, w, mode, k_chunks_without_lo_hi)
    add, scale = b.double(), p.abs + b.double().abs()
    if resid is not None:
        add, scale = add + resid.double(), scale + resid.double().abs()
    return p.emu + add, p.exact + add, scale


def dgrad_ref(dy, w, mode):
    """dx = dy w (a Linear's input gradient: B(n, k) = w[k][n]): (emu, exact, scale)"""
    p = Prod(dy, w.t(), mode)
    return p.emu, p.exact, p.abs


def scores_ref(q, k, mode, alpha=ALPHA):
    """q (.., r, 64), k (.., 197, 64) -> (lse emu, lse exact, scale, P emu): the row log-sum-exp of alpha q k^T, its error
    scale alpha max_j sum_d |q||k| (lse moves by at most the largest score error), and the float64 softmax."""
    p = Prod(q, k, mode)
    s, se = alpha * p.emu, alpha * p.exact
    return torch.logsumexp(s, -1), torch.logsumexp(se, -1), alpha * p.abs.amax(-1), torch.softmax(s, -1)


def pv_ref(P, v, mode):
    """O = P V with P (.., r, 197) float64 rounded to fp32 as the kernel stores it, v (.., 197, 64)"""
    p = Prod(P.float(), v.transpose(-1, -2), mode)
    return p.emu, p.exact, p.abs


def err(y, ref, scale):
    """per-element |y - ref| / scale (scale 0 only where both are 0)"""
    return (y.double() - ref).abs() / scale.clamp_min(1e-300)


def stats(e):
    """(worst, rms) of an error tensor"""
    e = e.double().flatten()
    return float(e.max()), float(e.square().mean().sqrt())


def heads(t):
    """(n, rows, 384) -> (n, 6, rows, 64)"""
    n, r, _ = t.shape
    return t.reshape(n, r, HEADS, HD).transpose(1, 2)


def unheads(t):
    n, _, r, _ = t.shape
    return t.transpose(1, 2).reshape(n, r, DIM)


def im2col(img224):
    """(3, 224, 224) -> (196, 768): col[p][c 256 + ky 16 + kx]"""
    return img224.reshape(3, GRID, 16, GRID, 16).permute(1, 3, 0, 2, 4).reshape(PATCHES, PATCHK)


def col2im(col):
    return col.reshape(GRID, GRID, 3, 16, 16).permute(2, 0, 3, 1, 4).reshape(3, RES, RES)


# --------------------------------------------------------------------------------------------------------------------
# bars
# --------------------------------------------------------------------------------------------------------------------
# (worst, rms) of the per-element error against the operand emulation, per stage and mode, about 4x the largest value
# measured on an H100 SXM (80 GB, 700 W) over n = 1, 2, 8 (n = 1, 8 through zero blocks).  DESIGN.md section 2 lists
# the measurements.
BARS = {
    "split": {
        "embed": (3.4e-6, 5.5e-7), "qkv": (3.5e-6, 4.6e-7), "lse": (1.1e-6, 2.4e-7), "pv": (1.6e-5, 3.3e-6),
        "proj": (2.9e-6, 3.9e-7), "fc1": (4.1e-6, 4.7e-7), "fc2": (6.6e-6, 1.0e-6),
        "dfc2": (4.1e-6, 3.7e-7), "dfc1": (1.6e-6, 4.0e-7), "dproj": (2.7e-6, 4.6e-7), "P": (1.8e-6, 2.1e-7),
        "dS": (1.3e-6, 1.4e-7), "dqkv": (1.1e-5, 1.5e-6), "dqkvW": (8.5e-6, 9.8e-7), "dln1": (7.1e-7, 9.3e-8),
        "dembed": (3.2e-6, 4.5e-7),
        # through zero-weight blocks: block 11's token gradient, block 0's dh and dx2
        "b11tok": (4.4e-6, 1.6e-7), "dh0": (7.0e-6, 2.1e-8), "dx2_0": (6.6e-6, 1.8e-7),
    },
    "f16": {
        "embed": (1.4e-6, 2.0e-7), "qkv": (2.1e-4, 5.1e-6), "lse": (6.1e-7, 1.3e-7), "pv": (3.0e-3, 5.3e-5),
        "proj": (1.2e-6, 1.4e-7), "fc1": (1.3e-4, 2.7e-6), "fc2": (5.6e-5, 1.2e-6),
        "dfc2": (2.5e-6, 1.4e-7), "dfc1": (5.7e-7, 1.4e-7), "dproj": (1.2e-6, 1.7e-7), "P": (9.3e-7, 1.2e-7),
        "dS": (7.3e-7, 6.6e-8), "dqkv": (6.4e-6, 6.4e-7), "dqkvW": (3.7e-6, 3.4e-7), "dln1": (7.4e-7, 9.3e-8),
        "dembed": (1.2e-6, 1.6e-7),
        # through zero-weight blocks: block 11's token gradient, block 0's dh and dx2
        "b11tok": (4.2e-5, 4.9e-7), "dh0": (6.8e-6, 5.4e-8), "dx2_0": (1.6e-5, 1.1e-7),
    },
    "bf16": {
        "embed": (1.1e-6, 1.3e-7), "qkv": (8.8e-4, 1.9e-5), "lse": (4.5e-7, 8.9e-8), "pv": (1.0e-2, 1.8e-4),
        "proj": (1.1e-6, 1.1e-7), "fc1": (1.1e-3, 9.1e-6), "fc2": (3.2e-4, 4.0e-6),
        "dfc2": (2.1e-6, 1.1e-7), "dfc1": (6.0e-7, 1.3e-7), "dproj": (8.7e-7, 1.2e-7), "P": (8.1e-7, 9.2e-8),
        "dS": (5.0e-7, 4.5e-8), "dqkv": (5.3e-6, 5.2e-7), "dqkvW": (3.3e-6, 3.0e-7), "dln1": (7.7e-7, 9.4e-8),
        "dembed": (9.0e-7, 1.2e-7),
        # through zero-weight blocks: block 11's token gradient, block 0's dh and dx2
        "b11tok": (1.9e-4, 3.7e-6), "dh0": (3.2e-5, 2.3e-7), "dx2_0": (3.7e-4, 3.2e-6),
    },
}
