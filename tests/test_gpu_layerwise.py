"""The field MLP's forward and backward kernels, layer by layer, against plain float64.

The end-to-end bars (render outputs to 1e-4, parameter gradients to 1e-3 per tensor) cannot see a kernel that drops a
low-order product of one K chunk, mishandles one 128-point tile of a 2 M-point training pass, or loses the last tile of
a wgrad slice.  Here every comparison starts from the kernel's OWN saved input of the layer, rounded the way the kernel
rounds its MMA operands, so errors do not compound and ReLU flips do not matter, and the error is normalised per
output:  e = |h - h_ref| / (|W| |x| + |b|).  Bounds sit about 10x above the distribution measured on an H100 SXM
(80 GB, 700 W) with correct kernels; the measured numbers are written beside each bound.

The float64 reference runs on the GPU in blocks of 64 k points; it never reads the reference checkout.
"""
import math

import pytest
import torch

from oracle import render_oracle as orc
from tests._common import rel_l2, room_params

DEV = "cuda:0"
NAMES = list(orc.param_shapes())          # the 24 tensors in state-dict order (the library's parameter order)
LAYERS = [f"xyz_encoding_{i + 1}.0" for i in range(8)]
MODES = ["fp32", "f16x3", "bf16x3", "bf16"]
BLOCK = 1 << 16                           # points per block of the float64 reference


# --------------------------------------------------------------------------------------------------------------------
# helpers: rounding of MMA operands, act16 decoding, float64 forward / backward
# --------------------------------------------------------------------------------------------------------------------
SPLIT_MODES = ("f16x3", "bf16x3")


def _known(mode):
    if mode not in ("fp32", "f16x3", "bf16x3", "bf16", "f16"):
        raise ValueError(f"unknown precision mode {mode!r}")


def rn16(x, mode):
    """fp32 -> the fp32 value of its round-to-nearest 16-bit form: fp16 saturated at +-65504 (f16x3, f16) or bf16
    (bf16x3, bf16)."""
    _known(mode)
    if mode in ("f16x3", "f16"):
        return x.clamp(-65504.0, 65504.0).half().float()
    if mode in ("bf16x3", "bf16"):
        return x.bfloat16().float()
    raise ValueError(f"mode {mode!r} has no 16-bit operands")


def rz16(x, mode):
    """Non-negative fp32 -> its 16-bit form rounded toward zero (cvt.rz[.satfinite]): fp16 (f16x3, f16) or bf16."""
    _known(mode)
    if mode in ("f16x3", "f16"):
        h = x.clamp(max=65504.0).half()
        over = h.float() > x
        return torch.where(over, (h.view(torch.int16) - 1).view(torch.float16), h).float()
    if mode in ("bf16x3", "bf16"):
        return (x.view(torch.int32) & -65536).view(torch.float32)
    raise ValueError(f"mode {mode!r} has no 16-bit operands")


def operand(x, mode, nonneg=False):
    """(hi, lo) of an fp32 tensor as split16 / split_pair form an MMA operand (lo None: single product).
    nonneg: a ReLU output of the training epilogue (one-sided saturation in fp16)."""
    _known(mode)
    x = x.float()
    if mode == "fp32":
        return x, None
    if mode in ("f16x3", "f16"):
        x = x.clamp(max=65504.0) if nonneg else x.clamp(-65504.0, 65504.0)
    hi = rn16(x, mode)
    if mode not in SPLIT_MODES:
        return hi, None
    return hi, rn16(x - hi, mode)


def operand_relu_inference(pre, mode):
    """(hi, lo) of relu(pre) as split_pair_relu forms the next layer's operand in the inference schedule:
    hi rounded toward zero, lo round-to-nearest of the residual (split modes); one round-to-nearest, saturated in
    fp16 (cvt.rn.relu[.satfinite]), in the single-product modes."""
    _known(mode)
    x = torch.relu(pre.float())
    if mode == "fp32":
        return x, None
    if mode not in SPLIT_MODES:
        return rn16(x, mode), None
    hi = rz16(x, mode)
    lo = torch.relu(rn16(x - hi, mode))
    return hi, lo


def prod(xo, wo):
    """sum_k x[k] w[n][k] over the products the kernel issues: xh wh (+ xl wh + xh wl), in float64."""
    xh, xl = xo
    wh, wl = wo
    out = xh.double() @ wh.double().t()
    if xl is not None:
        out += xl.double() @ wh.double().t() + xh.double() @ wl.double().t()
    return out


def absprod(xo, wo):
    xh, xl = xo
    wh, wl = wo
    x = xh.double() + (0 if xl is None else xl.double())
    w = wh.double() + (0 if wl is None else wl.double())
    return x.abs() @ w.abs().t()


def folded(p):
    """W' = Wd[:, :256] Wf and b' = bd + Wd[:, :256] bf, formed in float64 and rounded once to fp32 (pack_tc_kernel)."""
    Wd, bd = p["dir_encoding.0.weight"].double(), p["dir_encoding.0.bias"].double()
    Wf, bf = p["xyz_encoding_final.weight"].double(), p["xyz_encoding_final.bias"].double()
    return (Wd[:, :256] @ Wf).float(), (bd + Wd[:, :256] @ bf).float()


def shifted_softplus64(s):
    return torch.nn.functional.softplus(s - 1.0)


def widened_sigmoid64(x):
    return 0.5 * (1.0 + 1.002 * torch.tanh(0.5 * x))


def a16_pad(n):
    return (n + 127) // 128 * 128


def act16_sections(buf, P):
    """Views of the act16 buffer (csrc/act16.cuh): {'enc','dir','h0'..'h7','g'} -> int16 planes, 'mask' -> int32."""
    pp = a16_pad(P)
    secs, off = {}, 0
    for name, F in [("enc", 64), ("dir", 32)] + [(f"h{l}", 256) for l in range(8)] + [("g", 128)]:
        n = pp * F * 2
        secs[name] = (buf[off:off + n].view(torch.int16), F)
        off += n
    secs["mask"] = (buf[off:off + 8 * 8 * pp * 4].view(torch.int32), pp)
    return secs


def t32_rows(plane, F, idx):
    """Rows idx (int64, device) of a (Ppad, F) fp16 T32 tensor, as fp64: element (p, f) at 16-bit index
    ((p / 32) (F / 8) + f / 8) 256 + (p % 32) 8 + f % 8."""
    f = torch.arange(F, device=idx.device)
    i = ((idx[:, None] >> 5) * (F >> 3) + (f >> 3)[None, :]) * 256 + (idx[:, None] & 31) * 8 + (f & 7)[None, :]
    return plane[i].view(torch.float16).double()


def mask_rows(words, pp, layer, idx):
    """ReLU mask of h_{layer+1} at rows idx: bit c of word w of layer l, point p at (l 8 + w) Ppad + p."""
    w = torch.stack([words[(layer * 8 + k) * pp + idx] for k in range(8)], 1)            # (n, 8)
    bits = (w[..., None] >> torch.arange(32, device=idx.device, dtype=torch.int32)) & 1
    return bits.reshape(idx.shape[0], 256).bool()


def act16_rows(secs, idx):
    """Everything the fp64 chain needs at rows idx, decoded from act16."""
    words, pp = secs["mask"]
    return dict(enc=t32_rows(*secs["enc"], idx)[:, :63], dir=t32_rows(*secs["dir"], idx)[:, :27],
                G=t32_rows(*secs["g"], idx), H=[t32_rows(*secs[f"h{l}"], idx) for l in range(8)],
                M=[mask_rows(words, pp, l, idx) for l in range(8)])


def fp32_rows(save, idx):
    H = [save["h"][l][idx].double() for l in range(8)]
    return dict(enc=save["enc"][idx, :63].double(), dir=save["dir"][idx, :27].double(), G=save["g"][idx].double(),
                H=H, M=[h > 0 for h in H])


def chain64(p, g_raw, raw, a, grads):
    """Explicit float64 backward of the field MLP (models/nerf.py:105-148 with new_activation) for one block of points,
    accumulated into grads {name: fp64}.  p: {name: fp64}; g_raw (n,4) = dL/d[r,g,b,sigma]; raw (n,4) the forward's
    output; a: enc (n,63), dir (n,27), G (n,128) the shifted softplus output, H[0..7] (n,256) = h1..h8, M[0..7] their
    ReLU masks.  The bottleneck is not folded: feat = Wf h8 + bf."""
    g_raw, raw = g_raw.double(), raw.double()
    t = (2.0 * raw[:, :3] - 1.0) / 1.002                       # tanh(x/2) of the rgb pre-activation
    gp = g_raw[:, :3] * 0.2505 * (1.0 - t * t)
    gs = g_raw[:, 3:4]
    grads["rgb.0.weight"] += gp.t() @ a["G"]
    grads["rgb.0.bias"] += gp.sum(0)
    grads["sigma.weight"] += gs.t() @ a["H"][7]
    grads["sigma.bias"] += gs.sum(0)
    dS = (gp @ p["rgb.0.weight"]) * -torch.expm1(-a["G"])      # softplus'(s) = sigmoid(s) = 1 - exp(-softplus(s))
    Wd, Wf = p["dir_encoding.0.weight"], p["xyz_encoding_final.weight"]
    feat = a["H"][7] @ Wf.t() + p["xyz_encoding_final.bias"]
    grads["dir_encoding.0.weight"] += dS.t() @ torch.cat([feat, a["dir"]], 1)
    grads["dir_encoding.0.bias"] += dS.sum(0)
    dfeat = dS @ Wd[:, :256]
    grads["xyz_encoding_final.weight"] += dfeat.t() @ a["H"][7]
    grads["xyz_encoding_final.bias"] += dfeat.sum(0)
    dh = dfeat @ Wf + gs * p["sigma.weight"]
    for l in range(7, -1, -1):
        dY = dh * a["M"][l]
        x = a["enc"] if l == 0 else (torch.cat([a["enc"], a["H"][3]], 1) if l == 4 else a["H"][l - 1])
        grads[LAYERS[l] + ".weight"] += dY.t() @ x
        grads[LAYERS[l] + ".bias"] += dY.sum(0)
        if l > 0:
            dx = dY @ p[LAYERS[l] + ".weight"]
            dh = dx[:, 63:] if l == 4 else dx
    return grads


def zero_grads(dev):
    return {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in orc.param_shapes().items()}


def to_dev(p, dtype=torch.float32):
    return {k: v.to(DEV, dtype).contiguous() for k, v in p.items()}


def weights_of(tag):
    return orc.default_init_params(1) if tag == "default" else room_params("fine")


def packed(p, precision):
    from sinnerf_b200 import _lib
    from sinnerf_b200.nerf import NeRF
    lib = _lib.load()
    prec = _lib.precision_id(precision)
    if precision != "fp32" and lib.snb_packed_weights_bytes(prec) == 0:
        pytest.skip(f"precision mode {precision} is not built")
    m = NeRF(use_new_activation=True)
    m.load_state_dict({k: v.cpu() for k, v in p.items()})
    m = m.to(DEV)
    return m, m.packed_weights(prec)


def ray_batch(scene, n_rays, S, seed):
    """n_rays rays of a synthetic frame with S stratified, sorted depths in [near, far]."""
    from sinnerf_b200 import synthetic
    rays = synthetic.random_rays(scene, n_rays, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    t = (torch.arange(S, dtype=torch.float32)[None, :] + torch.rand(n_rays, S, generator=g)) / S
    z = rays[:, 6:7] + (rays[:, 7:8] - rays[:, 6:7]) * t
    return rays.to(DEV).contiguous(), z.to(DEV).contiguous()


def points32(rays, z):
    """(P,3) fp32 sample points with the mul and the add rounded separately (rendering.py:284-285)."""
    o, d = rays[:, None, 0:3], rays[:, None, 3:6]
    return (o + d * z[..., None]).reshape(-1, 3), rays[:, 3:6].repeat_interleave(z.shape[1], 0)


def forward_train(img, precision, rays, z):
    from sinnerf_b200 import _lib
    lib = _lib.load()
    n, S = z.shape
    P = n * S
    raw = torch.full((n, S, 4), float("nan"), device=DEV)
    save = {k: torch.full(shape, float("nan"), device=DEV)
            for k, shape in (("enc", (P, 64)), ("dir", (P, 32)), ("h", (8, P, 256)), ("g", (P, 128)))}
    _lib.check(lib.snb_field_forward_train(_lib.ptr(img), _lib.precision_id(precision), _lib.ptr(rays), _lib.ptr(z), n, S,
                                           _lib.ptr(raw), _lib.ptr(save["enc"]), _lib.ptr(save["dir"]),
                                           _lib.ptr(save["h"]), _lib.ptr(save["g"]), _lib.stream_ptr(torch.device(DEV))),
               "snb_field_forward_train")
    torch.cuda.synchronize()
    return raw.reshape(P, 4), save


class Stat:
    """max and rms of a normalised error, accumulated over blocks."""

    def __init__(self):
        self.max, self.ss, self.n = 0.0, 0.0, 0

    def add(self, e):
        e = e.double()
        self.max = max(self.max, float(e.max()))
        self.ss += float((e * e).sum())
        self.n += e.numel()

    @property
    def rms(self):
        return math.sqrt(self.ss / max(self.n, 1))


def report(title, stats):
    print(f"\n{title}")
    for k, s in stats.items():
        print(f"  {k:>8}: max {s.max:.3e}  rms {s.rms:.3e}")
    print(f"  peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


# --------------------------------------------------------------------------------------------------------------------
# 1. the float64 chain itself (CPU)
# --------------------------------------------------------------------------------------------------------------------
def test_fp64_chain_matches_autograd_through_the_oracle():
    """chain64 equals torch.autograd through oracle.render_oracle.field_mlp in float64, on 300 points."""
    g = torch.Generator().manual_seed(5)
    n = 300
    p = {k: v.double().requires_grad_(True) for k, v in orc.default_init_params(0).items()}
    xyz = torch.randn(n, 3, generator=g, dtype=torch.float64) * 1.5
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    enc, dirs = orc.embed(xyz, orc.N_XYZ_FREQS), orc.embed(d, orc.N_DIR_FREQS)
    g_raw = torch.randn(n, 4, generator=g, dtype=torch.float64) * torch.exp2(torch.randint(-8, 9, (n, 4), generator=g)).double()
    out = orc.field_mlp(p, enc, dirs)
    (out * g_raw).sum().backward()
    with torch.no_grad():                # the activations the chain takes, from a plain float64 forward
        q = {k: v.detach() for k, v in p.items()}
        H, h = [], enc
        for l in range(8):
            if l == 4:
                h = torch.cat([enc, h], 1)
            h = torch.relu(h @ q[LAYERS[l] + ".weight"].t() + q[LAYERS[l] + ".bias"])
            H.append(h)
        feat = h @ q["xyz_encoding_final.weight"].t() + q["xyz_encoding_final.bias"]
        G = shifted_softplus64(torch.cat([feat, dirs], 1) @ q["dir_encoding.0.weight"].t() + q["dir_encoding.0.bias"])
        assert torch.allclose(out.detach(), torch.cat([widened_sigmoid64(G @ q["rgb.0.weight"].t() + q["rgb.0.bias"]),
                                                       h @ q["sigma.weight"].t() + q["sigma.bias"]], 1), rtol=1e-12, atol=1e-12)
        acts = dict(enc=enc, dir=dirs, G=G, H=H, M=[x > 0 for x in H])
        got = chain64(q, g_raw, out.detach(), acts, zero_grads("cpu"))
    for k in NAMES:
        want = p[k].grad
        err = float((got[k] - want).abs().max() / want.abs().max().clamp_min(1e-300))
        assert err <= 1e-10, (k, err)


def test_operand_rounding_helpers():
    """rn16 / rz16 / operand / operand_relu_inference against torch.half and torch.bfloat16 on CPU: round to nearest
    (even), fp16 saturated at +-65504 (satfinite) instead of inf, toward zero where the split modes truncate; the f16
    mode is fp16 and a single product, bf16 a single product; unknown modes raise."""
    g = torch.Generator().manual_seed(3)
    x = torch.cat([torch.randn(4096, generator=g) * torch.exp2(torch.randint(-20, 17, (4096,), generator=g).float()),
                   torch.tensor([0.0, 1.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -8, 65504.0, 65519.0,
                                 65520.0, 7e4, 1e30, 2.0 ** -25, 2.0 ** -24 * 1.5])])
    x = torch.cat([x, -x])
    fp16 = x.clamp(-65504.0, 65504.0).half().float()
    assert torch.isfinite(fp16).all()
    for mode, want in (("f16x3", fp16), ("f16", fp16), ("bf16x3", x.bfloat16().float()), ("bf16", x.bfloat16().float())):
        assert torch.equal(rn16(x, mode), want), mode
        pos = x.abs()
        t = rz16(pos, mode)
        dt = torch.float16 if mode.startswith("f16") else torch.bfloat16
        assert torch.equal(t.to(dt).float(), t) and bool((t <= pos).all()), mode          # representable, not above
        up = (t.to(dt).view(torch.int16) + 1).view(dt).float()                            # the next 16-bit value
        assert bool(((up > pos) | (t == 65504.0)).all()), mode
        hi, lo = operand(x, mode)
        assert torch.equal(hi, want), mode
        if mode in SPLIT_MODES:
            xc = x.clamp(-65504.0, 65504.0) if mode == "f16x3" else x
            assert torch.equal(lo, (xc - hi).to(dt).float()), mode                        # the residual, to nearest
            mid = (x.abs() >= 0.25) & (x.abs() <= 60000.0)     # lo clear of fp16's subnormals, hi of its saturation
            assert bool(((x - hi - lo)[mid].abs() <= 2.0 ** (-21 if mode == "f16x3" else -15) * x[mid].abs()).all()), mode
        else:
            assert lo is None, mode
        hi, lo = operand_relu_inference(x, mode)
        r = torch.relu(x)
        if mode in SPLIT_MODES:
            assert torch.equal(hi, rz16(r, mode)) and bool((lo >= 0).all()), mode
        else:
            assert torch.equal(hi, rn16(r, mode)) and lo is None, mode
    assert operand(x, "fp32")[1] is None and torch.equal(operand(x, "fp32")[0], x)
    assert torch.equal(operand(torch.tensor([7e4]), "f16", nonneg=True)[0], torch.tensor([65504.0]))
    for fn in (rn16, rz16, operand, operand_relu_inference):
        with pytest.raises(ValueError):
            fn(x, "fp16")
    for fn in (rn16, rz16):
        with pytest.raises(ValueError):
            fn(x, "fp32")


# --------------------------------------------------------------------------------------------------------------------
# 2. training forward, layer by layer, in every precision mode
# --------------------------------------------------------------------------------------------------------------------
# Bounds on the normalised error, ~10x above the worst case measured with correct kernels over both weight sets and
# both ray batches (H100 SXM 80 GB, 700 W):
#              enc      h max    h rms    g        sigma    rgb
#   fp32       8.8e-8   9.2e-7   8.8e-8   1.1e-7   4.4e-7   5.6e-8
#   f16x3      8.8e-8   2.0e-6   4.7e-7   1.4e-6   2.5e-7   4.2e-8
#   bf16x3     8.8e-8   2.0e-6   3.7e-7   1.3e-6   2.7e-7   4.4e-8
#   bf16       4.8e-7   6.6e-7   1.0e-7   4.3e-7   2.8e-7   4.3e-8
# (the split modes' h errors exceed an exact fp32 accumulation of the three products, <= 3.5e-7 in a CPU emulation:
# the tensor cores' fp32 accumulation is not round-to-nearest; bf16 rounds both operands exactly like the reference,
# so only the accumulation is left)
FWD_BOUNDS = {
    #            enc      h max    h rms    g        sigma    rgb
    "fp32":   (1.0e-6, 1.0e-5, 1.0e-6, 1.5e-6, 5.0e-6, 6.0e-7),
    "f16x3":  (1.0e-6, 2.0e-5, 5.0e-6, 1.5e-5, 3.0e-6, 5.0e-7),
    "bf16x3": (1.0e-6, 2.0e-5, 4.0e-6, 1.5e-5, 3.0e-6, 5.0e-7),
    "bf16":   (5.0e-6, 7.0e-6, 1.0e-6, 5.0e-6, 3.0e-6, 5.0e-7),
}


def trunk_reference(pd, enc, H, op):
    """float64 (pre-activation, normaliser |W| |x| + |b|) of layers 1..8 and (sigma, normaliser) of the sigma head, each
    layer fed the input it is given: enc (n,63) to layer 1 and the skip, H[l - 1] (h_l) to layer l + 1, H[7] (h8) to
    the head.  op(x, nonneg) -> (hi, lo): the MMA operand formed from x (nonneg: a ReLU output)."""
    eo = op(enc, False)
    layers = []
    for l in range(8):
        Wo = op(pd[LAYERS[l] + ".weight"], False)
        if l == 0:
            xo = eo
        else:
            ho = op(H[l - 1], True)
            if l == 4:
                xo = (torch.cat([eo[0], ho[0]], 1), None if ho[1] is None else torch.cat([eo[1], ho[1]], 1))
            else:
                xo = ho
        b = pd[LAYERS[l] + ".bias"].double()
        layers.append((prod(xo, Wo) + b, absprod(xo, Wo) + b.abs()))
    ws, bs = pd["sigma.weight"].double(), pd["sigma.bias"].double()
    h8 = H[7].double()
    return layers, (h8 @ ws.t() + bs, h8 @ ws.abs().t() + bs.abs())


def add_trunk_errors(st, pd, precision, xyz, enc, H, sigma, b_hmax):
    """One block of points of a training forward: the saved xyz encoding enc (n,64) against float64 (padding column
    zero), the saved h1..h8 H (8,n,256) and sigma (n,1) against float64 from the kernel's own saved inputs, rounded as
    the training epilogue forms its MMA operands.  Accumulates into st['enc'], st['h1'..'h8'], st['sigma']; returns the
    number of ReLU flips (outputs the reference puts clearly below zero that are not exactly 0)."""
    st["enc"].add((enc[:, :63].double() - orc.embed(xyz.double(), orc.N_XYZ_FREQS)).abs())
    assert not bool(enc[:, 63:].any()), "xyz encoding padding"
    layers, (sig, sig_norm) = trunk_reference(pd, enc[:, :63], H, lambda x, nonneg: operand(x, precision, nonneg))
    flips = 0
    for l, (pre, norm) in enumerate(layers):
        h = H[l].double()
        st[f"h{l + 1}"].add((h - torch.relu(pre)).abs() / norm)
        neg = pre < -10.0 * b_hmax * norm                # clearly negative before the ReLU: exactly 0 after it
        flips += int((neg & (h != 0)).sum())
    st["sigma"].add((sigma.double() - sig).abs() / sig_norm)
    return flips


def assert_trunk_bounds(st, flips, bounds):
    b_enc, b_hmax, b_hrms, _, b_sig, _ = bounds
    assert flips == 0, f"{flips} outputs the reference puts clearly below zero are not exactly 0 after the ReLU"
    assert st["enc"].max <= b_enc, st["enc"].max
    for l in range(8):
        s_ = st[f"h{l + 1}"]
        assert s_.max <= b_hmax and s_.rms <= b_hrms, (f"h{l + 1}", s_.max, s_.rms)
    assert st["sigma"].max <= b_sig, st["sigma"].max


def check_forward_layers(precision, weights, scene, n_rays, S, seed, bounds=None):
    torch.cuda.reset_peak_memory_stats()
    p = weights_of(weights)
    pd = to_dev(p)
    _, img = packed(pd, precision)
    rays, z = ray_batch(scene, n_rays, S, seed)
    raw, save = forward_train(img, precision, rays, z)
    P = raw.shape[0]
    assert torch.isfinite(raw).all()
    xyz, dvec = points32(rays, z)
    Wp, bp = folded(pd)
    Wd, bd = pd["dir_encoding.0.weight"], pd["dir_encoding.0.bias"]
    Wpo, Wdo = operand(Wp, precision), operand(Wd[:, 256:], precision)
    st = {k: Stat() for k in ["enc", "dir"] + [f"h{l + 1}" for l in range(8)] + ["g", "sigma", "rgb"]}
    bounds = FWD_BOUNDS[precision] if bounds is None else bounds
    b_enc, b_hmax, b_hrms, b_g, b_sig, b_rgb = bounds
    flips = 0
    for p0 in range(0, P, BLOCK):
        sl = slice(p0, min(P, p0 + BLOCK))
        flips += add_trunk_errors(st, pd, precision, xyz[sl], save["enc"][sl], save["h"][:, sl], raw[sl, 3:4], b_hmax)
        st["dir"].add((save["dir"][sl, :27].double() - orc.embed(dvec[sl].double(), orc.N_DIR_FREQS)).abs())
        assert not bool(save["dir"][sl, 27:].any()), "direction encoding padding"
        h8 = save["h"][7, sl]
        dirv = save["dir"][sl, :27]
        if precision == "fp32":    # the SIMT kernel runs the bottleneck as a layer of its own
            Wf, bf = pd["xyz_encoding_final.weight"].double(), pd["xyz_encoding_final.bias"].double()
            feat = h8.double() @ Wf.t() + bf
            s = feat @ Wd[:, :256].double().t() + dirv.double() @ Wd[:, 256:].double().t() + bd.double()
            norm = (h8.double() @ Wf.abs().t() + bf.abs()) @ Wd[:, :256].double().abs().t() \
                + dirv.double().abs() @ Wd[:, 256:].double().abs().t() + bd.double().abs()
        else:
            h8o, dro = operand(h8, precision, nonneg=True), operand(dirv, precision)
            s = prod(h8o, Wpo) + prod(dro, Wdo) + bp.double()
            norm = absprod(h8o, Wpo) + absprod(dro, Wdo) + bp.double().abs()
        st["g"].add((save["g"][sl].double() - shifted_softplus64(s)).abs() / norm)
        Wr, br = pd["rgb.0.weight"].double(), pd["rgb.0.bias"].double()
        G = save["g"][sl].double()
        st["rgb"].add((raw[sl, :3].double() - widened_sigmoid64(G @ Wr.t() + br)).abs() / (G.abs() @ Wr.abs().t() + br.abs()))
    report(f"forward {precision} {weights} {scene} {n_rays}x{S}", st)
    assert_trunk_bounds(st, flips, bounds)
    assert st["dir"].max <= b_enc, st["dir"].max
    assert st["g"].max <= b_g, st["g"].max
    assert st["rgb"].max <= b_rgb, st["rgb"].max


@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("weights", ["default", "room"])
def test_training_forward_layerwise(precision, weights):
    """4096 lego rays x 128 samples (524 288 points) and a ragged DTU batch (333 x 97 = 32 301 points), every saved
    tensor of snb_field_forward_train against float64 computed from the kernel's own saved inputs."""
    check_forward_layers(precision, weights, "lego", 4096, 128, 21)
    check_forward_layers(precision, weights, "dtu", 333, 97, 22)


# --------------------------------------------------------------------------------------------------------------------
# 3. inference kernel: layers isolated by identity weights
# --------------------------------------------------------------------------------------------------------------------
# (sigma max, rgb max, sigma rms, rgb rms) bounds over l = 2..8 and the four entries.  The max bars are ~10x the worst
# measured (NVIDIA H100 80GB HBM3, 700 W): fp32 2.3e-7 / 4.8e-8, f16x3 8.1e-7 / 4.3e-8, bf16x3 4.4e-6 / 5.4e-8, bf16
# 9.1e-4 / 7.3e-6, f16 1.4e-4 / 1.3e-6 (the single-product modes round every layer's whole output to 8 (bf16) or 11
# (fp16) bits, so a last-bit difference in the fp32 accumulation or in the fast sin / cos of the encoding flips whole
# 16-bit steps).  The rms bars are ~4x the worst measured: fp32 4.1e-8 / 1.2e-8, f16x3 2.7e-7 / 1.1e-8, bf16x3 5.9e-7 /
# 1.2e-8, bf16 1.7e-5 / 1.2e-7, f16 5.8e-6 / 5.1e-8.  An rms over 67 584 points repeats to three digits between runs,
# and it is what sees a rounding-mode slip: f16 operands rounded toward zero instead of to nearest raise the max only
# 3x (4.6e-4 / 4.1e-6), inside a 10x max bar, but the rms 23x (1.3e-4 / 8.3e-7).
INF_BOUNDS = {"fp32": (2.5e-6, 5.0e-7, 1.7e-7, 5.0e-8), "f16x3": (8.0e-6, 5.0e-7, 1.1e-6, 4.5e-8),
              "bf16x3": (4.5e-5, 6.0e-7, 2.4e-6, 5.0e-8), "bf16": (1.0e-2, 7.5e-5, 7.0e-5, 5.0e-7),
              "f16": (1.5e-3, 1.3e-5, 2.3e-5, 2.0e-7)}


def isolating_params(l_dense, seed):
    """Layer 1 and layer l_dense dense (default init), every other trunk layer the identity with zero bias (the skip
    layer: identity on its h4 columns, zero on the encoding columns); bottleneck, direction layer and heads dense."""
    p = orc.default_init_params(seed)
    for l in range(1, 8):
        if l + 1 == l_dense:
            continue
        W = torch.zeros_like(p[LAYERS[l] + ".weight"])
        W[:, -256:] = torch.eye(256)
        p[LAYERS[l] + ".weight"], p[LAYERS[l] + ".bias"] = W, torch.zeros(256)
    return p


def inference_reference(pd, enc32, dir32, precision):
    """float64 sigma and rgb of the inference schedule: every trunk output re-rounded as split_pair_relu forms the next
    operand; the sigma layer's output (h8) as the training epilogue's split_pair."""
    Wo = {l: operand(pd[LAYERS[l] + ".weight"], precision) for l in range(8)}
    eo = operand(enc32, precision)
    xo, norm8 = eo, None
    for l in range(8):
        if l == 4:
            xo = (torch.cat([eo[0], xo[0]], 1), None if xo[1] is None else torch.cat([eo[1], xo[1]], 1))
        b = pd[LAYERS[l] + ".bias"].double()
        pre = prod(xo, Wo[l]) + b
        if l < 7:
            xo = operand_relu_inference(pre.float(), precision)
    h8 = torch.relu(pre)
    ws, bs = pd["sigma.weight"].double(), pd["sigma.bias"].double()
    sigma, sig_norm = h8 @ ws.t() + bs, h8 @ ws.abs().t() + bs.abs()
    Wd, bd = pd["dir_encoding.0.weight"], pd["dir_encoding.0.bias"]
    if precision == "fp32":
        Wf, bf = pd["xyz_encoding_final.weight"].double(), pd["xyz_encoding_final.bias"].double()
        s = (h8 @ Wf.t() + bf) @ Wd[:, :256].double().t() + dir32.double() @ Wd[:, 256:].double().t() + bd.double()
    else:
        Wp, bp = folded(pd)
        s = prod(operand(h8.float(), precision, nonneg=True), operand(Wp, precision)) \
            + prod(operand(dir32, precision), operand(Wd[:, 256:], precision)) + bp.double()
    G = shifted_softplus64(s)
    Wr, br = pd["rgb.0.weight"].double(), pd["rgb.0.bias"].double()
    rgb, rgb_norm = widened_sigmoid64(G @ Wr.t() + br), G.abs() @ Wr.abs().t() + br.abs()
    return sigma, sig_norm, rgb, rgb_norm


@pytest.mark.gpu
@pytest.mark.parametrize("precision", MODES + ["f16"])
def test_inference_layers_isolated_by_identity_weights(precision):
    """snb_field_forward and snb_mlp_forward (normal and sigma_only) on 2048 lego rays x 33 samples, with parameter sets
    in which only layer 1 and layer l (l = 2..8) are dense: sigma and rgb against float64 per point, max and rms."""
    from sinnerf_b200 import _lib
    lib = _lib.load()
    prec = _lib.precision_id(precision)
    rays, z = ray_batch("lego", 2048, 33, 31)
    n, S = z.shape
    P = n * S
    xyz, dvec = points32(rays, z)
    enc32 = orc.embed(xyz.double(), orc.N_XYZ_FREQS).float()
    dir32 = orc.embed(dvec.double(), orc.N_DIR_FREQS).float()
    x = torch.cat([enc32, dir32], 1).contiguous()
    st_ptr = _lib.stream_ptr(torch.device(DEV))
    b_sig, b_rgb, r_sig, r_rgb = INF_BOUNDS[precision]
    worst, rms = {}, {}
    for l_dense in range(2, 9):
        pd = to_dev(isolating_params(l_dense, seed=l_dense))
        _, img = packed(pd, precision)
        sigma, sig_norm, rgb, rgb_norm = inference_reference(pd, enc32, dir32, precision)
        for entry in ("field", "mlp"):
            for sigma_only in (False, True):
                out = torch.full((P, 1 if sigma_only else 4), float("nan"), device=DEV)
                if entry == "field":
                    rc = lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, int(sigma_only),
                                               _lib.ptr(out), st_ptr)
                else:
                    rc = lib.snb_mlp_forward(_lib.ptr(img), prec, _lib.ptr(x), x.shape[1], P, int(sigma_only), _lib.ptr(out),
                                             st_ptr)
                _lib.check(rc, entry)
                torch.cuda.synchronize()
                errs = [("sigma", (out[:, -1:].double() - sigma).abs() / sig_norm)]
                if not sigma_only:
                    errs.append(("rgb", (out[:, :3].double() - rgb).abs() / rgb_norm))
                for what, e in errs:
                    worst[(l_dense, entry, sigma_only, what)] = float(e.max())
                    rms[(l_dense, entry, sigma_only, what)] = float(e.pow(2).mean().sqrt())
    print(f"\ninference {precision} (bars {b_sig:.1e} / {b_rgb:.1e}), max: " +
          ", ".join(f"{k}: {v:.2e}" for k, v in worst.items()))
    print(f"inference {precision} (bars {r_sig:.1e} / {r_rgb:.1e}), rms: " + ", ".join(f"{k}: {v:.2e}" for k, v in rms.items()))
    for k, v in worst.items():
        assert v <= (b_sig if k[3] == "sigma" else b_rgb), (k, "max", v)
    for k, v in rms.items():
        assert v <= (r_sig if k[3] == "sigma" else r_rgb), (k, "rms", v)


# --------------------------------------------------------------------------------------------------------------------
# 4. backward: sparse probes and dense gradients at training size, scale bookkeeping
# --------------------------------------------------------------------------------------------------------------------
P_TRAIN = 16384 * 128          # the fine pass of a training step (4 x 4096 rays, 64 + 64 samples)
P_RAGGED = 16384 * 128 - 4097  # not a multiple of 32 or of 128


def slice_edges(n_tiles, tile, blocks, sm):
    """First and last point of every split-P slice of a wgrad launch with `blocks` CTAs per slice (launch_wgrad16 /
    launch_wgrad_tc: ctas = ceil(sm / blocks), tiles_per_cta = ceil(n_tiles / ctas))."""
    ctas = min((sm + blocks - 1) // blocks, n_tiles)
    tpc = (n_tiles + ctas - 1) // ctas
    ctas = (n_tiles + tpc - 1) // tpc
    pts = []
    for x in range(ctas):
        pts += [x * tpc * tile, min((x + 1) * tpc, n_tiles) * tile - 1]
    return pts


def probe_points(P, n_tiles, sm, seed):
    """~2k points where a kernel that mishandles a slice, tile or tail shows up at O(1)."""
    g = torch.Generator().manual_seed(seed)
    pts = []
    for blocks in (1, 2):
        pts += slice_edges(n_tiles, 32, blocks, sm)
    t = torch.randint(1, (P - 1) // 128, (384,), generator=g)
    pts += (t * 128 - 1).tolist() + (t * 128).tolist()
    pts += [P - 1, P - 2, P - 33, (P - 1) // 128 * 128, (P - 1) // 32 * 32]
    pts += torch.randint(0, P, (2048 - len(set(pts)),), generator=g).tolist()
    pts = sorted({q for q in pts if 0 <= q < P})
    return torch.tensor(pts, dtype=torch.int64)


def probe_g_raw(P, idx, seed):
    g = torch.Generator().manual_seed(seed)
    vals = torch.randn(idx.shape[0], 4, generator=g).sign() * torch.exp2(torch.rand(idx.shape[0], 4, generator=g) * 16 - 8)
    g_raw = torch.zeros(P, 4, device=DEV)
    g_raw[idx.to(DEV)] = vals.to(DEV)
    return g_raw


def grad_buffers(pd):
    return {k: torch.zeros_like(v) for k, v in pd.items()}


def run_backward16(pd, g_raw, raw, act16, P, grads=None, ws=None):
    import ctypes as C
    from sinnerf_b200 import _lib
    lib = _lib.load()
    grads = grad_buffers(pd) if grads is None else grads
    ws = torch.empty(lib.snb_bwd16_workspace_bytes(P), device=DEV, dtype=torch.uint8) if ws is None else ws
    parr = (C.c_void_p * 24)(*[pd[k].data_ptr() for k in NAMES])
    garr = (C.c_void_p * 24)(*[grads[k].data_ptr() for k in NAMES])
    _lib.check(lib.snb_field_backward16(parr, garr, 1, _lib.ptr(g_raw), _lib.ptr(raw), _lib.ptr(act16), P, _lib.ptr(ws),
                                        None, _lib.stream_ptr(torch.device(DEV))), "snb_field_backward16")
    torch.cuda.synchronize()
    return grads, ws


def run_backward32(pd, g_raw, raw, save, P):
    import ctypes as C
    from sinnerf_b200 import _lib
    lib = _lib.load()
    grads = grad_buffers(pd)
    ws = [torch.empty(P, 256, device=DEV), torch.empty(P, 256, device=DEV), torch.empty(P, 128, device=DEV),
          torch.empty(_lib.BWD_WS_FLOATS, device=DEV), torch.empty(P, 8, device=DEV, dtype=torch.int32)]
    parr = (C.c_void_p * 24)(*[pd[k].data_ptr() for k in NAMES])
    garr = (C.c_void_p * 24)(*[grads[k].data_ptr() for k in NAMES])
    _lib.check(lib.snb_field_backward(parr, garr, 1, _lib.ptr(g_raw), _lib.ptr(raw), _lib.ptr(save["enc"]),
                                      _lib.ptr(save["dir"]), _lib.ptr(save["h"]), _lib.ptr(save["g"]), P,
                                      *[_lib.ptr(w) for w in ws], _lib.stream_ptr(torch.device(DEV))), "snb_field_backward")
    torch.cuda.synchronize()
    return grads


def forward_train16(img, rays, z):
    from sinnerf_b200 import _lib
    lib = _lib.load()
    n, S = z.shape
    P = n * S
    raw = torch.empty(P, 4, device=DEV)
    act16 = torch.empty(lib.snb_act16_bytes(P), device=DEV, dtype=torch.uint8)
    _lib.check(lib.snb_field_forward_train16(_lib.ptr(img), _lib.precision_id("f16x3"), _lib.ptr(rays), _lib.ptr(z), n, S,
                                             _lib.ptr(raw), _lib.ptr(act16), _lib.stream_ptr(torch.device(DEV))),
               "snb_field_forward_train16")
    torch.cuda.synchronize()
    return raw, act16


def training_batch(P, seed):
    """P points on lego rays, 128 samples each.  A ragged P is passed as P one-sample rays (an (n, S) grid cannot
    hold it), which leaves the forward's point order unchanged."""
    n = (P + 127) // 128
    rays, z = ray_batch("lego", n, 128, seed)
    if n * 128 != P:
        pts_rays = rays.repeat_interleave(128, 0)[:P].contiguous()
        return pts_rays, z.reshape(-1, 1)[:P].contiguous()
    return rays, z


def grad_errors(got, want):
    return {k: (rel_l2(got[k], want[k]), float((got[k].double() - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-300)))
            for k in NAMES}


def print_errors(title, errs):
    print(f"\n{title}")
    for k, (r, m) in errs.items():
        print(f"  {k:>28}: rel-L2 {r:.3e}  max-rel {m:.3e}")
    print(f"  peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def bwd_bound(arm, name):
    """Per-tensor bar (rel-L2 and max-rel) against the float64 chain.  Worst measured (H100 SXM), sparse and dense:
    16-bit arm, trunk / bottleneck / direction layer 2.0e-4 .. 7.4e-4 (two 11-bit roundings per weight gradient: its
    layer's gradient and input); sigma / rgb head weights 9.8e-5 / 3.3e-5 (dense; 1.6e-6 / 6.7e-7 sparse: fp32
    accumulation over ~31 800 points per register accumulator); head biases <= 1.5e-6.  fp32 arm: every tensor
    <= 3.5e-5.  The 16-bit trunk bar is 4x its worst case (these are norms over >= 32 k elements and move by < 30 %
    between batches), the others 10x; a mishandled slice, tile or K step moves a tensor by 1e-2 .. 1."""
    if arm == "32":
        return 3.5e-4
    if name in ("sigma.weight", "rgb.0.weight"):
        return 1.0e-3
    if name in ("sigma.bias", "rgb.0.bias"):
        return 2.0e-5
    return 3.0e-3


@pytest.mark.gpu
@pytest.mark.parametrize("P", [P_TRAIN, P_RAGGED])
def test_backward16_sparse_probes_at_training_size(P):
    """snb_field_backward16 with g_raw zero except at ~2k probe points (the edges of every wgrad slice, both sides of
    sampled 128-point tile boundaries, the ragged tail), magnitudes spanning 2^+-8: float64 chain on those rows."""
    torch.cuda.reset_peak_memory_stats()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    pd = to_dev(orc.default_init_params(1))
    _, img = packed(pd, "f16x3")
    rays, z = training_batch(P, 41)
    raw, act16 = forward_train16(img, rays, z)
    idx = probe_points(P, a16_pad(P) // 32, sm, 5)
    g_raw = probe_g_raw(P, idx, 6)
    got, _ = run_backward16(pd, g_raw, raw, act16, P)
    idx_d = idx.to(DEV)
    want = chain64(to_dev(orc.default_init_params(1), torch.float64), g_raw[idx_d], raw[idx_d],
                   act16_rows(act16_sections(act16, P), idx_d), zero_grads(DEV))
    errs = grad_errors(got, want)
    print_errors(f"backward16 sparse P={P} ({idx.shape[0]} probes)", errs)
    for k, (r, m) in errs.items():
        bound = bwd_bound("16", k)
        assert r <= bound and m <= bound, (k, r, m, bound)


@pytest.mark.gpu
def test_backward16_dense_at_training_size():
    """snb_field_backward16 on 2 097 152 points with a dense seeded g_raw: the full float64 chain over the decoded
    fp16 activations, blocked over points; per-tensor rel-L2 and max-rel."""
    torch.cuda.reset_peak_memory_stats()
    P = P_TRAIN
    pd = to_dev(orc.default_init_params(1))
    p64 = to_dev(orc.default_init_params(1), torch.float64)
    _, img = packed(pd, "f16x3")
    rays, z = training_batch(P, 43)
    raw, act16 = forward_train16(img, rays, z)
    g = torch.Generator(device=DEV).manual_seed(9)
    g_raw = torch.randn(P, 4, device=DEV, generator=g)
    got, _ = run_backward16(pd, g_raw, raw, act16, P)
    secs = act16_sections(act16, P)
    want = zero_grads(DEV)
    for p0 in range(0, P, BLOCK):
        idx = torch.arange(p0, min(P, p0 + BLOCK), device=DEV)
        chain64(p64, g_raw[idx], raw[idx], act16_rows(secs, idx), want)
    errs = grad_errors(got, want)
    print_errors(f"backward16 dense P={P}", errs)
    for k, (r, m) in errs.items():
        bound = bwd_bound("16", k)
        assert r <= bound and m <= bound, (k, r, m, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_backward_fp32_storage(dense):
    """snb_field_backward (fp32 saves, 8.9 KB per point) on 524 288 points and on a ragged 524 288 - 77: sparse probes
    and a dense g_raw against the float64 chain over the saved fp32 activations."""
    torch.cuda.reset_peak_memory_stats()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    pd = to_dev(orc.default_init_params(1))
    p64 = to_dev(orc.default_init_params(1), torch.float64)
    _, img = packed(pd, "f16x3")
    for P in ((4096 * 128,) if dense else (4096 * 128, 4096 * 128 - 77)):
        rays, z = training_batch(P, 47)
        raw, save = forward_train(img, "f16x3", rays, z)
        if dense:
            g = torch.Generator(device=DEV).manual_seed(10)
            g_raw = torch.randn(P, 4, device=DEV, generator=g)
            blocks = [torch.arange(p0, min(P, p0 + BLOCK), device=DEV) for p0 in range(0, P, BLOCK)]
        else:
            idx = probe_points(P, (P + 31) // 32, sm, 7)
            g_raw = probe_g_raw(P, idx, 8)
            blocks = [idx.to(DEV)]
        got = run_backward32(pd, g_raw, raw, save, P)
        want = zero_grads(DEV)
        for idx in blocks:
            chain64(p64, g_raw[idx], raw[idx], fp32_rows(save, idx), want)
        errs = grad_errors(got, want)
        print_errors(f"backward fp32 storage {'dense' if dense else 'sparse'} P={P}", errs)
        del save
        for k, (r, m) in errs.items():
            bound = bwd_bound("32", k)
            assert r <= bound and m <= bound, (k, r, m, bound)


def bwd16_layout(P):
    """Byte offsets of the backward workspace (make_bwd16_layout in csrc/act16.cuh)."""
    pp = a16_pad(P)
    off, L = 0, {}
    for name, F in (("ds", 128), ("hg", 8), ("dya", 256), ("dyb", 256), ("ds_lo", 128), ("dya_lo", 256), ("dyb_lo", 256)):
        L[name] = off
        off += pp * F * 2
    L["fold"] = off
    off += (2 * 128 * 256 + 128) * 4
    L["state"] = off
    return L


ST_AMAX_G, ST_AMAX_DS, ST_AMAX_H0, ST_SCALE_HG, ST_SCALE_DS, ST_SCALE_H0 = 0, 1, 2, 10, 11, 12


@pytest.mark.gpu
def test_backward16_gradient_scale_bookkeeping():
    """g_raw 2^k (k = -64..64) gives 2^k times the k = 0 gradients within the run-to-run noise of the atomics; the
    workspace's fp16 gradient planes are bit-identical across k and every state scale is exactly 2^-k times its k = 0
    value.  pow2_scale clamps exponents to +-100: with default-init weights and |g_raw| ~ 1 the scales sit at 2^11 ..
    2^19 (measured), so the exact range ends below k = -81, where the largest scale would pass 2^100, and above k = 111;
    k = -64..64 stays inside.
    An all-zero g_raw gives exactly zero gradients."""
    P = 300 * 128 + 37
    pd = to_dev(orc.default_init_params(1))
    _, img = packed(pd, "f16x3")
    rays, z = training_batch(P, 51)
    raw, act16 = forward_train16(img, rays, z)
    g = torch.Generator(device=DEV).manual_seed(12)
    g_raw = torch.randn(P, 4, device=DEV, generator=g)
    L = bwd16_layout(P)
    base, ws0 = run_backward16(pd, g_raw, raw, act16, P)
    again, _ = run_backward16(pd, g_raw, raw, act16, P)
    noise = max(rel_l2(again[k], base[k]) for k in NAMES)
    planes0 = ws0[:L["fold"]].clone()
    state0 = ws0[L["state"]:L["state"] + 64 * 4].view(torch.float32).clone()
    e0 = torch.log2(state0[ST_SCALE_HG:ST_SCALE_H0 + 8])
    print(f"\nscale exponents at k = 0: {e0.tolist()}; atomics noise (rel-L2) {noise:.2e}")
    for k in (-64, -40, -8, 8, 40, 64):
        assert bool(((e0 - k).abs() <= 100).all()), f"k={k} reaches the +-100 exponent clamp"
        got, ws = run_backward16(pd, g_raw * 2.0 ** k, raw, act16, P)
        assert torch.equal(ws[:L["fold"]], planes0), f"k={k}: the fp16 gradient planes differ"
        state = ws[L["state"]:L["state"] + 64 * 4].view(torch.float32)
        assert torch.equal(state[ST_SCALE_HG:ST_SCALE_H0 + 8], state0[ST_SCALE_HG:ST_SCALE_H0 + 8] * 2.0 ** -k), k
        assert torch.equal(state[ST_AMAX_DS:ST_AMAX_H0 + 8], state0[ST_AMAX_DS:ST_AMAX_H0 + 8]), k
        assert float(state[ST_AMAX_G]) == float(state0[ST_AMAX_G]) * 2.0 ** k, k
        for n in NAMES:
            r = rel_l2(got[n].double() * 2.0 ** -k, base[n])
            assert r <= max(4 * noise, 1e-6), (k, n, r, noise)
    zero, _ = run_backward16(pd, torch.zeros_like(g_raw), raw, act16, P)
    for n in NAMES:
        assert not bool(zero[n].any()), n
