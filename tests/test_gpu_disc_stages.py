"""The discriminator kernels (csrc/disc.cu) stage by stage against float64.

tests/test_gpu_discriminator.py holds the output and the gradients to the float64 oracle end to end, at bars loose
enough for a LeakyReLU kink flipped by rounding; a wrong term in one backward stage, one dropped K tail or one
misplaced tile fits under them.  Here the kernels run through the C ABI with a workspace this file allocates (filled
with NaN first) and DiffAugment draws it chooses, and every stage the workspace brackets is recomputed in float64 from
the kernel's OWN inputs (tests/disc_emulation.py), with the GEMM operands rounded the way the kernel rounds them, so
errors do not compound and no kink can flip.  A backward call with one weight gradient and no input gradient stops
after that layer, so calling it once per layer leaves every layer's scaled output gradient, dcol and fold behind.

Bit for bit: the power-iteration words (max |W|, 1 / sigma, alpha, the scaled weight copy, u and v copied to the
module), the DiffAugment words and cutout box, the im2col gather, the upstream scale, the rescale after each fold, every
partial backward's dW against the full one, repeated backwards, the saved state after all backwards, four input
layouts, n = 8 against eight n = 1 calls, scaling W by 2^j and scaling the upstream gradient by 2^j (down to 2^-149).
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from sinnerf_b200 import _lib
from sinnerf_b200.discriminator import Discriminator, output_sizes
from tests import disc_emulation as de

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NAN = float("nan")
MODE_LIST = list(de.MODES)
# (imsize, h, w, n, augmented, training, input layout): every branch at its recipe size and its smallest, odd sizes,
# n = 1, 3, 8, both modes, augmentation off and on (the cutout at each clamped corner and inside, saturation factor
# 0 / 1 / 2, contrast 0.5 / 1.5 spread over the images), four input layouts
CASES = [(128, 128, 128, 1, True, True, "nchw"), (128, 128, 128, 3, False, False, "rays"),
         (64, 64, 64, 8, True, True, "cl_pad"), (64, 67, 75, 3, True, False, "nchw"),
         (32, 32, 32, 1, False, True, "rays"), (32, 33, 47, 8, True, True, "nchw"),
         (-1, 63, 84, 3, True, True, "rays"), (-1, 56, 70, 8, False, True, "cl_pad"),
         (-1, 16, 16, 1, True, False, "nchw")]
CORNERS = ("top-left", "top-right", "bottom-left", "bottom-right", "inside")


def case_id(c):
    return f"{c[0]}-{c[1]}x{c[2]}-n{c[3]}-{'aug' if c[4] else 'noaug'}-{'train' if c[5] else 'eval'}-{c[6]}"


# --------------------------------------------------------------------------------------------------------------------
# driving the C ABI
# --------------------------------------------------------------------------------------------------------------------
def state(imsize, seed=0):
    """(weight_orig, weight_u, weight_v) of the module's seeded initialisation, on the GPU"""
    torch.manual_seed(seed)
    D = Discriminator(False, "color,cutout", imsize=imsize)
    return ([m.weight_orig.detach().to(DEV).contiguous() for m in D.convs()],
            [m.weight_u.to(DEV).clone() for m in D.convs()], [m.weight_v.to(DEV).clone() for m in D.convs()])


def placed(x, layout):
    """(n, 3, h, w) values -> a GPU view holding them: contiguous NCHW, the '(b p q) c -> b c p q' view of a ray-major
    tensor, or channels-last inside a padded buffer (odd strides, 4-byte offset); 'expand': image 0 with batch
    stride 0"""
    n, c, h, w = x.shape
    if layout == "nchw":
        return x.to(DEV).contiguous()
    if layout == "rays":
        return x.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous().to(DEV).view(n, h, w, c).permute(0, 3, 1, 2)
    if layout == "expand":
        return x[:1].to(DEV).expand(n, c, h, w)
    assert layout == "cl_pad"
    v = torch.zeros(n, h, w + 1, 5, device=DEV)[:, :, :w, 1:4].permute(0, 3, 1, 2)
    v.copy_(x.to(DEV))
    return v


def padded_grad(n, h, w):
    """(buffer, view): a NaN-filled buffer and an (n, 3, h, w) view inside it with odd strides and an offset"""
    buf = torch.full((n, h + 1, w + 2, 7), NAN, device=DEV)
    return buf, buf[:, 1:, 1:w + 1, 2:5].permute(0, 3, 1, 2)


def draws(n, h, w, start):
    """DiffAugment draws for n images, image i taking combination start + i of: the cutout centred on each corner (its
    box clamped there) or inside, saturation draw 0 / 0.5 / 1 (factor 0 / 1 / 2), contrast draw 0 / 1 (0.5 / 1.5)"""
    j = torch.arange(start, start + n)
    corner = {"top-left": (0, 0), "top-right": (0, w - 1), "bottom-left": (h - 1, 0), "bottom-right": (h - 1, w - 1),
              "inside": (h // 2, w // 3)}
    oy, ox = (torch.tensor([corner[CORNERS[int(k) % 5]][a] for k in j]) for a in (0, 1))
    rb = 0.15 + 0.1 * (j % 7).float()
    rs = torch.tensor([0.0, 0.5, 1.0])[j % 3]
    rc = torch.tensor([0.0, 1.0])[j % 2]
    return tuple(t.to(DEV) for t in (rb.float(), rs, rc, oy.long(), ox.long()))


def c_ptrs(ts):
    return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def forward(imsize, mode, training, W, U, V, x, aug):
    """(out, workspace) of snb_disc_forward on a NaN-filled save = 1 workspace; U / V are advanced in training mode"""
    lib = _lib.load()
    n, _, h, w = x.shape
    ws = torch.full((lib.snb_disc_workspace_bytes(imsize, n, h, w, 1) // 4,), NAN, device=DEV)
    out = torch.full((n, 1, *output_sizes(imsize, h, w)[-1]), NAN, device=DEV)
    a = None if aug is None else C.byref(_lib.SnbDiscAug(*[t.data_ptr() for t in aug]))
    _lib.check(lib.snb_disc_forward(imsize, de.MODES[mode], int(training), c_ptrs(W), c_ptrs(U), c_ptrs(V),
                                    _lib.ptr(x), (C.c_int64 * 4)(*x.stride()), n, h, w, a, _lib.ptr(out),
                                    _lib.ptr(ws), _lib.stream_ptr(DEV)), "snb_disc_forward")
    return out, ws


def backward(imsize, mode, W, shape, d_out, ws, want, d_input=None):
    """[dW or None] of snb_disc_backward for the layers in `want` (NaN-filled first); d_input: a view to write"""
    lib = _lib.load()
    n, _, h, w = shape
    dws = [torch.full_like(t, NAN) if i in want else None for i, t in enumerate(W)]
    strides = None if d_input is None else (C.c_int64 * 4)(*d_input.stride())
    _lib.check(lib.snb_disc_backward(imsize, de.MODES[mode], c_ptrs(W), n, h, w, _lib.ptr(d_out.contiguous()),
                                     _lib.ptr(d_input), strides, c_ptrs(dws), _lib.ptr(ws), _lib.stream_ptr(DEV)),
               "snb_disc_backward")
    return dws


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a.float()), bits(b.float()))


# --------------------------------------------------------------------------------------------------------------------
# the stage record
# --------------------------------------------------------------------------------------------------------------------
class Stages:
    """per stage: the largest worst and rms over the stage's instances (per layer, per image set), against the
    emulation and, for the GEMMs, against the exact product; and the bit-for-bit checks that failed.  Everything is
    printed before anything is asserted."""

    def __init__(self, mode, what):
        self.mode, self.what, self.e, self.bad = mode, what, {}, []

    def add(self, stage, y, ref, scale, exact=None):
        if torch.isnan(y).any():
            self.bad.append((stage, "NaN"))
            return
        new = de.stats(de.err(y, ref, scale)) + (de.stats(de.err(y, exact, scale)) if exact is not None else (0.0, 0.0))
        old = self.e.get(stage, (0.0,) * 4)
        self.e[stage] = tuple(max(a, b) for a, b in zip(old, new))

    def exact(self, what, ok):
        if not ok:
            self.bad.append((what, "bits"))

    def check(self):
        for stage, (w, r, wx, rx) in sorted(self.e.items()):
            bw, br = de.BARS[self.mode][stage]
            ex = f" | vs exact product: worst {wx:.2e} rms {rx:.2e}" if wx else ""
            print(f"disc stages {self.what} {self.mode:5s} {stage:8s}: worst {w:.2e} rms {r:.2e} "
                  f"(bars {bw:.0e} {br:.0e})" + ex)
            if not (w <= bw and r <= br):
                self.bad.append((stage, w, r))
        assert not self.bad, self.bad


def mask_matches_gather(st, y, col, mask, what):
    """the fold's LeakyReLU mask equals the sign the forward gather gave the same element: every col entry a pixel
    feeds is > 0 where the mask is set and <= 0 elsewhere"""
    n = y["n"]

    def fold(c):
        c = c.view(n, y["P"], y["K"]).transpose(1, 2)
        return F.fold(c, (y["hin"], y["win"]), 4, padding=y["pad"], stride=y["stride"]).reshape(n, y["cin"], -1)
    pos, cover = fold((col > 0).double()), fold(torch.ones_like(col, dtype=torch.float64))
    m = mask.transpose(0, 1)
    st.exact(what, bool(((pos == cover) == m)[cover > 0].all()) and bool((pos[~m] == 0).all()))


# --------------------------------------------------------------------------------------------------------------------
# stage by stage
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODE_LIST)
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_stages(case, mode):
    imsize, h, w, n, aug_on, training, layout = case
    W, U, V = state(imsize, seed=h + n)
    U0, V0 = [u.clone() for u in U], [v.clone() for v in V]
    g = torch.Generator().manual_seed(1000 * h + w + n)
    xc = torch.rand(n, 3, h, w, generator=g)
    x = placed(xc, layout)
    aug = draws(n, h, w, start=h + n) if aug_on else None
    out, wsp = forward(imsize, mode, training, W, U, V, x, aug)
    torch.cuda.synchronize()
    b = de.workspace_views(wsp, imsize, n, h, w)
    layers = de.net(imsize, n, h, w)
    L = len(layers)
    st = Stages(mode, case_id(case))
    fwd_state = {k: v.clone() for k, v in b.items() if not k.startswith(("part", "gexp", "dot", "dy", "dcol", "dx"))}

    # ---- spectral norm
    for i, y in enumerate(layers):
        Wm = W[i].reshape(y["cout"], -1)
        r = de.sn_ref(Wm, U0[i], V0[i], training, b[f"t{i}"], b[f"s{i}"], b[f"u{i}"])
        for k in (("t", "v", "s", "u") if training else ("s",)):
            st.add(k, b[f"{k}{i}"], *r[k])
        st.add("sigma", b["sigma"][i:i + 1], *r["sigma"])
        st.exact(f"rmax{i}", same_bits(b[f"rmax{i}"], Wm.abs().amax(1)))
        inv, alpha, wscale = de.sn_words(b["sigma"][i], b[f"rmax{i}"])
        st.exact(f"inv_sigma/alpha/wscale{i}", same_bits(b["inv_sigma"][i], inv) and same_bits(b["alpha"][i], alpha)
                 and same_bits(b["wscale"][i], wscale))
        st.exact(f"ws{i}", same_bits(b[f"ws{i}"], Wm * wscale))
        if training:
            st.exact(f"u/v{i} to the module", same_bits(U[i], b[f"u{i}"]) and same_bits(V[i], b[f"v{i}"]))
        else:
            st.exact(f"u/v{i} eval", same_bits(U[i], U0[i]) and same_bits(V[i], V0[i]) and
                     same_bits(b[f"u{i}"], U0[i]) and same_bits(b[f"v{i}"], V0[i]) and bool(b[f"t{i}"].isnan().all()))

    # ---- DiffAugment words and layer 0's gather
    xd = xc.to(DEV)
    col0 = b["col0"]
    if aug is None:
        st.exact("aug off", bool((b["aug"][:, 0] == 0).all()))
        st.exact("gather0 copy", same_bits(col0, de.unfold(xd, layers[0])))
    else:
        f, box = de.aug_words(aug, h, w)
        st.exact("aug words", same_bits(b["aug"][:, :4], f) and torch.equal(b["aug"][:, 5:9], box.float()))
        st.add("aug_mean", b["aug"][:, 4], *de.aug_mean_ref(xd, b["aug"][:, 1], b["aug"][:, 2]))
        ref, mag, cut = de.gather0_ref(layers, xd, b["aug"][:, :4], b["aug"][:, 4], box)
        st.add("gather0", col0, ref, mag * 2.0 ** -24)
        st.exact("cutout zeros", bool((col0[cut] == 0).all()))
    st.exact("gather0 padding", bool((bits(col0)[de.pad_mask(layers[0], DEV)] == 0).all()))

    # ---- per layer: gather (layers >= 1), GEMM, InstanceNorm statistics
    for i, y in enumerate(layers):
        if i > 0:
            want = de.gather_ref(layers, i, b[f"y{i - 1}"], b.get(f"mean{i - 1}"), b.get(f"rstd{i - 1}"))
            st.exact(f"gather{i}", same_bits(b[f"col{i}"], want))
            st.exact(f"gather{i} padding", bool((bits(b[f"col{i}"])[de.pad_mask(y, DEV)] == 0).all()))
        emu, exact, sc = de.gemm_fwd_ref(b[f"ws{i}"], b[f"col{i}"], b["alpha"][i], de.col_scale(layers, i), mode)
        got = b[f"y{i}"].reshape(y["cout"], -1) if y["act"] else out.reshape(1, -1)
        st.add("fwd", got, emu, sc, exact)
        if y["in_norm"]:
            m, r, msc, rsc = de.in_stats_ref(b[f"y{i}"])
            st.add("in_mean", b[f"mean{i}"], m, msc)
            st.add("in_rstd", b[f"rstd{i}"], r, rsc)

    # ---- backward, one weight gradient per call: each call stops after its layer
    d_out = torch.randn(out.shape, generator=g).to(DEV)
    dy_top, k0 = de.scaled_upstream(d_out.reshape(1, -1))
    partial = []
    for k in range(L - 1, -1, -1):
        (dWk,) = [t for t in backward(imsize, mode, W, x.shape, d_out, wsp, {k}) if t is not None]
        torch.cuda.synchronize()
        partial.append((k, dWk))
        gexp = [int(e) for e in b["gexp"][:L]]
        y = layers[k]
        dy = b[de.dy_buffer(L, k)][:y["cout"] * n * y["P"]].view(y["cout"], -1)
        if k == L - 1:
            st.exact("upstream scale", same_bits(dy, dy_top) and gexp[L - 1] == -k0)
        else:   # layer k + 1's dgrad, fold, and the rescale that made layer k's dy
            z = layers[k + 1]
            dyz = b[de.dy_buffer(L, k + 1)][:z["cout"] * n * z["P"]].view(z["cout"], -1)
            dcol = b["dcol"][:n * z["P"] * z["K"]].view(n * z["P"], z["K"])
            emu, exact, sc = de.dgrad_ref(dyz, b[f"ws{k + 1}"], b["alpha"][k + 1], mode)
            st.add("dgrad", dcol, emu, sc, exact)
            kk = gexp[k + 1] - gexp[k]
            unscaled = dy.double() * 2.0 ** -kk
            st.exact(f"rescale{k}", de.pow2_exponent(unscaled.abs().max()) == kk and
                     same_bits(de.ldexp32(unscaled, kk), dy))
            ref, sc, mask = de.fold_ref(layers, k + 1, dcol, b[f"y{k}"], b.get(f"mean{k}"), b.get(f"rstd{k}"))
            st.add("fold", unscaled.view_as(ref), ref, sc)
            mask_matches_gather(st, z, b[f"col{k + 1}"], mask, f"mask{k}")
        raw, _, rsc = de.wgrad_ref(dy, b[f"col{k}"], de.col_scale(layers, k), mode)
        Wm = W[k].reshape(y["cout"], -1)
        st.add("part", b[f"part{k}"], *de.part_ref(raw, rsc, Wm))
        ref, sc = de.sn_fix_ref(raw, rsc, b[f"part{k}"], b["inv_sigma"][k], b[f"u{k}"], b[f"v{k}"], gexp[k])
        st.add("wgrad", dWk.reshape(y["cout"], -1), ref, sc)

    # ---- the input gradient alone: layer 0's dgrad and fold, then the DiffAugment backward
    buf, dxv = padded_grad(n, h, w)
    backward(imsize, mode, W, x.shape, d_out, wsp, set(), d_input=dxv)
    torch.cuda.synchronize()
    gexp = [int(e) for e in b["gexp"][:L]]
    y = layers[0]
    dy = b[de.dy_buffer(L, 0)][:y["cout"] * n * y["P"]].view(y["cout"], -1)
    dcol = b["dcol"][:n * y["P"] * y["K"]].view(n * y["P"], y["K"])
    emu, exact, sc = de.dgrad_ref(dy, b["ws0"], b["alpha"][0], mode)
    st.add("dgrad", dcol, emu, sc, exact)
    ref, sc, _ = de.fold_ref(layers, 0, dcol, None, None, None)
    st.add("fold", b["dx"], ref, sc)
    if aug is None:
        st.exact("input gradient", same_bits(dxv, de.ldexp32(b["dx"].transpose(0, 1).reshape(n, 3, h, w), gexp[0])))
    else:
        st.add("aug_bwd", dxv, *de.aug_bwd_ref(b["dx"], b["aug"][:, :4], de.aug_words(aug, h, w)[1], gexp[0], h, w))
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:, 1:, 1:w + 1, 2:5] = False
    st.exact("input gradient padding untouched", bool(buf[outside].isnan().all()))

    # ---- the full backward: the same dW as each partial call, the same input gradient, twice
    for rep in range(2):
        full_dx = torch.full((n, 3, h, w), NAN, device=DEV)
        full = backward(imsize, mode, W, x.shape, d_out, wsp, set(range(L)), d_input=full_dx)
        torch.cuda.synchronize()
        st.exact(f"full backward {rep}: partial dW", all(same_bits(full[k], dWk) for k, dWk in partial))
        st.exact(f"full backward {rep}: input gradient", same_bits(full_dx, dxv))
    st.exact("saved forward state", all(same_bits(b[k], v) if v.dtype == torch.float32 else torch.equal(b[k], v)
                                        for k, v in fwd_state.items()))
    st.check()


# --------------------------------------------------------------------------------------------------------------------
# bit-for-bit properties
# --------------------------------------------------------------------------------------------------------------------
def call(imsize, mode, W, U, V, x, aug, d_out, training=True):
    """(out, u, v, sigma, dW list, input gradient) of one forward + full backward, u / v reset to the given values"""
    U, V = [u.clone() for u in U], [v.clone() for v in V]
    out, ws = forward(imsize, mode, training, W, U, V, x, aug)
    n, _, h, w = x.shape
    dx = torch.full((n, 3, h, w), NAN, device=DEV)
    dW = backward(imsize, mode, W, x.shape, d_out, ws, set(range(len(W))), d_input=dx)
    L = len(W)
    return out, U, V, ws[:de.MAX_LAYERS][:L].clone(), dW, dx


@pytest.mark.parametrize("mode", MODE_LIST)
def test_input_layouts_give_the_same_bits(mode):
    """NCHW, the ray-major view, padded channels-last and a stride-0 batch of one repeated image"""
    imsize, n, h, w = -1, 3, 56, 70
    W, U, V = state(imsize, 4)
    x = torch.rand(1, 3, h, w, generator=torch.Generator().manual_seed(2)).expand(n, 3, h, w).contiguous()
    aug = draws(n, h, w, 0)
    d_out = torch.randn(n, 1, *output_sizes(imsize, h, w)[-1], generator=torch.Generator().manual_seed(3)).to(DEV)
    def flat(r):
        out, u, v, sigma, dW, dx = r
        return [out, *u, *v, sigma, *dW, dx]
    ref = flat(call(imsize, mode, W, U, V, placed(x, "nchw"), aug, d_out))
    for layout in ("rays", "cl_pad", "expand"):
        got = flat(call(imsize, mode, W, U, V, placed(x, layout), aug, d_out))
        assert all(same_bits(a, c) for a, c in zip(ref, got)), layout


@pytest.mark.parametrize("mode", MODE_LIST)
def test_batch_of_8_equals_single_calls(mode):
    """an image's output, and sigma, u and v, do not depend on the other images of the call"""
    imsize, n, h, w = 64, 8, 64, 64
    W, U, V = state(imsize, 6)
    x = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(5))
    aug = draws(n, h, w, 0)
    U8, V8 = [u.clone() for u in U], [v.clone() for v in V]
    out8, ws8 = forward(imsize, mode, True, W, U8, V8, placed(x, "nchw"), aug)
    for i in range(n):
        U1, V1 = [u.clone() for u in U], [v.clone() for v in V]
        out1, ws1 = forward(imsize, mode, True, W, U1, V1, placed(x[i:i + 1], "rays"), tuple(t[i:i + 1] for t in aug))
        assert same_bits(out1[0], out8[i]), i
        assert same_bits(ws1[:de.MAX_LAYERS], ws8[:de.MAX_LAYERS]), i
        assert all(same_bits(a, c) for a, c in zip(U1 + V1, U8 + V8)), i


@pytest.mark.parametrize("mode", MODE_LIST)
def test_weight_scaling_is_exact(mode):
    """W 2^j for j in [-30, 30] (clear of the eps clamp and of underflow in sum t^2): output, u and v bit-identical,
    dW_orig exactly 2^-j times the j = 0 result, the input gradient unchanged"""
    imsize, n, h, w = -1, 2, 63, 84
    W, U, V = state(imsize, 7)
    x = placed(torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(8)), "rays")
    aug = draws(n, h, w, 3)
    d_out = torch.randn(n, 1, *output_sizes(imsize, h, w)[-1], generator=torch.Generator().manual_seed(9)).to(DEV)
    out, u, v, _, dW, dx = call(imsize, mode, W, U, V, x, aug, d_out)
    for j in (-30, -17, -1, 5, 30):
        o2, u2, v2, _, dW2, dx2 = call(imsize, mode, [t * 2.0 ** j for t in W], U, V, x, aug, d_out)
        assert same_bits(o2, out) and all(same_bits(a, c) for a, c in zip(u2 + v2, u + v)), j
        assert same_bits(dx2, dx), j
        assert all(same_bits(a, de.ldexp32(c, -j)) for a, c in zip(dW2, dW)), j


@pytest.mark.parametrize("mode", MODE_LIST)
def test_upstream_scaling_is_exact(mode):
    """d_out 2^j from 2^100 down to 2^-149: every gradient is ldexpf(its j = 0 value, j), rounded once, bit for bit.
    d_out holds integers below 2^10, so d_out 2^j is itself exact down to 2^-149."""
    imsize, n, h, w = 64, 2, 64, 64
    W, U, V = state(imsize, 10)
    x = placed(torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(11)), "nchw")
    aug = draws(n, h, w, 1)
    d_out = torch.randint(-1000, 1001, (n, 1, 1, 1), generator=torch.Generator().manual_seed(12)).float().to(DEV)
    out, ws = forward(imsize, mode, True, W, U, V, x, aug)

    def grads(scale):
        dx = torch.full((n, 3, h, w), NAN, device=DEV)
        return backward(imsize, mode, W, x.shape, d_out * scale, ws, set(range(len(W))), d_input=dx) + [dx]
    g0 = grads(1.0)
    assert all(torch.isfinite(t).all() and float(t.abs().max()) > 0 for t in g0)
    for j in (100, 64, 10, -30, -100, -126, -130, -135, -136, -140, -145, -147, -149):
        gj = grads(2.0 ** j)
        want = [de.ldexp32(t, j) for t in g0]
        nz = sum(int((t != 0).sum()) for t in want)
        differ = [int((a != c).sum()) for a, c in zip(gj, want)]
        print(f"disc upstream 2^{j} {mode}: {nz} nonzero expected elements, elements differing per gradient {differ}")
        assert not any(differ), (j, differ)


@pytest.mark.parametrize("mode", MODE_LIST)
def test_degenerate_upstream(mode):
    """an all-zero upstream gives exact zeros; a NaN in it gives NaN gradients, not finite ones"""
    imsize, n, h, w = -1, 2, 56, 70
    W, U, V = state(imsize, 13)
    x = placed(torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(14)), "nchw")
    out, ws = forward(imsize, mode, True, W, U, V, x, draws(n, h, w, 2))

    def grads(d):
        dx = torch.full((n, 3, h, w), NAN, device=DEV)
        return backward(imsize, mode, W, x.shape, d, ws, set(range(len(W))), d_input=dx) + [dx]
    for t in grads(torch.zeros_like(out)):
        assert bool((t == 0).all())
    d = torch.randn(out.shape, generator=torch.Generator().manual_seed(15)).to(DEV)
    d.view(-1)[d.numel() // 2] = NAN
    for i, t in enumerate(grads(d)):
        assert bool(t.isnan().any()), i
