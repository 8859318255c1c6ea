"""The discriminator's gradient-penalty kernels (csrc/disc.cu, snb_disc_penalty_*) stage by stage against float64.

tests/test_gpu_disc_penalty.py holds reg and its gradients to the float64 oracle end to end, at rel-L2 bars loose
enough for LeakyReLU kinks flipped by rounding; a wrong sub-term of the second-order fold, a misaligned exponent or a
mis-addressed GEMM slice fits under them.  Here the kernels run through the C ABI on a workspace this file allocates
(filled with NaN first), and every stage the workspace brackets is recomputed in float64 from the kernel's OWN inputs
(tests/disc_penalty_emulation.py), so errors do not compound and no kink can flip.  A penalty backward with no d_out,
one wanted weight gradient and no input gradient stops after that layer: calling it once per layer leaves each
layer's adjoints, dcols and fold behind.

Bit for bit: the penalty direction and its exponent, the tangent DiffAugment words, the tangent gathers (as copies,
with the primal's slope), every rescale, the combined exponent, the write of the penalty dW, partial against full
backwards; and the properties at the end of the file (g against the plain backward, d_reg 2^j down to 2^-149, W 2^j,
a zero d_reg image, d_out plus penalty, determinism, saved state, input layouts, degenerate d_reg).
"""
import ctypes as C

import pytest
import torch

from sinnerf_b200 import _lib
from sinnerf_b200.discriminator import output_sizes
from tests import disc_emulation as de
from tests import disc_penalty_emulation as dp
from tests.test_gpu_disc_stages import DEV, NAN, bits, c_ptrs, draws, padded_grad, placed, same_bits, state

pytestmark = pytest.mark.gpu
MODE_LIST = list(de.MODES)
# (imsize, h, w, n, augmented, training, input layout, d_reg pattern): every branch at its recipe size, odd sizes and
# the smallest legal size, n = 1, 3, 8, training and eval, augmentation off and on (the draws put the cutout at each
# clamped corner and inside, saturation 0 / 1 / 2), d_reg uniform 10 / n, spread over the images by up to 2^+-8, and
# with one image at exactly 0
CASES = [(128, 128, 128, 1, True, True, "nchw", "uniform"), (64, 64, 64, 3, False, True, "rays", "spread"),
         (64, 67, 75, 8, True, False, "cl_pad", "zero"), (32, 32, 32, 3, True, True, "nchw", "zero"),
         (32, 33, 47, 1, False, False, "rays", "uniform"), (-1, 63, 84, 8, True, True, "nchw", "spread"),
         (-1, 56, 70, 3, False, True, "cl_pad", "uniform"), (-1, 16, 16, 8, True, True, "rays", "zero")]


def case_id(c):
    return (f"{c[0]}-{c[1]}x{c[2]}-n{c[3]}-{'aug' if c[4] else 'noaug'}-{'train' if c[5] else 'eval'}-{c[6]}-"
            f"{c[7]}")


def d_reg_of(pattern, n):
    if pattern == "uniform":
        return torch.full((n,), 10.0 / n, device=DEV)
    e = torch.linspace(-8, 8, n) if n > 1 else torch.zeros(1)
    d = (10.0 / n) * torch.pow(2.0, e.round())
    if pattern == "zero":
        d[n // 2] = 0.0
    return d.float().to(DEV)


# --------------------------------------------------------------------------------------------------------------------
# driving the C ABI
# --------------------------------------------------------------------------------------------------------------------
def pen_forward(imsize, mode, training, W, U, V, x, aug):
    """(out, reg, workspace) of snb_disc_penalty_forward on a NaN-filled workspace; U / V advance in training mode"""
    lib = _lib.load()
    n, _, h, w = x.shape
    ws = torch.full((lib.snb_disc_penalty_workspace_bytes(imsize, n, h, w) // 4,), NAN, device=DEV)
    out = torch.full((n, 1, *output_sizes(imsize, h, w)[-1]), NAN, device=DEV)
    reg = torch.full((n,), NAN, device=DEV)
    a = None if aug is None else C.byref(_lib.SnbDiscAug(*[t.data_ptr() for t in aug]))
    _lib.check(lib.snb_disc_penalty_forward(imsize, de.MODES[mode], int(training), c_ptrs(W), c_ptrs(U), c_ptrs(V),
                                            _lib.ptr(x), (C.c_int64 * 4)(*x.stride()), n, h, w, a, _lib.ptr(out),
                                            _lib.ptr(reg), _lib.ptr(ws), _lib.stream_ptr(DEV)),
               "snb_disc_penalty_forward")
    return out, reg, ws


def pen_backward(imsize, mode, W, shape, d_out, d_reg, ws, want, d_input=None, init=None):
    """[dW or None] of snb_disc_penalty_backward for the layers in `want` (NaN-filled first, or copies of `init`);
    d_input: a view to write (or to add to, with d_out)"""
    lib = _lib.load()
    n, _, h, w = shape
    if init is None:
        dws = [torch.full_like(t, NAN) if i in want else None for i, t in enumerate(W)]
    else:
        dws = [init[i].clone() if i in want else None for i in range(len(W))]
    strides = None if d_input is None else (C.c_int64 * 4)(*d_input.stride())
    _lib.check(lib.snb_disc_penalty_backward(imsize, de.MODES[mode], c_ptrs(W), n, h, w,
                                             None if d_out is None else _lib.ptr(d_out.contiguous()),
                                             None if d_reg is None else _lib.ptr(d_reg.contiguous()),
                                             _lib.ptr(d_input), strides, c_ptrs(dws), _lib.ptr(ws),
                                             _lib.stream_ptr(DEV)), "snb_disc_penalty_backward")
    return dws


def plain_backward(imsize, mode, W, shape, d_out, ws, want, d_input=None):
    lib = _lib.load()
    n, _, h, w = shape
    dws = [torch.full_like(t, NAN) if i in want else None for i, t in enumerate(W)]
    strides = None if d_input is None else (C.c_int64 * 4)(*d_input.stride())
    _lib.check(lib.snb_disc_backward(imsize, de.MODES[mode], c_ptrs(W), n, h, w, _lib.ptr(d_out.contiguous()),
                                     _lib.ptr(d_input), strides, c_ptrs(dws), _lib.ptr(ws), _lib.stream_ptr(DEV)),
               "snb_disc_backward")
    return dws


def plain_forward(imsize, mode, training, W, U, V, x, aug):
    lib = _lib.load()
    n, _, h, w = x.shape
    ws = torch.full((lib.snb_disc_workspace_bytes(imsize, n, h, w, 1) // 4,), NAN, device=DEV)
    out = torch.full((n, 1, *output_sizes(imsize, h, w)[-1]), NAN, device=DEV)
    a = None if aug is None else C.byref(_lib.SnbDiscAug(*[t.data_ptr() for t in aug]))
    _lib.check(lib.snb_disc_forward(imsize, de.MODES[mode], int(training), c_ptrs(W), c_ptrs(U), c_ptrs(V),
                                    _lib.ptr(x), (C.c_int64 * 4)(*x.stride()), n, h, w, a, _lib.ptr(out),
                                    _lib.ptr(ws), _lib.stream_ptr(DEV)), "snb_disc_forward")
    return out, ws


# --------------------------------------------------------------------------------------------------------------------
# the stage record
# --------------------------------------------------------------------------------------------------------------------
class Stages:
    """per stage: the largest worst and rms over its instances; the bit-for-bit checks that failed.  Everything is
    printed before anything is asserted."""

    def __init__(self, mode, what):
        self.mode, self.what, self.e, self.bad = mode, what, {}, []

    def add(self, stage, y, ref, scale):
        if torch.isnan(y).any():
            self.bad.append((stage, "NaN"))
            return
        new = de.stats(de.err(y, ref, scale))
        old = self.e.get(stage, (0.0, 0.0))
        self.e[stage] = tuple(max(a, b) for a, b in zip(old, new))

    def exact(self, what, ok):
        if not ok:
            self.bad.append((what, "bits"))

    def check(self):
        for stage, (w, r) in sorted(self.e.items()):
            bw, br = dp.PEN_BARS[self.mode][stage]
            print(f"disc penalty stages {self.what} {self.mode:5s} {stage:9s}: worst {w:.2e} rms {r:.2e} "
                  f"(bars {bw:.0e} {br:.0e})")
            if not (w <= bw and r <= br):
                self.bad.append((stage, w, r))
        assert not self.bad, self.bad


def forward_state(b):
    """copies of what the penalty forward leaves for the backwards: each layer's col, y, InstanceNorm statistics,
    scaled weight, u and v, the sigma words, the DiffAugment words, g and the all-ones upstream"""
    keys = [k for k in b if k.rstrip("0123456789") in ("col", "y", "mean", "rstd", "ws", "u", "v")]
    return {k: b[k].clone() for k in keys + ["sigma", "inv_sigma", "alpha", "wscale", "aug", "g", "ones"]}


def rescaled(st, what, scaled, e_hi, e_lo):
    """scaled = fold output 2^k with k = e_hi - e_lo, its largest |.| in [2^14, 2^15) (bit for bit; a zero output:
    k = 0): -> the unscaled output, float64"""
    k = e_hi - e_lo
    un = scaled.double() * 2.0 ** -k
    st.exact(what, de.pow2_exponent(un.abs().max()) == k and same_bits(de.ldexp32(un, k), scaled))
    return un


def tangent_col_check(st, layers, i, tcol, col, zref, zscale, f):
    """layer i >= 1's tangent col: a copy, bit for bit, of one value per source element (the gather), zero in the
    padding, with the LeakyReLU slope exactly where the forward gather's primal col is <= 0; the copied values against
    the float64 tangent zref (C, n, P) 2^f of the previous stage ('zdot')"""
    y = layers[i]
    src = dp.source_index(y, DEV)
    pad = src < 0
    st.exact(f"tgather{i} padding", bool((bits(tcol)[pad] == 0).all()))
    rep = torch.full((y["n"] * y["cin"] * y["hin"] * y["win"],), NAN, device=DEV)
    rep[src[~pad]] = tcol[~pad]
    st.exact(f"tgather{i} copies", same_bits(torch.where(pad, torch.zeros_like(tcol), rep[src.clamp_min(0)]), tcol))
    pos = torch.zeros_like(rep, dtype=torch.bool)
    pos[src[~pad]] = col[~pad] > 0
    st.exact(f"tgather{i} primal sign consistent", bool(((col > 0) == pos[src.clamp_min(0)])[~pad].all()))
    shape = (y["n"], y["cin"], y["hin"], y["win"])
    if zref is None:
        return rep.view(shape), pos.view(shape)
    sl = torch.where(pos.view(shape), 1.0, dp.SLOPE).double()
    ref = (zref.transpose(0, 1).reshape(shape) * 2.0 ** f) * sl
    sc = (zscale.transpose(0, 1).reshape(shape) * 2.0 ** f) * sl
    covered = ~rep.isnan().view(shape)
    st.add("zdot", rep.view(shape)[covered], ref[covered], sc[covered])
    return rep.view(shape), pos.view(shape)


# --------------------------------------------------------------------------------------------------------------------
# stage by stage
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODE_LIST)
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_stages(case, mode):
    imsize, h, w, n, aug_on, training, layout, pattern = case
    W, U, V = state(imsize, seed=h + n)
    g0 = torch.Generator().manual_seed(1000 * h + w + n)
    xc = torch.rand(n, 3, h, w, generator=g0)
    x = placed(xc, layout)
    aug = draws(n, h, w, start=h + n) if aug_on else None
    out, reg, wsp = pen_forward(imsize, mode, training, W, U, V, x, aug)
    torch.cuda.synchronize()
    b = dp.workspace_views(wsp, imsize, n, h, w)
    layers = de.net(imsize, n, h, w)
    L = len(layers)
    st = Stages(mode, case_id(case))
    saved = forward_state(b)
    st.add("reg", reg, *dp.reg_ref(b["g"]))
    st.exact("ones", bool((b["ones"] == 1).all()))
    d_reg = d_reg_of(pattern, n)

    # ---- the tangent forward (identical in every penalty backward): checked after the first
    partial = []
    for k in range(L - 1, -1, -1):
        (dWk,) = [t for t in pen_backward(imsize, mode, W, x.shape, None, d_reg, wsp, {k}) if t is not None]
        torch.cuda.synchronize()
        partial.append((k, dWk))
        ev, gt, gp, gu, gw = ([int(e) for e in b[key][:L]] for key in ("ev", "gt", "gp", "gu", "gw"))
        if k == L - 1:
            dreg, vt, ev0 = dp.pen_dir_ref(b["g"], d_reg)
            st.exact("dreg", same_bits(b["dreg"], dreg))
            st.exact("pen_dir + tangent scale", same_bits(b["vt"], vt) and ev[0] == ev0)
            if aug is None:
                st.exact("taug off", bool((b["taug"][:, 0] == 0).all()))
                st.exact("tgather0 copy", same_bits(b["tcol0"], de.unfold(b["vt"], layers[0])))
            else:
                tf, box = dp.taug_words(b["aug"])
                st.exact("taug words", same_bits(b["taug"][:, :4], tf) and same_bits(b["taug"][:, 5:9], box))
                st.add("taug_mean", b["taug"][:, 4], *dp.taug_mean_ref(b["vt"], tf[:, 2]))
                ref, mag, cut = de.gather0_ref(layers, b["vt"], b["taug"][:, :4], b["taug"][:, 4], box)
                st.add("tgather0", b["tcol0"], ref, mag * 2.0 ** -24)
                st.exact("tangent cutout zeros", bool((b["tcol0"][cut] == 0).all()))
            st.exact("tgather0 padding", bool((bits(b["tcol0"])[de.pad_mask(layers[0], DEV)] == 0).all()))
            for i, y in enumerate(layers[:-1]):
                ty = b[f"ty{i}"]
                emu, _, sc = de.gemm_fwd_ref(b[f"ws{i}"], b[f"tcol{i}"], b["alpha"][i], 1.0, mode)
                st.add("ty", ty.reshape(y["cout"], -1), emu, sc)
                if y["in_norm"]:
                    m, q, msc, qsc = dp.in_tangent_ref(ty, b[f"y{i}"], b[f"mean{i}"], b[f"rstd{i}"], b[f"tmean{i}"])
                    st.add("tmean", b[f"tmean{i}"], m, msc)
                    st.add("tq", b[f"tq{i}"], q, qsc)
                    z, zsc = dp.zdot_ref(ty, b[f"y{i}"], b[f"mean{i}"], b[f"rstd{i}"], b[f"tmean{i}"], b[f"tq{i}"])
                    rep, _ = tangent_col_check(st, layers, i + 1, b[f"tcol{i + 1}"], b[f"col{i + 1}"], z, zsc,
                                               ev[i] - ev[i + 1])
                else:   # no InstanceNorm: the rescaled GEMM output itself, gathered with the primal's slope
                    rep, _ = tangent_col_check(st, layers, i + 1, b[f"tcol{i + 1}"], b[f"col{i + 1}"], None, None, 0)
                    st.exact(f"tgather{i + 1}", same_bits(b[f"tcol{i + 1}"], dp.tangent_gather(
                        layers, i + 1, de.ldexp32(ty, ev[i] - ev[i + 1]), b[f"y{i}"], None, None)))
                # the largest rescaled tangent is in [2^14, 2^15): the rescale's exponent is ev[i] - ev[i + 1]
                nv = de.normalized(b[f"y{i}"], b.get(f"mean{i}"), b.get(f"rstd{i}"))
                zs = torch.where(nv.reshape(rep.shape) > 0, rep.double(), rep.double() / dp.SLOPE)
                mx = float(zs.nan_to_num(0).abs().max())
                st.exact(f"tangent rescale{i + 1} range", mx == 0 or 2.0 ** 14 * (1 - 2 ** -22) <= mx < 2.0 ** 15)
            st.exact(f"tcol{L - 1} written", not bool(b[f"tcol{L - 1}"].isnan().any()))
            st.exact("top tangent adjoint", bool((b["dy0"][:n * layers[-1]["P"]] == 2.0 ** 14).all())
                     and gt[L - 1] == -14)

        y = layers[k]
        t = b[dp.t_buffer(L, k)][:y["cout"] * n * y["P"]].view(y["cout"], -1)
        p = b[dp.p_buffer(L, k)][:y["cout"] * n * y["P"]].view(y["cout"], -1)
        if k < L - 1:   # layer k + 1's dual dgrad, its second-order fold and the two rescales that made t / p
            z = layers[k + 1]
            rows = n * z["P"]
            tz = b[dp.t_buffer(L, k + 1)][:z["cout"] * rows].view(z["cout"], -1)
            pz = b[dp.p_buffer(L, k + 1)][:z["cout"] * rows].view(z["cout"], -1)
            have_p = k + 1 < L - 1
            dcol = b["dcol"][:rows * z["K"]].view(rows, z["K"])
            dcolp = b["dcolp"][:rows * z["K"]].view(rows, z["K"])
            emu, _, sc = de.dgrad_ref(tz, b[f"ws{k + 1}"], b["alpha"][k + 1], mode)
            st.add("dgrad_t", dcol, emu, sc)
            if have_p:
                emu, _, sc = de.dgrad_ref(pz, b[f"ws{k + 1}"], b["alpha"][k + 1], mode)
                st.add("dgrad_p", dcolp, emu, sc)
            ot, op, eo, sct, scp = dp.fold2_ref(layers, k + 1, dcol, dcolp if have_p else None, b[f"y{k}"],
                                                b.get(f"mean{k}"), b.get(f"rstd{k}"), b[f"ty{k}"], b.get(f"tmean{k}"),
                                                b.get(f"tq{k}"), gt[k + 1], gp[k + 1] if have_p else None, ev[k])
            st.exact(f"fold2 exponent{k}", gu[k] == eo)
            ut = rescaled(st, f"rescale t{k}", t, gt[k + 1], gt[k])
            up = rescaled(st, f"rescale p{k}", p, gu[k], gp[k])
            st.add("fold2_t", ut.view_as(ot), ot, sct)
            st.add("fold2_p", up.view_as(op), op, scp)
        # the weight gradient: the primal stream's raw GEMM, the combine at the larger exponent, part, the correction
        Wm = W[k].reshape(y["cout"], -1)
        et = gt[k] + ev[k]
        if k < L - 1:
            emu, _, sc_p = de.wgrad_ref(p, b[f"col{k}"], de.col_scale(layers, k), mode)
            st.add("wgrad_p", b[f"dwp{k}"], emu, sc_p)
            st.exact(f"combine exponent{k}", gw[k] == max(et, gp[k]))
            dwp = b[f"dwp{k}"].double() * 2.0 ** (gp[k] - gw[k])
            dwp_abs = dwp.abs()
        else:
            st.exact(f"combine exponent{k}", gw[k] == et)
            dwp, dwp_abs = 0.0, 0.0
        emu, _, sc_t = de.wgrad_ref(t, b[f"tcol{k}"], 1.0, mode)
        comb = emu * 2.0 ** (et - gw[k]) + dwp
        comb_abs = sc_t * 2.0 ** (et - gw[k]) + dwp_abs
        st.add("part", b[f"part{k}"], *de.part_ref(comb, comb_abs, Wm))
        ref, sc = de.sn_fix_ref(comb, comb_abs, b[f"part{k}"], b["inv_sigma"][k], b[f"u{k}"], b[f"v{k}"], gw[k])
        st.add("wgrad_t", dWk.reshape(y["cout"], -1), ref, sc)
        st.exact(f"pen_add write{k}", same_bits(dWk.reshape(y["cout"], -1), b[f"dwt{k}"]))

    # ---- the input gradient alone: the primal stream's layer-0 dgrad and fold, then the DiffAugment backward at gp[0]
    buf, dxv = padded_grad(n, h, w)
    pen_backward(imsize, mode, W, x.shape, None, d_reg, wsp, set(), d_input=dxv)
    torch.cuda.synchronize()
    gp0 = int(b["gp"][0])
    y = layers[0]
    p = b[dp.p_buffer(L, 0)][:y["cout"] * n * y["P"]].view(y["cout"], -1)
    dcolp = b["dcolp"][:n * y["P"] * y["K"]].view(n * y["P"], y["K"])
    emu, _, sc = de.dgrad_ref(p, b["ws0"], b["alpha"][0], mode)
    st.add("dgrad_p", dcolp, emu, sc)
    ref, sc, _ = de.fold_ref(layers, 0, dcolp, None, None, None)
    st.add("fold", b["dx"], ref, sc)
    if aug is None:
        st.exact("input gradient", same_bits(dxv, de.ldexp32(b["dx"].transpose(0, 1).reshape(n, 3, h, w), gp0)))
    else:
        st.add("aug_bwd", dxv, *de.aug_bwd_ref(b["dx"], b["aug"][:, :4], de.aug_words(aug, h, w)[1], gp0, h, w))
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:, 1:, 1:w + 1, 2:5] = False
    st.exact("input gradient padding untouched", bool(buf[outside].isnan().all()))

    # ---- the full backward: the same dW as each partial call and the same input gradient, twice
    for rep in range(2):
        full_dx = torch.full((n, 3, h, w), NAN, device=DEV)
        full = pen_backward(imsize, mode, W, x.shape, None, d_reg, wsp, set(range(L)), d_input=full_dx)
        torch.cuda.synchronize()
        st.exact(f"full backward {rep}: partial dW", all(same_bits(full[k], dWk) for k, dWk in partial))
        st.exact(f"full backward {rep}: input gradient", same_bits(full_dx, dxv))
    st.exact("saved forward state", all(same_bits(b[k], v) for k, v in saved.items()))
    st.check()


# --------------------------------------------------------------------------------------------------------------------
# bit-for-bit properties
# --------------------------------------------------------------------------------------------------------------------
def setup(imsize, n, h, w, seed, layout="nchw"):
    W, U, V = state(imsize, seed)
    x = placed(torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed + 1)), layout)
    return W, U, V, x, draws(n, h, w, seed % 5)


def grads(imsize, mode, W, x, d_out, d_reg, ws, d_input=None, init=None):
    n, _, h, w = x.shape
    dx = torch.full((n, 3, h, w), NAN, device=DEV) if d_input is None else d_input
    return pen_backward(imsize, mode, W, x.shape, d_out, d_reg, ws, set(range(len(W))), d_input=dx, init=init) + [dx]


@pytest.mark.parametrize("mode", MODE_LIST)
def test_g_is_the_plain_backward_from_ones(mode):
    """the penalty workspace's g is snb_disc_backward from an all-ones upstream into a contiguous input gradient"""
    for imsize, n, h, w in ((64, 3, 64, 64), (-1, 2, 63, 84)):
        W, U, V, x, aug = setup(imsize, n, h, w, 20)
        _, _, wsp = pen_forward(imsize, mode, True, W, [u.clone() for u in U], [v.clone() for v in V], x, aug)
        out, ws1 = plain_forward(imsize, mode, True, W, [u.clone() for u in U], [v.clone() for v in V], x, aug)
        g = torch.full((n, 3, h, w), NAN, device=DEV)
        plain_backward(imsize, mode, W, x.shape, torch.ones_like(out), ws1, set(), d_input=g)
        assert same_bits(dp.workspace_views(wsp, imsize, n, h, w)["g"], g), imsize


@pytest.mark.parametrize("mode", MODE_LIST)
def test_d_reg_scaling_is_exact(mode):
    """d_reg 2^j from 2^100 down to 2^-149: every penalty gradient is ldexpf(its j = 0 value, j), rounded once, bit for
    bit.  d_reg holds integers below 2^10, so d_reg 2^j is itself exact down to 2^-149."""
    imsize, n, h, w = 64, 2, 64, 64
    W, U, V, x, aug = setup(imsize, n, h, w, 30)
    _, _, ws = pen_forward(imsize, mode, True, W, U, V, x, aug)
    d_reg = torch.tensor([700.0, 3.0], device=DEV)
    g0 = grads(imsize, mode, W, x, None, d_reg, ws)
    assert all(torch.isfinite(t).all() and float(t.abs().max()) > 0 for t in g0)
    bad = {}
    for j in (100, 64, 10, -30, -100, -126, -130, -140, -149):
        gj = grads(imsize, mode, W, x, None, d_reg * 2.0 ** j, ws)
        want = [de.ldexp32(t, j) for t in g0]
        nz = sum(int((t != 0).sum()) for t in want)
        differ = [int((a != c).sum()) for a, c in zip(gj, want)]
        print(f"disc penalty d_reg 2^{j} {mode}: {nz} nonzero expected elements, elements differing per gradient "
              f"{differ}")
        if any(differ):
            bad[j] = differ
    assert not bad, bad


@pytest.mark.parametrize("mode", MODE_LIST)
def test_weight_scaling_is_exact(mode):
    """W 2^j for j in [-30, 30]: out, reg, u and v bit-identical, the penalty dW exactly 2^-j times its j = 0 value,
    the penalty input gradient unchanged"""
    imsize, n, h, w = -1, 2, 63, 84
    W, U, V, x, aug = setup(imsize, n, h, w, 40, "rays")
    d_reg = torch.tensor([5.0, 0.75], device=DEV)

    def call(Ws):
        U2, V2 = [u.clone() for u in U], [v.clone() for v in V]
        out, reg, ws = pen_forward(imsize, mode, True, Ws, U2, V2, x, aug)
        return out, reg, U2 + V2, grads(imsize, mode, Ws, x, None, d_reg, ws)
    out, reg, uv, g = call(W)
    for j in (-30, -17, -1, 5, 30):
        o2, r2, uv2, g2 = call([t * 2.0 ** j for t in W])
        assert same_bits(o2, out) and same_bits(r2, reg) and all(same_bits(a, c) for a, c in zip(uv2, uv)), j
        assert same_bits(g2[-1], g[-1]), j
        assert all(same_bits(a, de.ldexp32(c, -j)) for a, c in zip(g2[:-1], g[:-1])), j


@pytest.mark.parametrize("mode", MODE_LIST)
def test_zero_d_reg_image(mode):
    """an image with d_reg = 0 gets an exactly zero penalty input gradient; every other image's gradient is that of a
    call without it within the stage bars"""
    imsize, n, h, w = 32, 3, 33, 47
    W, U, V, x, aug = setup(imsize, n, h, w, 50)
    _, _, ws = pen_forward(imsize, mode, True, W, U, V, x, aug)
    d_reg = torch.tensor([2.0, 0.0, 0.5], device=DEV)
    dx = grads(imsize, mode, W, x, None, d_reg, ws)[-1]
    assert bool((dx[1] == 0).all())
    for b in (0, 2):
        one = torch.zeros(n, device=DEV)
        one[b] = d_reg[b]
        dxb = grads(imsize, mode, W, x, None, one, ws)[-1]
        # the images only meet in the weight-gradient GEMMs and the common exponents: another image's d_reg changes
        # the rounding of this one's gradient, nothing more
        e = float(((dx[b] - dxb[b]).abs().max() / dxb[b].abs().max()))
        assert e <= 1e-5, (b, e)


@pytest.mark.parametrize("mode", MODE_LIST)
def test_d_out_plus_penalty(mode):
    """with d_out given, every gradient is the first-order backward's plus the d_out = NULL penalty result, added in
    fp32 (bit for bit)"""
    imsize, n, h, w = 64, 2, 67, 75
    W, U, V, x, aug = setup(imsize, n, h, w, 60, "cl_pad")
    out, _, ws = pen_forward(imsize, mode, True, W, U, V, x, aug)
    d_out = torch.randn(out.shape, generator=torch.Generator().manual_seed(61)).to(DEV)
    d_reg = torch.tensor([3.0, 7.0], device=DEV)
    first = grads(imsize, mode, W, x, d_out, None, ws)
    pen = grads(imsize, mode, W, x, None, d_reg, ws)
    both = grads(imsize, mode, W, x, d_out, d_reg, ws)
    for i, (a, f, p) in enumerate(zip(both, first, pen)):
        assert same_bits(a, f + p), i


@pytest.mark.parametrize("mode", MODE_LIST)
def test_repeat_and_saved_state(mode):
    """two identical backwards give the same bits, and no backward touches the forward's saved state"""
    imsize, n, h, w = 128, 2, 128, 128
    W, U, V, x, aug = setup(imsize, n, h, w, 70)
    out, _, wsp = pen_forward(imsize, mode, True, W, U, V, x, aug)
    b = dp.workspace_views(wsp, imsize, n, h, w)
    saved = forward_state(b)
    d_out = torch.randn(out.shape, generator=torch.Generator().manual_seed(71)).to(DEV)
    d_reg = torch.tensor([5.0, 5.0], device=DEV)
    r1 = grads(imsize, mode, W, x, d_out, d_reg, wsp)
    r2 = grads(imsize, mode, W, x, d_out, d_reg, wsp)
    assert all(same_bits(a, c) for a, c in zip(r1, r2))
    assert all(same_bits(b[k], v) for k, v in saved.items())


@pytest.mark.parametrize("mode", MODE_LIST)
def test_input_gradient_layouts_give_the_same_bits(mode):
    """the penalty input gradient written NCHW, ray-major and padded channels-last: the same bits, the padding of the
    padded view left NaN; with d_out, the same holds for the accumulated gradient"""
    imsize, n, h, w = -1, 3, 56, 70
    W, U, V, x, aug = setup(imsize, n, h, w, 80)
    out, _, ws = pen_forward(imsize, mode, True, W, U, V, x, aug)
    d_reg = torch.tensor([1.0, 3.0, 0.25], device=DEV)
    d_out = torch.randn(out.shape, generator=torch.Generator().manual_seed(81)).to(DEV)
    for d in (None, d_out):
        ref = grads(imsize, mode, W, x, d, d_reg, ws)[-1]
        rays = torch.full((n * h * w, 3), NAN, device=DEV)
        got = grads(imsize, mode, W, x, d, d_reg, ws, d_input=rays.view(n, h, w, 3).permute(0, 3, 1, 2))[-1]
        assert same_bits(got, ref)
        buf, view = padded_grad(n, h, w)
        got = grads(imsize, mode, W, x, d, d_reg, ws, d_input=view)[-1]
        assert same_bits(got, ref)
        outside = torch.ones_like(buf, dtype=torch.bool)
        outside[:, 1:, 1:w + 1, 2:5] = False
        assert bool(buf[outside].isnan().all())


@pytest.mark.parametrize("mode", MODE_LIST)
def test_degenerate_d_reg(mode):
    """an all-zero d_reg gives exact zeros; a NaN in d_reg gives NaN gradients, never finite ones"""
    imsize, n, h, w = -1, 2, 56, 70
    W, U, V, x, aug = setup(imsize, n, h, w, 90)
    _, _, ws = pen_forward(imsize, mode, True, W, U, V, x, aug)
    for t in grads(imsize, mode, W, x, None, torch.zeros(n, device=DEV), ws):
        assert bool((t == 0).all())
    for i, t in enumerate(grads(imsize, mode, W, x, None, torch.tensor([1.0, NAN], device=DEV), ws)):
        assert bool(t.isnan().any()), i
