"""CPU side of the gradient-penalty stage tests (tests/test_gpu_disc_penalty_stages.py):
- the restated penalty workspace layout (tests/disc_penalty_emulation.py) against the library's byte count;
- the second-order fold's closed form against float64 autograd's double backward of InstanceNorm -> LeakyReLU, an
  independent derivation;
- the chained stage references against the float64 oracle (tests/disc_oracle.py under create_graph=True) and the
  reference module's golden file;
- the per-stage bars have teeth: defects planted in the emulation each exceed the bar of the stage that sees them.
  Each defect's end-to-end error against the oracle is printed next to the bars of tests/test_gpu_disc_penalty.py."""
import os

import numpy as np
import pytest
import torch

from sinnerf_b200 import _lib, build
from sinnerf_b200.discriminator import Discriminator
from tests import disc_emulation as de
from tests import disc_oracle as do
from tests import disc_penalty_emulation as dp
from tests._common import rel_l2
from tests.golden.make_disc_penalty_golden import case_name, inputs

BRANCHES = [(128, 128, 128), (64, 64, 64), (64, 67, 75), (32, 32, 32), (32, 33, 47), (-1, 63, 84), (-1, 56, 70),
            (-1, 16, 16)]
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "disc_penalty.npz")
# tests/test_gpu_disc_penalty.py's split-mode rel-L2 bars for reg and for the gradients
E2E_BARS = (1e-4, 1e-4)


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


@pytest.mark.parametrize("imsize,h,w", BRANCHES)
def test_workspace_layout_matches_library(lib, imsize, h, w):
    for n in (1, 3, 8):
        bufs, total = dp.workspace_layout(imsize, n, h, w)
        assert lib.snb_disc_penalty_workspace_bytes(imsize, n, h, w) == 4 * total, n
        spans = sorted((o, o + torch.Size(s).numel(), k) for k, (o, s) in bufs.items())
        exps = {"ev", "gt", "gp", "gu", "gw"}
        assert all(o % 64 == 0 for o, _, k in spans if k not in exps - {"ev"})
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), n       # no overlap
        L = len(de.net(imsize, n, h, w))
        assert f"tcol{L - 1}" in bufs and f"ty{L - 1}" not in bufs and f"tmean{L - 1}" not in bufs


# --------------------------------------------------------------------------------------------------------------------
# the second-order fold's closed form against autograd
# --------------------------------------------------------------------------------------------------------------------
def autograd_in_lrelu(gt, gp, y, yd, in_norm):
    """float64 (d/dyd, d/dy) of <gp, a> + <gt, a_dot> for a = lrelu(IN(y)), a_dot its tangent along yd, by torch.func's
    reverse mode over its forward mode (rows of (C, n, P)); gt / gp here are the adjoints BEFORE the slope"""
    def norm(t):
        if not in_norm:
            return t
        m = t.mean(-1, keepdim=True)
        var = (t - m).square().mean(-1, keepdim=True)
        return (t - m) / torch.sqrt(var + de.IN_EPS)

    def loss(y, yd):
        z, zd = torch.func.jvp(norm, (y,), (yd,))
        slope = torch.where(z > 0, 1.0, dp.SLOPE).detach()
        return (gp * z * slope).sum() + (gt * zd * slope).sum()
    d_y, d_yd = torch.func.grad(loss, argnums=(0, 1))(y, yd)
    return d_yd, d_y, norm(y)


@pytest.mark.parametrize("in_norm", [True, False])
def test_fold2_closed_form_matches_autograd(in_norm):
    """the kernel's formula, with gt / gp / yd at distinct exponents and out_p aligned at the tangent's, equals the
    double backward of InstanceNorm -> LeakyReLU"""
    g = torch.Generator().manual_seed(3)
    C, n, P = 5, 3, 37
    d = torch.float64
    y = torch.randn(C, n, P, generator=g, dtype=d) * 3 + 0.5
    yd = torch.randn(C, n, P, generator=g, dtype=d)
    gt_raw = torch.randn(C, n, P, generator=g, dtype=d)
    gp_raw = torch.randn(C, n, P, generator=g, dtype=d)
    d_yd, d_y, z = autograd_in_lrelu(gt_raw, gp_raw, y, yd, in_norm)
    slope = torch.where(z > 0, 1.0, dp.SLOPE)
    mean = rstd = tmean = tq = None
    if in_norm:
        mean = y.mean(-1)
        rstd = 1.0 / torch.sqrt((y - mean.unsqueeze(-1)).square().mean(-1) + de.IN_EPS)
        tmean = yd.mean(-1)
        zz = (y - mean.unsqueeze(-1)) * rstd.unsqueeze(-1)
        tq = (zz * (yd - tmean.unsqueeze(-1))).mean(-1)
    # the kernel's operands carry exponents: gt at gt_in, gp at eg, yd at ev; out_p is written at ex = gt_in + ev
    gt_in, eg, ev = -7, 11, 5
    ex = gt_in + ev
    ot, op, eo, _, _ = dp.in_lrelu_adjoint(slope * gt_raw * 2.0 ** -gt_in, slope * gp_raw * 2.0 ** -eg, y, mean, rstd,
                                           yd * 2.0 ** -ev, tmean if tmean is None else tmean * 2.0 ** -ev, tq, eg, ex)
    if not in_norm:
        assert eo == eg
        assert torch.allclose(op * 2.0 ** eo, d_y, rtol=1e-12, atol=0)
        assert torch.allclose(ot * 2.0 ** gt_in, d_yd, rtol=1e-12, atol=0)
        return
    assert eo == ex
    # tq is mean(z yc): the tangent's exponent scales it too
    ot, op, eo, _, _ = dp.in_lrelu_adjoint(slope * gt_raw * 2.0 ** -gt_in, slope * gp_raw * 2.0 ** -eg, y, mean, rstd,
                                           yd * 2.0 ** -ev, tmean * 2.0 ** -ev, tq * 2.0 ** -ev, eg, ex)
    assert rel_l2(ot * 2.0 ** gt_in, d_yd) <= 1e-12
    assert rel_l2(op * 2.0 ** ex, d_y) <= 1e-12
    # each sub-term matters: dropping it or flipping its sign moves out_p far off
    for k in dp.CROSS_TERMS:
        for defect in (dict(drop=k), dict(flip=k)):
            bad = dp.in_lrelu_adjoint(slope * gt_raw * 2.0 ** -gt_in, slope * gp_raw * 2.0 ** -eg, y, mean, rstd,
                                      yd * 2.0 ** -ev, tmean * 2.0 ** -ev, tq * 2.0 ** -ev, eg, ex, **defect)[1]
            assert rel_l2(bad * 2.0 ** ex, d_y) > 1e-3, defect


# --------------------------------------------------------------------------------------------------------------------
# the emulation against the oracle and the golden file
# --------------------------------------------------------------------------------------------------------------------
def weights(imsize, seed):
    torch.manual_seed(seed)
    D = Discriminator(False, "color,cutout", imsize=imsize)
    return ([m.weight_orig.detach().clone() for m in D.convs()], [m.weight_u.clone() for m in D.convs()],
            [m.weight_v.clone() for m in D.convs()])


def draws(n, h, w):
    """saturation factors 0 / 1 / 2 / 0.5, contrast 1.5 / 0.5 / 1.25 / 0.9, the cutout at the clamped right edge, the
    bottom-left corner, the interior and the top-left corner"""
    rb = torch.tensor([0.3, 0.7, 0.55, 0.2][:n])
    rs = torch.tensor([0.0, 0.5, 1.0, 0.25][:n])
    rc = torch.tensor([1.0, 0.0, 0.75, 0.4][:n])
    oy = torch.tensor([h // 2, h - 1, h // 3, 0][:n])
    ox = torch.tensor([w, 0, w // 2, 0][:n])
    return rb, rs, rc, oy, ox


def oracle(Ws, us, vs, x, imsize, training, aug, c):
    """float64 reg and the gradients of <c, reg> (compute_grad2's double backward)"""
    w2 = [w.double().clone().requires_grad_(True) for w in Ws]
    xo = x.double().clone().requires_grad_(True)
    out, *_ = do.forward(w2, [u.double() for u in us], [v.double() for v in vs], xo, imsize, training,
                         None if aug is None else tuple(t.double() if t.is_floating_point() else t for t in aug))
    (g,) = torch.autograd.grad(out.sum(), xo, create_graph=True)
    reg = g.pow(2).flatten(1).sum(1)
    (reg * c.double()).sum().backward()
    return reg.detach(), xo.grad, [w.grad for w in w2]


def run(imsize, h, w, n, mode, aug, d_reg, seed=0, training=True, x=None, Wuv=None):
    Ws, us, vs = weights(imsize, seed) if Wuv is None else Wuv
    if x is None:
        x = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed))
    a = draws(n, h, w) if aug is True else aug or None
    fwd = dp.emulate_penalty_forward(imsize, Ws, us, vs, x, training, a, mode)
    b = dp.emulate_penalty_backward(dict(fwd), Ws, d_reg, mode)
    return dict(b=b, fwd=fwd, Ws=Ws, us=us, vs=vs, x=x, aug=a, d_reg=d_reg)


def e2e(R, want):
    """rel-L2 of the emulated reg, input gradient and worst weight gradient against the oracle's"""
    b = R["b"]
    return {"reg": rel_l2(b["reg"], want[0]), "dx": rel_l2(b["pd_input"], want[1]),
            "dw": max(rel_l2(b[f"pdW{i}"], wt) for i, wt in enumerate(want[2]))}


@pytest.mark.parametrize("imsize,h,w", [(64, 64, 64), (-1, 63, 84), (32, 33, 47)])
@pytest.mark.parametrize("aug", [False, True])
def test_emulation_chains_to_the_oracle(imsize, h, w, aug):
    """the stage references, chained, are compute_grad2's double backward (an index, sign or exponent slip in a
    reference gives errors of order 1); d_reg spread over the images by 2^8"""
    d_reg = torch.tensor([10.0 / 3 * 2.0 ** 8, 10.0 / 3, 10.0 / 3 * 2.0 ** -8])
    R = run(imsize, h, w, 3, "split", aug, d_reg)
    e = e2e(R, oracle(R["Ws"], R["us"], R["vs"], R["x"], imsize, True, R["aug"], d_reg))
    print(f"penalty emulation vs oracle {imsize} {h}x{w} aug={aug}: " + " ".join(f"{k} {v:.1e}" for k, v in e.items()))
    assert e["reg"] <= 1e-4 and e["dx"] <= 1e-3 and e["dw"] <= 1e-3, e


@pytest.mark.parametrize("imsize,H,W,B,fire", [(64, 64, 64, 2, True), (-1, 56, 70, 1, False), (32, 32, 32, 2, True)])
def test_emulation_matches_golden(imsize, H, W, B, fire):
    """the emulated split-mode penalty against the reference module's own double backward (the golden file)"""
    gold = np.load(GOLDEN)
    name = case_name(imsize, H, W, B, fire)
    seed = int(gold[f"{name}/meta"][5])
    x, c = inputs(seed, B, H, W)
    aug = None
    if fire:
        dr = gold[f"{name}/draws"]
        aug = tuple(torch.from_numpy(dr[k]).float() for k in range(3)) + tuple(
            torch.from_numpy(dr[k]).long() for k in (3, 4))
    R = run(imsize, H, W, B, "split", aug, c.float(), seed=seed, x=x.float(), Wuv=weights(imsize, seed))
    b = R["b"]
    errs = {"reg": rel_l2(b["reg"], torch.from_numpy(gold[f"{name}/reg"])),
            "dx": rel_l2(b["pd_input"].reshape(-1)[torch.from_numpy(gold[f"{name}/dx_idx"])],
                         torch.from_numpy(gold[f"{name}/dx_sample"]))}
    errs["dw"] = max(rel_l2(b[f"pdW{i}"].reshape(-1)[torch.from_numpy(gold[f"{name}/sample_idx"][i])],
                            torch.from_numpy(gold[f"{name}/dw_sample"][i])) for i in range(len(b["layers"])))
    print(f"penalty emulation vs golden {name}: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert errs["reg"] <= 1e-4 and errs["dx"] <= 1e-2 and errs["dw"] <= 1e-2, errs


# --------------------------------------------------------------------------------------------------------------------
# planted defects
# --------------------------------------------------------------------------------------------------------------------
IMSIZE, H, W, N = 64, 64, 64, 3
D_REG = torch.tensor([10.0 / 3 * 2.0 ** 5, 10.0 / 3, 10.0 / 3 * 2.0 ** -3])


@pytest.fixture(scope="module")
def em():
    """the 64 branch at 64 x 64, three augmented images, per mode: the emulated penalty's buffers, and the oracle"""
    R = {m: run(IMSIZE, H, W, N, m, True, D_REG, seed=1) for m in de.MODES}
    s = R["split"]
    return R, oracle(s["Ws"], s["us"], s["vs"], s["x"], IMSIZE, True, s["aug"], D_REG)


def caught(stage, mode, y_bad, ref, scale):
    w, r = de.stats(de.err(y_bad.float(), ref, scale))
    bw, br = dp.PEN_BARS[mode][stage]
    print(f"planted penalty defect in {stage} ({mode}): worst {w:.2e} rms {r:.2e} (bars {bw:.0e} {br:.0e})")
    return w > bw or r > br


def stage_view(b, defect, mode):
    """the correct reference of the stage that sees `defect`, from the defective chain's kernel-side inputs, and the
    defective value: (stage, bad value, ref, scale), or (None, exact-check outcome) for a defect an exact check sees"""
    name, arg = defect
    L = b["layers"]
    if name in ("cross_drop", "cross_flip", "p_start_one"):   # the fold into layer 2's output (q = 2), or the top
        i = 3 if name != "p_start_one" else len(L) - 1
        q = i - 1
        ts = b[f"pt{i}"]
        ps = b[f"pp{i}"]
        dcol_t = de.dgrad_ref(ts, b[f"ws{i}"], b["alpha"][i], mode)[0].float()
        dcol_p = None if ps is None else de.dgrad_ref(ps, b[f"ws{i}"], b["alpha"][i], mode)[0].float()
        args = (L, i, dcol_t, dcol_p, b[f"y{q}"], b[f"mean{q}"], b[f"rstd{q}"], b[f"ty{q}"], b[f"tmean{q}"],
                b[f"tq{q}"], b["gt"][i], b["gp"][i] if ps is not None else None, b["ev"][q])
        if name == "p_start_one":   # the correct chain has no primal adjoint at the top
            ref = dp.fold2_ref(*args[:3], None, *args[4:11], None, args[12])
            bad = dp.fold2_ref(*args)
        else:
            ref = dp.fold2_ref(*args)
            bad = dp.fold2_ref(*args, **{name.split("_")[1]: arg})
        return "fold2_p", bad[1], ref[1], ref[4]
    if name in ("taug_shift", "taug_mean") and not (name == "taug_mean" and arg == "unsat"):
        aug_ws = torch.zeros(N, de.AUG_FLOATS)
        aug_ws[:, :4], aug_ws[:, 4], aug_ws[:, 5:9] = b["aug_f"], b["aug_mean"], b["box"].float()
        tf, box = dp.taug_words(aug_ws)
        tm = dp.taug_mean_ref(b["vt"], tf[:, 2])[0]
        ref, mag, _ = de.gather0_ref(L, b["vt"], tf, tm, box)
        return "tgather0", b["tcol0"], ref, mag * 2.0 ** -24
    if name == "taug_mean":
        ref, sc = dp.taug_mean_ref(b["vt"], b["aug_f"][:, 2])
        return "taug_mean", b["taug_mean"], ref, sc
    if name == "ev_off":   # tcol{arg} read at the exponent ev[arg]
        i = arg - 1
        zs, sc = dp.zdot_ref(b[f"ty{i}"], b[f"y{i}"], b[f"mean{i}"], b[f"rstd{i}"], b[f"tmean{i}"], b[f"tq{i}"])
        f = 2.0 ** (b["ev"][i] - b["ev"][arg])
        nv = de.normalized(b[f"y{i}"], b[f"mean{i}"], b[f"rstd{i}"]).transpose(0, 1)
        sl = torch.where(nv > 0, 1.0, dp.SLOPE).double()
        y = L[arg]
        shape = (y["n"], L[i]["cout"], y["hin"], y["win"])
        ref = de.unfold((zs * f * sl).transpose(0, 1).reshape(shape).contiguous(), y)
        scale = de.unfold((sc * f * sl).transpose(0, 1).reshape(shape).contiguous(), y)
        return "zdot", b[f"tcol{arg}"], ref, scale
    if name == "alpha_p":
        i = 2
        ref, _, sc = de.dgrad_ref(b[f"pp{i}"], b[f"ws{i}"], b["alpha"][i], mode)
        bad = de.dgrad_ref(b[f"pp{i}"], b[f"ws{i}"], b["alpha"][i], mode, alpha_times=2)[0]
        return "dgrad_p", bad, ref, sc
    if name == "dwp_no_cs":
        i = 2
        ref, _, sc = de.wgrad_ref(b[f"pp{i}"], b[f"col{i}"], de.col_scale(L, i), mode)
        return "wgrad_p", b[f"dwp{i}"], ref, sc
    if name == "combine_smaller":   # gw must be the larger of the two streams' exponents, exactly
        return None, all(b[f"gw{i}"] == max(b["gt"][i] + b["ev"][i], b["gp"][i]) for i in range(len(L) - 1))
    raise AssertionError(name)


DEFECTS = ([("cross_drop", k) for k in dp.CROSS_TERMS] + [("cross_flip", k) for k in dp.CROSS_TERMS] +
           [("taug_mean", "primal"), ("taug_shift", None), ("ev_off", 2), ("combine_smaller", None),
            ("alpha_p", None), ("dwp_no_cs", None), ("p_start_one", None)])


def defect_id(d):
    return d[0] if d[1] is None else f"{d[0]}-{d[1]}"


@pytest.mark.parametrize("defect", DEFECTS, ids=defect_id)
@pytest.mark.parametrize("mode", list(de.MODES))
def test_bars_catch_planted_defects(em, mode, defect):
    R, want = em
    s = R[mode]
    bad = dict(s, b=dp.emulate_penalty_backward(dict(s["fwd"]), s["Ws"], D_REG, mode, defect))
    view = stage_view(bad["b"], defect, mode)
    if mode == "split":
        e, e0 = e2e(bad, want), e2e(s, want)
        seen = e["reg"] > E2E_BARS[0] or max(e["dx"], e["dw"]) > E2E_BARS[1]
        print(f"planted penalty defect {defect_id(defect)}: end to end rel-L2 reg {e['reg']:.1e} dx {e['dx']:.1e} "
              f"dw {e['dw']:.1e} (defect-free {e0['dx']:.1e} {e0['dw']:.1e}; test_gpu_disc_penalty.py bars "
              f"{E2E_BARS[0]:.0e} / {E2E_BARS[1]:.0e}: {'seen' if seen else 'MISSED'})")
    if view[0] is None:
        assert not view[1], defect
    else:
        assert caught(view[0], mode, *view[1:]), defect


def test_unsaturated_tangent_mean_is_not_a_defect(em):
    """saturation keeps every pixel's channel mean, so the contrast mean over the saturated tangent equals the mean over
    the unsaturated one in exact arithmetic: taking it over the unsaturated tangent changes rounding only"""
    b = em[0]["split"]["b"]
    sat = b["aug_f"][:, 2]
    a, sc = dp.taug_mean_ref(b["vt"], sat)
    u, _ = dp.taug_mean_ref(b["vt"], sat, "unsat")
    assert float(((a - u).abs() / sc).max()) < 1e-12
