"""The patch-loss stage harness tested without a GPU: the checkers of tests/test_gpu_patch_loss_stages.py run on the CPU
stand-in of tests/patch_loss_emulation.py.  The faithful stand-in passes every checker; with one planted defect at a
time the checker that is there for it fails, while the assertions tests/test_gpu_patch_loss.py holds (loss within 1e-5
relative, gradients within 1e-4 rel-L2 and max|diff| / max|ref|), restated here on the same inputs, miss the defects
marked in CATCH.  The float64 references are tied to tests/patch_loss_oracle.py: the closed-form coefficient maps to
its autograd with respect to mu1, f(x^2) and f(xy), the adjoint to an explicitly built reflect-pad matrix."""
import numpy as np
import pytest
import torch

from tests import patch_loss_emulation as emu
from tests import patch_loss_oracle as plo
from tests import test_gpu_patch_loss_stages as st
from tests._common import assert_close

f32 = np.float32
OK = emu.StandIn()
CPU = "cpu"


def fails(fn, *a, **k):
    try:
        fn(*a, **k)
    except AssertionError:
        return True
    return False


# ------------------------------------------------------------------------------------------------ faithful stand-in
@pytest.mark.parametrize("hw", st.SHAPES[::3] + ((17, 33), (33, 17)), ids=lambda s: f"{s[0]}x{s[1]}")
def test_faithful_ssim(hw):
    H, W = hw
    for k, kind in enumerate(st.SSIM_KINDS):
        B, Cc = st._bc(H + W + k)
        x, y, mv, eps = st.ssim_case(kind, B, Cc, H, W, CPU, k)
        lay = st.LAYOUTS[(H + k) % len(st.LAYOUTS)]
        x, y = st.place(x, lay if lay != "expand" else "nchw"), st.place(y, lay)
        coef = st.check_ssim_forward(OK, x, y, mv, eps, f"{kind} {lay}")
        st.check_ssim_backward(OK, x, y, coef, f"{kind} {lay}")


@pytest.mark.parametrize("hw", ((6, 7), (11, 10), (17, 33), (33, 64)), ids=lambda s: f"{s[0]}x{s[1]}")
def test_faithful_injected_maps(hw):
    H, W = hw
    x, y = torch.rand(121, 1, H, W), torch.rand(121, 1, H, W)
    st.check_ssim_backward(OK, x, y, st.lattice_maps(121, 1, H, W, CPU), "lattice")
    x, y = torch.rand(2, 3, H, W), torch.rand(2, 3, H, W)
    st.check_ssim_backward(OK, st.place(x, "crop"), y, torch.randn(3, 2, 3, H, W, dtype=torch.float64), "random")


def test_faithful_smoothness_caps_scratch_and_non_finite():
    for H, W in ((2, 2), (6, 7), (17, 33), (64, 84)):
        for kind in ("depth", "far_depth"):
            d, img = st.smooth_case(kind, 2, 3, H, W, CPU, H)
            st.check_smooth(OK, st.place(d, "rays"), st.place(img, "crop"), kind)
    B, Cc, H, W = st.past_smooth_caps(OK)
    st.check_smooth(OK, *st.smooth_case("depth", B, Cc, H, W, CPU, 2), "past the caps", scales=False)
    x, y, _, _ = st.ssim_case("rgb", 1, 3, 40, 40, CPU, 4)
    d, i = st.smooth_case("depth", 1, 3, 40, 40, CPU, 6)
    st.check_scratch(OK, [lambda ws: st.ssim_loss_call(OK, x, y, ws), lambda ws: st.smooth_loss_call(OK, d, i, ws)])
    st.check_nonfinite(OK)


def test_faithful_ssim_past_the_launch_caps():
    B, Cc, H, W = st.past_ssim_caps(OK)
    x, y, mv, eps = st.ssim_case("rgb", B, Cc, H, W, CPU, 1)
    st.check_ssim_forward(OK, x, y, mv, eps, "past the caps")


# ------------------------------------------------------------------------------------------------ planted defects
def old_assertions(impl):
    """tests/test_gpu_patch_loss.py::test_smoothness_vs_float64 and ::test_ssim_rgb_vs_float64 restated on the
    implementation, NCHW, with their inputs and bars."""
    ws = lambda: torch.zeros(emu.LOSS_WS_FLOATS)
    for B, H, W in ((1, 64, 64), (1, 63, 84), (1, 56, 70), (2, 64, 64), (1, 2, 2)):
        g = torch.Generator().manual_seed(H * W + B)
        d = torch.rand(B, 1, H, W, generator=g) * 4 + 2
        img = torch.rand(B, 3, H, W, generator=g)
        img[:, :, : H // 2, : W // 3] = 1.0
        d[:, :, H // 3:, W // 2:] = 3.5
        loss, gd, gi = torch.zeros(()), torch.zeros_like(d), torch.zeros_like(img)
        impl.smooth_forward(d, img, loss, ws())
        impl.smooth_backward(d, img, torch.ones(1), gd, gi)
        r = emu.smooth64(d, img)
        assert abs(float(loss) - float(r["loss"])) <= 1e-5 * abs(float(r["loss"]))
        assert_close(gd, r["g_d"], 1e-4, "g_idepth")
        assert_close(gi, r["g_img"], 1e-4, "g_image")
    for B, H, W in ((1, 64, 64), (1, 63, 84), (1, 56, 70), (2, 64, 64), (1, 6, 7)):
        for Cc in (3, 1):
            g = torch.Generator().manual_seed(H * W + Cc)
            x = torch.rand(B, Cc, H, W, generator=g)
            y = (x + 0.2 * torch.rand(B, Cc, H, W, generator=g)).clamp(0, 1)
            x[:, :, : H // 3, : W // 2] = 1.0
            y[:, :, : H // 3, : W // 2] = 1.0
            loss, coef, gx = torch.zeros(()), torch.zeros(3 * x.numel(), dtype=torch.float64), torch.zeros_like(x)
            impl.ssim_forward(x, y, 1.0, 1e-12, loss, coef, ws())
            impl.ssim_backward(x, y, coef, torch.ones(1), gx)
            xr = x.double().requires_grad_(True)
            ref = plo.ssim_loss(xr, y.double(), 11)
            (rg,) = torch.autograd.grad(ref, xr)
            assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
            assert_close(gx, rg, 1e-4, "g_img1")


def _lattice(impl, H, W):
    x, y = torch.rand(121, 1, H, W, generator=torch.Generator().manual_seed(1)), torch.rand(121, 1, H, W)
    st.check_ssim_backward(impl, x, y, st.lattice_maps(121, 1, H, W, CPU), "lattice")


def _forward(kind, B, Cc, H, W):
    def run(impl):
        x, y, mv, eps = st.ssim_case(kind, B, Cc, H, W, CPU, 3)
        st.check_ssim_forward(impl, x, y, mv, eps, kind)
    return run


def _random_maps(impl):
    x, y = torch.rand(2, 3, 12, 40), torch.rand(2, 3, 12, 40)
    st.check_ssim_backward(impl, x, y, torch.randn(3, 2, 3, 12, 40, dtype=torch.float64), "random maps")


def _smooth(impl):
    d, img = st.smooth_case("depth", 2, 3, 12, 17, CPU, 1)
    st.check_smooth(impl, d, img, "smooth")


def _past_caps(impl):
    B, Cc, H, W = st.past_ssim_caps(impl)
    x, y, mv, eps = st.ssim_case("rgb", B, Cc, H, W, CPU, 1)
    st.check_ssim_forward(impl, x, y, mv, eps, "past the caps")


CATCH = {   # defect -> (the new check that must fail, whether the restated old assertions miss it)
    "mirror_q1": (lambda i: _lattice(i, 12, 12), False),
    "mirror_n6": (lambda i: _lattice(i, 12, 12), False),
    "halo_shift": (_forward("rgb", 1, 3, 16, 40), False),
    "taps_fp32": (_forward("depth", 1, 1, 16, 16), True),
    "coef_next_plane": (_random_maps, False),
    "strict_gate": (_forward("identical_eps0", 1, 1, 24, 24), True),
    "last_tile_skipped": (_past_caps, True),
    "clamp_swallows_nan": (st.check_nonfinite, True),
    "sign0_is_1": (_smooth, False),
    "no_inv_c": (_smooth, False),
    "ticket_not_reset": (_smooth, True),
}


def test_every_defect_has_a_check():
    assert set(CATCH) == set(emu.DEFECTS)


@pytest.mark.parametrize("defect", emu.DEFECTS)
def test_planted_defect_is_caught(defect):
    new, old_misses = CATCH[defect]
    assert fails(new, emu.StandIn(defect)), f"{defect}: the stage check did not notice"
    new(OK)
    if old_misses:
        assert not fails(old_assertions, emu.StandIn(defect)), f"{defect}: the earlier assertions already catch this"


def test_old_assertions_pass_on_the_faithful_stand_in():
    old_assertions(OK)


def test_which_defects_the_old_assertions_catch():
    """Reported with -s: which planted defects tests/test_gpu_patch_loss.py's assertions would have noticed."""
    caught = [d for d in emu.DEFECTS if fails(old_assertions, emu.StandIn(d))]
    print("defects the earlier patch-loss assertions catch:", ", ".join(caught))
    assert set(caught) == {d for d, (_, miss) in CATCH.items() if not miss}


# ------------------------------------------------------------------------------------------------ the references
def test_closed_form_coefficients_match_oracle_autograd(monkeypatch):
    """emu.ssim64's coefficient maps == float64 autograd of plo.ssim_loss with mu1, f(x^2), f(xy) as the leaves."""
    for kind, eps in (("rgb", 1e-12), ("depth", 1e-12), ("max_val", 1e-6), ("identical_eps0", 0.0)):
        x, y, mv, _ = st.ssim_case(kind, 2, 3, 13, 21, CPU, 9)
        r = emu.ssim64(x, y, mv, eps)
        X, Y = x.double(), y.double()
        maps = [emu._filter(t).detach() for t in (X, Y, X * X, Y * Y, X * Y)]
        leaves = [maps[0].requires_grad_(True), maps[1], maps[2].requires_grad_(True), maps[3],
                  maps[4].requires_grad_(True)]
        it = iter(leaves)
        monkeypatch.setattr(plo, "filter2d", lambda t, k: next(it))
        loss = plo.ssim_loss(X, Y, 11, mv, eps)
        monkeypatch.undo()
        auto = torch.autograd.grad(loss, [leaves[0], leaves[2], leaves[4]])
        assert abs(float(loss) - float(r["loss"])) <= 1e-15
        for m in range(3):
            err = ((auto[m] - r["coef"][m]).abs() / (r["coef_bound"][m] + 1e-300)).max()
            assert float(err) <= 1e-14, (kind, m, float(err))
        assert bool((r["coef"].abs() <= r["coef_bound"] * (1 + 1e-12)).all())


@pytest.mark.parametrize("n", (6, 7, 11, 17, 33))
def test_adjoint_is_the_transpose_of_the_reflect_filter(n):
    """adjoint64 against the matrix of reflect-pad + correlate built from its definition, index by index."""
    g = plo.gaussian_1d(11, 1.5).numpy()
    refl = lambda k, m: -k if k < 0 else (2 * (m - 1) - k if k >= m else k)
    Mh, Mw = np.zeros((n, n)), np.zeros((n + 3, n + 3))
    for M_, m in ((Mh, n), (Mw, n + 3)):
        for p in range(m):
            for k in range(-5, 6):
                M_[p, refl(p + k, m)] += g[k + 5]
    c = torch.randn(3, 1, 2, n, n + 3, dtype=torch.float64)
    x, y = torch.rand(1, 2, n, n + 3), torch.rand(1, 2, n, n + 3)
    got, bound = emu.adjoint64(c, x, y)
    A = [np.einsum("pi,bcpq,qj->bcij", Mh, c[m].numpy(), Mw) for m in range(3)]
    want = A[0] + 2 * x.double().numpy() * A[1] + y.double().numpy() * A[2]
    assert np.abs(got.numpy() - want).max() <= 1e-14 * bound.numpy().max()
    assert bool((got.abs() <= bound * (1 + 1e-12)).all())


def test_smoothness_reference_bounds():
    d, img = st.smooth_case("depth", 2, 3, 9, 13, CPU, 4)
    r = emu.smooth64(d, img)
    assert float(r["loss_bound"]) == pytest.approx(float(r["loss"]), rel=1e-15)
    assert bool((r["g_d"].abs() <= r["g_d_bound"] * (1 + 1e-12)).all())
    assert bool((r["g_img"].abs() <= r["g_img_bound"] * (1 + 1e-12)).all())


def test_launch_geometry_crosses_every_cap():
    B, Cc, H, W = st.past_ssim_caps(OK)
    n = emu.ssim_tiles(B, Cc, H, W)
    assert n > emu.MAX_LOSS_BLOCKS == 2046 and n > 8 * OK.sm_count
    B, Cc, H, W = st.past_smooth_caps(OK)
    assert B * H * W > 2046 * 256 and B * H * W > 16 * OK.sm_count * 256
