"""The ray-stage harness tested without a GPU: the checkers of tests/test_gpu_ray_stages.py run on the CPU stand-in
of tests/ray_emulation.py.  The faithful stand-in passes every checker; with one planted defect at a time the checker
that is there for it fails, while the assertions the suite held before (whole-tensor rel-L2 at 1e-5 / 1e-4, "at most 8
samples a bin away"), restated here on the same data, do not notice.  The float64 truth and the float32 emulation are
tied to oracle/render_oracle.py and to the reference-generated fixtures of tests/golden/stages.npz."""
import numpy as np
import pytest
import torch

from oracle import render_oracle as orc
from tests import ray_emulation as emu
from tests import test_gpu_ray_stages as st
from tests._common import load_npz, rel_l2

f32 = np.float32
OK = emu.StandIn()


def fails(fn, *a, **k):
    try:
        fn(*a, **k)
    except AssertionError:
        return True
    return False


# ------------------------------------------------------------------------------------------------ faithful stand-in
@pytest.mark.parametrize("S", st.S_ALL)
def test_faithful_composite(S):
    quad = S % 4 == 0 and 4 <= S <= 128
    for cfg in st.CONFIGS:
        for n in st.ray_counts(OK, S, quad)[:2] + [9]:
            st.check_composite(OK, S, n, cfg)


def test_faithful_offset_views_degenerate_losses_amax():
    st.check_offset_views(OK)
    st.check_degenerate(OK)
    for S in (8, 30, 64, 128, 132):
        for mode in ("scalar", "per_ray", "rgb_only", "depth_only"):
            st.check_losses(OK, S, 21, mode)
        st.check_losses(OK, S, 5, "per_ray", g_loss=(0.37, -2.5), wb=False)
        st.check_amax(OK, S, 21)
    st.check_amax(OK, 64, 1)


@pytest.mark.parametrize("M", (1, 2, 31, 32, 33, 62, 126, 254))
def test_faithful_sample_pdf(M):
    for Ni in (1, 5, 32, 64, 100):
        st.check_sample_pdf(OK, M, Ni, shared_u=True)
        st.check_sample_pdf(OK, M, Ni, shared_u=False)


@pytest.mark.parametrize("kind", ("linspace", "random", "one_swap", "ties", "coarse_tie", "general"))
def test_faithful_merge(kind):
    for S in (3, 4, 17, 33, 34, 64, 128):
        for Ni in (1, 5, 16, 64, 100, 256):
            st.check_merge(OK, S, Ni, kind, n=6)


# ------------------------------------------------------------------------------------------------ planted defects
def old_composite_assertions(impl):
    """tests/test_gpu_parity.py::test_composite_known_answer_and_oracle and test_gpu_backward.py's compositing test,
    restated: 77 rays, sigma = 30 randn, whole-tensor rel-L2 against the float32 oracle."""
    g = torch.Generator().manual_seed(11)
    for S in (2, 4, 31, 36, 64, 96, 100, 128, 132):
        n = 77
        rays = torch.randn(n, 8, generator=g)
        z = torch.sort(torch.rand(n, S, generator=g) * 4 + 2, -1)[0]
        raw = torch.randn(n, S, 4, generator=g)
        raw[..., 3] = raw[..., 3] * 30
        raw[..., :3] = torch.rand(n, S, 3, generator=g)
        noise = torch.randn(n, S, generator=g)
        ref = orc.composite(raw[..., 3], z, torch.norm(rays[:, 3:6].unsqueeze(1), dim=-1), raw[..., :3], noise * 0.7, True)
        got = impl.composite_forward(raw, 4, z, rays, noise, 0.7, True)
        for a, b in zip(got, ref):
            assert rel_l2(a, b) <= 1e-5
        r = raw.clone().requires_grad_(True)
        o = orc.composite(r[..., 3], z, torch.norm(rays[:, 3:6].unsqueeze(1), dim=-1), r[..., :3], noise * 0.7, True)
        gr, gd, gw = torch.randn(n, 3, generator=g), torch.randn(n, generator=g), torch.randn(n, S, generator=g)
        ((o[0] * gr).sum() + (o[1] * gd).sum() + (o[2] * gw).sum()).backward()
        assert rel_l2(impl.composite_backward(raw, 4, z, rays, noise, 0.7, True, gr, gd, gw), r.grad) <= 1e-4


def old_pdf_assertions(impl):
    """tests/test_gpu_parity.py::test_sample_pdf_known_answers_and_golden restated on the stages.npz fixture."""
    ST = load_npz("stages.npz")
    b, w = torch.from_numpy(ST["pdf_bins"]), torch.from_numpy(ST["pdf_w"])
    width = float((b[:, 1:] - b[:, :-1]).max())
    for u, key in ((torch.linspace(0, 1, 64), "pdf_det_out"), (torch.from_numpy(ST["pdf_rand_u"]), "pdf_rand_out")):
        diff = (impl.sample_pdf(b, w, u.contiguous()) - torch.from_numpy(ST[key])).abs()
        assert int((diff > 2e-5).sum()) <= 8 and float(diff.max()) <= width * 1.001


def old_merge_assertions(impl):
    """tests/test_gpu_round2.py::test_importance_merge_general_path_matches_torch_sort restated: the order of whatever
    z_new the implementation itself produced, on random weights."""
    z, w, u = st.merge_inputs(64, 64, "random", 16, 1)
    fine, new = impl.importance_merge(torch.from_numpy(z), torch.from_numpy(w), torch.from_numpy(u))
    assert torch.equal(fine, torch.sort(torch.cat([torch.from_numpy(z), new], 1), 1)[0])


CATCH = {   # defect -> (the new check that must fail, the restated old assertions that must not)
    "search_lt": (lambda i: st.check_sample_pdf(i, 32, 64, shared_u=False), old_pdf_assertions),
    "above_clamp": (lambda i: st.check_sample_pdf(i, 32, 64, shared_u=False), None),
    "denom_le": (lambda i: st.check_sample_pdf(i, 1, 5, shared_u=False), old_pdf_assertions),
    "merge_lt": (lambda i: st.check_merge(i, 64, 16, "coarse_tie"), old_merge_assertions),
    "rank_no_tiebreak": (lambda i: st.check_merge(i, 33, 16, "ties"), old_merge_assertions),
    "last_delta_no_dnorm": (lambda i: st.check_composite(i, 64, 9, st.CONFIGS[0]), None),
    "quad_scan_gt": (lambda i: st.check_composite(i, 64, 9, st.CONFIGS[0]), None),
    "quad_tail_kept": (lambda i: st.check_composite(i, 64, 9, st.CONFIGS[0]), old_composite_assertions),
    "warp_no_carry_step2": (lambda i: st.check_composite(i, 132, 9, st.CONFIGS[0]), None),
    "warp_suffix_late": (lambda i: st.check_composite(i, 132, 9, st.CONFIGS[0]), None),
    "warp_mse_no_2": (lambda i: st.check_losses(i, 132, 21, "scalar"), None),
    "amax_no_gw": (lambda i: st.check_amax(i, 64, 21), None),
    "ticket_not_reset": (lambda i: st.check_losses(i, 64, 21, "scalar"), None),
    "second_trip_cdf": (lambda i: st.check_sample_pdf(i, 62, 64, shared_u=False), None),
}


def test_every_defect_has_a_check():
    assert set(CATCH) == set(emu.DEFECTS)


@pytest.mark.parametrize("defect", emu.DEFECTS)
def test_planted_defect_is_caught(defect):
    new, old = CATCH[defect]
    assert fails(new, emu.StandIn(defect)), f"{defect}: the stage check did not notice"
    new(OK)
    if old is not None:
        old(OK)
        assert not fails(old, emu.StandIn(defect)), f"{defect}: the earlier assertions already caught this"


# ------------------------------------------------------------------------------------------------ truth and emulation
def test_truth_matches_oracle_and_closed_form():
    sc = st.scene(33, 36, 3, "cpu")
    dn = sc["rays"][:, 3:6].norm(dim=1)
    for wb in (False, True):
        raw64 = sc["raw"].double().requires_grad_(True)
        c = emu.composite64(raw64, sc["z"], dn, sc["noise"], 0.7, wb)
        ref = orc.composite(sc["raw"][..., 3], sc["z"], dn[:, None], sc["raw"][..., :3], sc["noise"] * 0.7, wb)
        for a, b in zip((c["rgb"], c["depth"], c["weights"]), ref):
            assert float((a - b.double()).abs().max()) <= 2e-6
        G = [sc[k].double() for k in ("g_rgb", "g_depth", "g_w")]
        auto, = torch.autograd.grad((G[0] * c["rgb"]).sum() + (G[1] * c["depth"]).sum() + (G[2] * c["weights"]).sum(), raw64)
        c = {k: v.detach() for k, v in c.items()}
        closed = emu.g_raw_closed_form64(c, sc["raw"], sc["z"], wb, *G)
        bound = emu.g_raw_bound64(c, sc["raw"], sc["z"], wb, *G)
        assert float(((auto - closed).abs() / (bound + 1e-300)).max()) <= 1e-12
        assert bool((closed.abs() <= bound * (1 + 1e-12) + 1e-300).all())


def test_emulated_scan_is_a_cumsum_where_sums_are_exact():
    g = np.random.default_rng(0)
    for M in (1, 2, 31, 32, 33, 64, 100, 254):
        w = g.integers(0, 8, (5, M)).astype(f32)
        w[0] = 0
        pad = 2 ** int(np.ceil(np.log2(w.sum(1).max() + 8))) - w.sum(1)      # totals that are powers of two: exact quotients
        w[:, -1] += pad.astype(f32)
        cdf = emu.build_cdf32(w, 0.0)
        want = np.concatenate([np.zeros((5, 1)), np.cumsum(w.astype(np.float64), 1)], 1) / w.sum(1, keepdims=True, dtype=np.float64)
        assert np.array_equal(cdf.astype(np.float64), want), M


def test_emulation_matches_oracle_and_golden_fixtures():
    ST = load_npz("stages.npz")
    bins = torch.tensor([[0., 1., 2., 3., 4.]])
    for tag, w, n in (("ones", [1., 1., 1., 1.], 5), ("spike", [0., 0., 1., 0.], 5), ("zero", [0., 0., 0., 0.], 5),
                      ("ramp", [.1, .2, .3, .4], 8)):
        got = emu.sample_pdf32(bins.numpy(), np.array([w], f32), np.linspace(0, 1, n, dtype=f32))
        assert np.allclose(got, ST[f"pdf_kat_{tag}"], atol=2e-6), tag
    b, w = ST["pdf_bins"], ST["pdf_w"]
    width = float((b[:, 1:] - b[:, :-1]).max())
    for u, key in ((np.linspace(0, 1, 64, dtype=f32), "pdf_det_out"), (ST["pdf_rand_u"], "pdf_rand_out")):
        got = emu.sample_pdf32(b, w, u)
        knots = emu.knot_samples(w, u, ulps=4)
        diff = np.abs(got - ST[key])
        # the exceptional samples are named, not counted; 1e-4: a cdf rounded to 2^-24 divided by a bin's small cdf step
        assert float(diff[~knots].max()) <= 1e-4, key
        assert float(diff.max()) <= width * 1.001
        ref = orc.sample_pdf(torch.from_numpy(b), torch.from_numpy(w), 64, det=key == "pdf_det_out",
                             u=None if key == "pdf_det_out" else torch.from_numpy(u)).numpy()
        assert float(np.abs(got - ref)[~knots].max()) <= 1e-4
        assert float(np.abs(got - emu.sample_pdf64(b, w, u)[0])[~knots].max()) <= 1e-4
    z = np.sort(np.random.default_rng(1).random((4, 9)).astype(f32), 1)
    zn = np.random.default_rng(2).random((4, 5)).astype(f32)
    zn[0, 0] = z[0, 3]
    want = torch.sort(torch.cat([torch.from_numpy(z), torch.from_numpy(zn)], 1), dim=1, stable=True)[0].numpy()
    assert np.array_equal(emu.merge32(z, zn), want) and np.array_equal(emu.sort_like_torch(np.concatenate([z, zn], 1)), want)


# ------------------------------------------------------------------------------------------------ the C ABI on the host
def test_misaligned_raw_and_too_many_importance_samples_are_refused_before_any_launch():
    """raw (N,S,4) is read as 16-byte rows by every compositing kernel: a misaligned pointer is SNB_ERR_INVALID.  The
    pointers below are never dereferenced: the checks return before any CUDA call."""
    import ctypes as C
    from sinnerf_b200 import _lib, build
    build.build()
    lib = _lib.load()
    ok, off = C.c_void_p(0x10000), C.c_void_p(0x10004)
    assert lib.snb_composite_forward(off, 4, ok, ok, None, 0.0, 0, 4, 64, ok, ok, ok, None) == -1
    assert b"16-byte aligned" in lib.snb_last_error()
    assert lib.snb_composite_backward(off, ok, ok, None, 0.0, 0, ok, ok, None, 4, 64, ok, None) == -1
    assert lib.snb_composite_backward(ok, ok, ok, None, 0.0, 0, ok, ok, None, 4, 64, off, None) == -1
    spec = _lib.SnbLossSpec(ok, None, None, None, 1.0, 0.0)
    assert lib.snb_composite_forward_loss(off, ok, ok, None, 0.0, 0, 4, 64, C.byref(spec), ok, ok, ok, ok, ok, None) == -1
    assert lib.snb_composite_backward_loss(off, ok, ok, None, 0.0, 0, None, None, None, C.byref(spec), ok, ok, None, 4, 64,
                                           ok, None, None) == -1
    assert b"16-byte aligned" in lib.snb_last_error()
    assert lib.snb_importance_merge(ok, ok, ok, 0, 4, 64, 257, 1e-5, ok, None, None) == -3
    assert b"N_importance > 256" in lib.snb_last_error()
