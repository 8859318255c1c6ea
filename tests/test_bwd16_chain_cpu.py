"""The single-probe checkers of tests/bwd16_emulation.py on a CPU stand-in of the 16-bit training backward.

Every checker passes on the faithful stand-in (StandIn()) at probes placed like the GPU test's and fails on the
planted defect aimed at it; the aggregate per-tensor bars of tests/test_gpu_layerwise.py (bwd_bound against the
float64 chain) are restated on the same stand-in to show which defects they let through.
"""
import pytest
import torch

from oracle import render_oracle as orc
from tests import bwd16_emulation as em
from tests.test_gpu_layerwise import NAMES, bwd_bound, chain64, zero_grads

P = 4463                        # 140 tiles of 32: more tiles than a wgrad launch has slices, a ragged tail
LAYERS = em.LAYERS


def _forward(seed=1):
    """A training forward in float32 with its saves as act16 holds them (fp16 cells, masks from the fp32 signs)."""
    g = torch.Generator().manual_seed(seed)
    p = orc.default_init_params(1)
    xyz = (torch.rand(P, 3, generator=g) * 2 - 1) * 1.5
    d = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1)
    enc, dirs = orc.embed(xyz, orc.N_XYZ_FREQS).float(), orc.embed(d, orc.N_DIR_FREQS).float()
    H, M, h = [], [], enc
    for l in range(8):
        if l == 4:
            h = torch.cat([enc, h], 1)
        h = torch.relu(h @ p[LAYERS[l] + ".weight"].t() + p[LAYERS[l] + ".bias"])
        H.append(h.half().float())
        M.append(h > 0)
    feat = h @ p["xyz_encoding_final.weight"].t() + p["xyz_encoding_final.bias"]
    s = torch.cat([feat, dirs], 1) @ p["dir_encoding.0.weight"].t() + p["dir_encoding.0.bias"]
    G = torch.nn.functional.softplus(s - 1.0).half().float()
    rgb = 0.5 * (1.0 + 1.002 * torch.tanh(0.5 * (G @ p["rgb.0.weight"].t() + p["rgb.0.bias"])))
    raw = torch.cat([rgb, h @ p["sigma.weight"].t() + p["sigma.bias"]], 1)
    a = dict(enc=enc.half().float(), dir=dirs.half().float(), G=G, H=H, M=M)
    return p, a, raw


@pytest.fixture(scope="module")
def fwd():
    return _forward()


def probe_g(pt, vec):
    g = torch.zeros(P, 4)
    g[pt] = torch.tensor(vec)
    return g


def run(fwd, defect, pt, vec, sigma_only=False):
    p, a, raw = fwd
    g_raw = probe_g(pt, vec)
    si = em.StandIn(defect)
    if sigma_only:
        grads, ws = si.backward(p, a, None, raw, sigma_only=True, g_sigma=g_raw[:, 3])
    else:
        grads, ws = si.backward(p, a, g_raw, raw)
    return em.check_probe(grads, ws, p, a, raw, g_raw, pt, sigma_only)


# probes: first / last point, a tile seam, the last point of the second slice of a 2-block wgrad launch (the tile
# defect 8 skips), magnitudes 2^+-8, one sigma-only and one rgb-only
SL = em.slice_tiles((P + 127) // 128 * 4, 2)
PROBES = [(0, [0.3, -1.2, 0.7, 2.0]), (P - 1, [2.0 ** 8, -3.0, 1.0, -2.0 ** -8]), (127, [0.0, 0.0, 0.0, 1.5]),
          (SL[1][1] * 32 - 1, [1.0, 0.5, -0.25, 0.0]), (2 * 32, [-2.0 ** -8, 0.9, 1.1, 0.6])]
CHECKERS = ("head", "hg", "residual", "hi_only", "wgrad", "unfold")


def test_standin_slicing_matches_the_gpu_tests_slice_edges():
    """slice_tiles is the wgrad16 launch's slicing, as tests/test_gpu_layerwise.py's slice_edges states it."""
    from tests.test_gpu_layerwise import slice_edges
    for n_tiles in (1, 12, 140, 65536):
        for blocks in (1, 2, 3):
            edges = [e for t0, t1 in em.slice_tiles(n_tiles, blocks, 132) for e in (t0 * 32, t1 * 32 - 1)]
            assert edges == slice_edges(n_tiles, 32, blocks, 132)


def test_pow2_scale_and_ulp16():
    for b in (1e-30, 3e-5, 0.7, 1.0, 16384.0, 16385.0, 1e20):
        s = em.pow2_scale(b)
        assert s * b <= 16384.0 < 2 * s * b or s in (2.0 ** 100, 2.0 ** -100)
    assert em.pow2_scale(0.0) == 1.0 and em.pow2_scale(float("nan")) == 1.0
    v = torch.tensor([0.0, 2.0 ** -20, 2.0 ** -14, 1.0, 1.5, 65504.0], dtype=torch.float64)
    assert em.ulp16(v).tolist() == [2.0 ** -24, 2.0 ** -24, 2.0 ** -24, 2.0 ** -10, 2.0 ** -10, 32.0]


@pytest.mark.parametrize("sigma_only", [False, True])
def test_checkers_pass_on_the_faithful_standin(fwd, sigma_only):
    for pt, vec in PROBES:
        if sigma_only and vec[3] == 0:
            continue
        worst = run(fwd, None, pt, vec, sigma_only)
        print(pt, {k: f"{v:.3f}" for k, v in worst.items()})
        for k, v in worst.items():
            assert v <= 1.0, (pt, k, v)


AIMED = {1: "residual", 2: "residual", 3: "hi_only", 4: "hg", 5: "residual", 6: "head", 7: "wgrad", 8: "wgrad"}


@pytest.mark.parametrize("defect", sorted(em.DEFECTS))
def test_each_checker_fails_on_its_defect(fwd, defect):
    """The checker aimed at the defect fails at one of the probes (defect 8: at the probe in the skipped tile)."""
    worst = {}
    for pt, vec in PROBES:
        for k, v in run(fwd, defect, pt, vec).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(defect, em.DEFECTS[defect], {k: f"{v:.3g}" for k, v in worst.items()})
    assert worst[AIMED[defect]] > 1.0, (defect, worst)


# Which defects the aggregate bars (rel-L2 and max-rel per tensor against the float64 chain, bwd_bound) let through
# on a dense upstream gradient over this stand-in's 4463 points: all six precision defects stay inside them (worst
# 0.23 of a bar, the faithful stand-in 0.14); the two wgrad defects fail.  On an H100 the same bars, at the training
# size, also catch defect 4 (the head weights' bar at P_RAGGED) and no other precision defect.
LET_THROUGH = {1, 2, 3, 4, 5, 6}


def test_which_defects_the_aggregate_bars_let_through(fwd):
    p, a, raw = fwd
    g = torch.Generator().manual_seed(9)
    g_raw = torch.randn(P, 4, generator=g)
    want = chain64({k: v.double() for k, v in p.items()}, g_raw, raw, dict(a, H=[h.double() for h in a["H"]], enc=a["enc"].double(),
                                                                          dir=a["dir"].double(), G=a["G"].double()), zero_grads("cpu"))
    passed = set()
    for defect in [None] + sorted(em.DEFECTS):
        got, _ = em.StandIn(defect).backward(p, a, g_raw, raw)
        worst = 0.0
        ok = True
        for k in NAMES:
            r = float((got[k].double() - want[k]).norm() / want[k].norm())
            m = float((got[k].double() - want[k]).abs().max() / want[k].abs().max())
            worst = max(worst, r / bwd_bound("16", k), m / bwd_bound("16", k))
            ok &= r <= bwd_bound("16", k) and m <= bwd_bound("16", k)
        print(defect, "passes" if ok else "fails", f"worst fraction of the bar {worst:.3f}")
        if defect is None:
            assert ok
        elif ok:
            passed.add(defect)
    assert passed == LET_THROUGH, passed
