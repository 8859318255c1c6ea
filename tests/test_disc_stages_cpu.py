"""CPU side of the discriminator stage tests (tests/test_gpu_disc_stages.py):
- the restated workspace layout (tests/disc_emulation.py) against the library's byte counts, so a layout change fails
  here by name instead of turning the GPU comparisons into garbage;
- the shapes whose input-gradient GEMM would exceed the launch grid, refused on the host exactly at the boundary;
- the chained stage references against the float64 oracle (tests/disc_oracle.py), so that the references index
  every buffer the way the network does;
- the per-stage bars have teeth: defects planted in the emulation at the kernels' shapes each exceed the bar of the
  stage that would see them."""
import ctypes

import pytest
import torch

from sinnerf_b200 import _lib, build
from sinnerf_b200.discriminator import Discriminator
from tests import disc_emulation as de
from tests import disc_oracle as do
from tests._common import rel_l2

BRANCHES = [(128, 128, 128), (64, 64, 64), (64, 67, 75), (32, 32, 32), (32, 33, 47), (-1, 63, 84), (-1, 56, 70),
            (-1, 16, 16)]


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


@pytest.mark.parametrize("imsize,h,w", BRANCHES)
def test_workspace_layout_matches_library(lib, imsize, h, w):
    for n in (1, 3, 8):
        for save in (0, 1):
            bufs, total = de.workspace_layout(imsize, n, h, w, save)
            assert lib.snb_disc_workspace_bytes(imsize, n, h, w, save) == 4 * total, (n, save)
            spans = sorted((o, o + torch.Size(s).numel(), k) for k, (o, s) in bufs.items())
            assert all(o % 64 == 0 for o, _, _ in spans)
            assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))       # no overlap
            L = len(de.net(imsize, n, h, w))
            assert ("dx" in bufs) == bool(save) and f"col{L - 1}" in bufs and f"y{L - 1}" not in bufs


# (imsize, h, w, n): n P of layer 0 exactly 65535 x 64 = 4194240 rows, the largest the input-gradient GEMM's grid takes,
# and the 128 / 64 branches' square patches one image below and at the first batch past the boundary
@pytest.mark.parametrize("imsize,h,w,n_ok", [(128, 510, 514, 64), (128, 128, 128, 1023), (64, 64, 64, 4095),
                                             (64, 510, 514, 64)])
def test_large_batches_refused_at_the_gemm_grid(lib, imsize, h, w, n_ok):
    rows = n_ok * de.net(imsize, n_ok, h, w)[0]["P"]
    assert rows <= 65535 * 64 < rows + de.net(imsize, 1, h, w)[0]["P"]
    for save in (0, 1):
        assert lib.snb_disc_workspace_bytes(imsize, n_ok, h, w, save) > 0
        assert lib.snb_disc_workspace_bytes(imsize, n_ok + 1, h, w, save) == 0
    # the forward refuses the same shape before it looks at any pointer, naming the layer
    nul = (ctypes.c_void_p * _lib.DISC_MAX_LAYERS)()
    st = (ctypes.c_int64 * 4)(1, 1, 1, 1)
    assert lib.snb_disc_forward(imsize, 1, 1, nul, nul, nul, None, st, n_ok + 1, h, w, None, None, None, None) == -1
    assert b"layer 0" in lib.snb_last_error()


# --------------------------------------------------------------------------------------------------------------------
# the emulation
# --------------------------------------------------------------------------------------------------------------------
def weights(imsize, seed):
    torch.manual_seed(seed)
    D = Discriminator(False, "color,cutout", imsize=imsize)
    return ([m.weight_orig.detach().clone() for m in D.convs()], [m.weight_u.clone() for m in D.convs()],
            [m.weight_v.clone() for m in D.convs()])


def draws(n, h, w):
    """augmentation draws for n images: saturation factors 0 / 1 / 2, contrast 0.5 / 1.5, the cutout at the clamped
    right edge (image 0), the bottom-left corner and the interior"""
    rb = torch.tensor([0.3, 0.7, 0.55, 0.2][:n])
    rs = torch.tensor([0.0, 0.5, 1.0, 0.25][:n])
    rc = torch.tensor([1.0, 0.0, 0.75, 0.4][:n])
    oy = torch.tensor([h // 2, h - 1, h // 3, 0][:n])
    ox = torch.tensor([w, 0, w // 2, 0][:n])
    return rb, rs, rc, oy, ox


def run_emulation(imsize, h, w, n, mode, aug, seed=0):
    Ws, us, vs = weights(imsize, seed)
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, h, w, generator=g)
    a = draws(n, h, w) if aug else None
    b = de.emulate_forward(imsize, Ws, us, vs, x, True, a, "split" if mode is None else mode)
    d_out = torch.randn(b["out"].shape, generator=g)
    de.emulate_backward(b, Ws, d_out, "split" if mode is None else mode)
    return dict(b=b, Ws=Ws, us=us, vs=vs, x=x, aug=a, d_out=d_out)


@pytest.mark.parametrize("imsize,h,w", [(64, 64, 64), (-1, 63, 84), (32, 33, 47)])
@pytest.mark.parametrize("aug", [False, True])
def test_emulation_chains_to_the_oracle(imsize, h, w, aug):
    """the stage references, chained, are the network: the emulated split-mode call against the float64 oracle
    (an index or layout slip in a reference gives errors of order 1)"""
    R = run_emulation(imsize, h, w, 2, None, aug)
    b = R["b"]
    ws = [t.double().requires_grad_(True) for t in R["Ws"]]
    x = R["x"].double().requires_grad_(True)
    out, us2, vs2, sig = do.forward(ws, R["us"], R["vs"], x, imsize, True, R["aug"])
    (out * R["d_out"].double()).sum().backward()
    e = {"out": rel_l2(b["out"], out.detach()), "dx": rel_l2(b["d_input"], x.grad),
         "dw": max(rel_l2(b[f"dW{i}"], wt.grad) for i, wt in enumerate(ws)),
         "uv": max(max(rel_l2(b[f"u{i}"], u), rel_l2(b[f"v{i}"], v)) for i, (u, v) in enumerate(zip(us2, vs2))),
         "sigma": rel_l2(b["sigma"], torch.stack(sig))}
    print(f"emulation vs oracle {imsize} {h}x{w} aug={aug}: " + " ".join(f"{k} {v:.1e}" for k, v in e.items()))
    assert e["out"] <= 1e-4 and e["uv"] <= 1e-6 and e["sigma"] <= 1e-6, e
    assert e["dx"] <= 1e-2 and e["dw"] <= 1e-2, e


# --------------------------------------------------------------------------------------------------------------------
# planted defects
# --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def em():
    """the 64 branch at 64 x 64 with n = 3 augmented images, per mode: the emulated call's buffers"""
    return {m: run_emulation(64, 64, 64, 3, m, True, seed=1) for m in de.MODES}


def caught(stage, mode, y_bad, ref, scale):
    """the defect's (worst, rms) against the correct reference exceeds the stage's bar in one of the two"""
    w, r = de.stats(de.err(y_bad.float(), ref, scale))
    bw, br = de.BARS[mode][stage]
    print(f"planted defect in {stage} ({mode}): worst {w:.2e} rms {r:.2e} (bars {bw:.0e} {br:.0e})")
    return w > bw or r > br


def fold_args(b, i):
    return b["layers"], i, b[f"dcol{i}"], b[f"y{i - 1}"], b.get(f"mean{i - 1}"), b.get(f"rstd{i - 1}")


@pytest.mark.parametrize("mode", list(de.MODES))
def test_bars_catch_planted_defects(em, mode):
    R = em[mode]
    b = R["b"]
    L = b["layers"]
    n, C = 3, L[1]["cout"]
    # layer 0 (K = 48 in one partial 64-deep chunk) without its last 16 (the blue channel's taps)
    ref, _, sc = de.gemm_fwd_ref(b["ws0"], b["col0"], b["alpha"][0], 1.0, mode)
    col = b["col0"].clone()
    col[:, 32:] = 0
    assert caught("fwd", mode, de.gemm_fwd_ref(b["ws0"], col, b["alpha"][0], 1.0, mode)[0], ref, sc)
    # the fold: the InstanceNorm statistics row b C + c for (channel c, image b), the n mean(g n) term dropped, the
    # LeakyReLU mask taken on the pre-norm y
    ref, sc, _ = de.fold_ref(*fold_args(b, 2))
    swap = (torch.arange(n).view(1, n) * C + torch.arange(C).view(C, 1)).reshape(-1)
    for defect in (dict(row_index=swap), dict(drop_gn=True), dict(mask_on_y=True)):
        assert caught("fold", mode, de.fold_ref(*fold_args(b, 2), **defect)[0], ref, sc), defect
    # the cutout box one column short at the clamped right edge (image 0's box ends at column 63)
    assert int(b["box"][0, 3]) == 63
    ref, sc, _ = de.gather0_ref(L, R["x"], b["aug_f"], b["aug_mean"], b["box"])
    box = b["box"].clone()
    box[0, 3] -= 1
    bad = de.gather0_ref(L, R["x"], b["aug_f"], b["aug_mean"], box)[0]
    assert caught("gather0", mode, bad, ref, sc * 2.0 ** -24)
    # 1 / sigma applied twice in the dgrad of layer 1
    ref, _, sc = de.dgrad_ref(b["dy1"], b["ws1"], b["alpha"][1], mode)
    assert caught("dgrad", mode, ref * float(b["inv_sigma"][1]), ref, sc)
    # the spectral-norm correction with 1 / sigma instead of 1 / sigma^2 (layer 1).  dW is nearly orthogonal to W, so
    # the correction is ~1e-5 of the wgrad's error scale, just above the bars; the exact weight-scaling invariance of
    # test_gpu_disc_stages.py (W 2^j: dW_orig 2^-j, part 2^j, 1 / sigma 2^-j) catches it by a wide margin
    raw, _, rsc = de.wgrad_ref(b["dy1"], b["col1"], de.col_scale(L, 1), mode)
    fix = (b["part1"], b["inv_sigma"][1], b["u1"], b["v1"], b["gexp"][1])
    ref, sc = de.sn_fix_ref(raw, rsc, *fix)
    bad = de.sn_fix_ref(raw, rsc, *fix, sigma_power=1)[0]
    assert caught("wgrad", mode, bad, ref, sc)
    fix_j = (b["part1"] * 2.0 ** 7, b["inv_sigma"][1] * 2.0 ** -7) + fix[2:]
    assert torch.equal(de.sn_fix_ref(raw, rsc, *fix_j)[0] * 2.0 ** 7, ref)
    assert not torch.equal(de.sn_fix_ref(raw, rsc, *fix_j, sigma_power=1)[0] * 2.0 ** 7, bad)
    # a wgrad tile (the first 64 x 64 of dW) reading image 1's col in place of image 0's
    col = b["col1"].clone()
    P = L[1]["P"]
    col[:P, :64] = b["col1"][P:2 * P, :64]
    bad = de.sn_fix_ref(de.wgrad_ref(b["dy1"], col, de.col_scale(L, 1), mode)[0], rsc, *fix)[0]
    assert caught("wgrad", mode, bad, ref, sc)
    # the contrast backward averaging over the cut pixels too
    ref, sc = de.aug_bwd_ref(b["dx"], b["aug_f"], b["box"], b["gexp"][0], 64, 64)
    bad = de.aug_bwd_ref(b["dx"], b["aug_f"], b["box"], b["gexp"][0], 64, 64, cut_in_mean=True)[0]
    assert caught("aug_bwd", mode, bad, ref, sc)


@pytest.mark.parametrize("chunk", [0, 7, 15])
def test_bar_catches_missing_lo_hi_chunk(em, chunk):
    """layer 1 (K = 1024, sixteen 64-deep chunks) with one chunk missing its lo.hi product"""
    b = em["split"]["b"]
    cs = de.col_scale(b["layers"], 1)
    ref, _, sc = de.gemm_fwd_ref(b["ws1"], b["col1"], b["alpha"][1], cs, "split")
    bad = de.gemm_fwd_ref(b["ws1"], b["col1"], b["alpha"][1], cs, "split", k_chunks_without_lo_hi=(chunk,))[0]
    assert caught("fwd", "split", bad, ref, sc)
