"""CPU side of the layer-by-layer ViT tests (tests/test_gpu_vit_layerwise.py):
- the restated weight-image and workspace layouts (tests/vit_emulation.py) against the library's byte counts, so a
  layout change fails here by name instead of turning the GPU comparisons into garbage;
- the operand emulation's own invariants;
- the per-stage bars have teeth: defects planted in the emulation at the kernels' shapes (a missing lo.hi product in
  one 64-deep K chunk of fc2, P.V's last 5 keys dropped, a 64-row tile from the wrong image, alpha applied twice, the
  wrong head's V) each exceed the bar of the stage that would see them."""
import pytest
import torch

from sinnerf_b200 import _lib, build, synthetic
from tests import vit_emulation as ve
from tests import vit_oracle as vo

PRECISIONS = {"split": (0, 1, 2), "bf16": (3,), "f16": (4,)}


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_workspace_layout_matches_library(lib):
    for n in range(1, _lib.VIT_MAX_IMAGES + 1):
        for save in (0, 1):
            bufs, total = ve.workspace_layout(n, save)
            assert lib.snb_vit_workspace_bytes(n, save) == 4 * total, (n, save)
            spans = sorted((o, o + torch.Size(s).numel(), k) for k, (o, s) in bufs.items())
            assert all(o % 64 == 0 for o, _, _ in spans)
            assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))       # no overlap
            assert ("blk11.lse" in bufs) == bool(save) and ("c0" in bufs) == bool(save)


def test_pack_layout_matches_library(lib):
    for mode, precs in PRECISIONS.items():
        for p in precs:
            assert lib.snb_vit_pack_bytes(p) == ve.pack_bytes(mode), (mode, p)
    L = ve.pack_layout("split")
    assert L["planes"] == 2 and ve.pack_layout("f16")["planes"] == ve.pack_layout("bf16")["planes"] == 1
    assert L["blk"][11]["fc2"] + 2 * ve.DIM * ve.MLP <= L["n_halfs"]


def test_operand_emulation():
    x = torch.tensor([1e5, -7e4, 65519.0, 0.3, 1e-3, 3e-6, 2.0 ** -24, 0.0])
    hi, lo = ve.operand(x, "split")
    assert hi[0] == 65504 and lo[0] == 0 and hi[1] == -65504 and hi[2] == 65504
    assert torch.equal(ve.operand(x, "f16")[0], hi) and ve.operand(x, "f16")[1] is None
    # lo keeps fp16 subnormals: hi + lo recovers |x| < 0.25 to fp16's fixed 2^-24 resolution, not 22 bits
    small = torch.tensor([1e-3, 0.1, 0.2])
    h, l = ve.operand(small, "split")
    assert (l != 0).all() and ((h + l - small).abs() <= 2.0 ** -25).all()
    assert torch.equal(ve.operand(x, "bf16")[0], x.bfloat16().float())
    # the three products of the split: the missing lo.lo is the only difference to (hi + lo)(hi + lo)
    a, b = torch.randn(5, 70), torch.randn(3, 70)
    p = ve.Prod(a, b, "split")
    (ah, al), (bh, bl) = ve.operand(a, "split"), ve.operand(b, "split")
    full = (ah + al).double() @ (bh + bl).double().t()
    assert torch.allclose(p.emu, full - al.double() @ bl.double().t(), rtol=0, atol=1e-12)


@pytest.fixture(scope="module")
def block0():
    """block 0 of two images (64 x 64 and 63 x 84) with the synthetic weights: fp32 stage inputs as the kernels see
    them (each one the split-mode emulation of the stage before, rounded to fp32)"""
    sd = {k: v.float() for k, v in synthetic.dino_vits16_state_dict(0).items()}
    sd64 = {k: v.double() for k, v in sd.items()}
    g = torch.Generator().manual_seed(0)
    xs = [torch.rand(1, 3, h, w, generator=g, dtype=torch.float64) for h, w in ((64, 64), (63, 84))]
    t = torch.cat([vo.tokens(sd64, vo.preprocess(x)) for x in xs]).float()
    p = "blocks.0."
    B = {k: sd[p + v] for k, v in (("n1w", "norm1.weight"), ("n1b", "norm1.bias"), ("Wqkv", "attn.qkv.weight"),
                                   ("bqkv", "attn.qkv.bias"), ("Wp", "attn.proj.weight"), ("bp", "attn.proj.bias"),
                                   ("n2w", "norm2.weight"), ("n2b", "norm2.bias"), ("W1", "mlp.fc1.weight"),
                                   ("b1", "mlp.fc1.bias"), ("W2", "mlp.fc2.weight"), ("b2", "mlp.fc2.bias"))}
    ln1 = ve.ln64(t, B["n1w"], B["n1b"]).float()
    qkv = ve.linear_ref(ln1, B["Wqkv"], B["bqkv"], "split")[0].float()
    q, k, v = (ve.heads(qkv[..., j * ve.DIM:(j + 1) * ve.DIM]) for j in range(3))
    Pm = ve.scores_ref(q, k, "split")[3]
    O = ve.unheads(ve.pv_ref(Pm, v, "split")[0].float())
    x_mid = ve.linear_ref(O, B["Wp"], B["bp"], "split", resid=t)[0].float()
    pre = ve.linear_ref(ve.ln64(x_mid, B["n2w"], B["n2b"]).float(), B["W1"], B["b1"], "split")[0].float()
    return dict(B=B, ln1=ln1, q=q, k=k, v=v, x_mid=x_mid, h=ve.gelu64(pre).float())


def caught(stage, mode, y_bad, ref, scale):
    """the defect's (worst, rms) against the correct emulation exceeds the stage's bar in one of the two"""
    w, r = ve.stats(ve.err(y_bad.float(), ref, scale))
    bw, br = ve.BARS[mode][stage]
    print(f"planted defect in {stage} ({mode}): worst {w:.2e} rms {r:.2e} (bars {bw:.0e} {br:.0e})")
    return w > bw or r > br


@pytest.mark.parametrize("chunk", [0, 11, 23])
def test_bar_catches_missing_lo_hi_chunk_in_fc2(block0, chunk):
    d = block0
    emu, _, sc = ve.linear_ref(d["h"], d["B"]["W2"], d["B"]["b2"], "split", resid=d["x_mid"])
    bad = ve.linear_ref(d["h"], d["B"]["W2"], d["B"]["b2"], "split", resid=d["x_mid"], k_chunks_without_lo_hi=(chunk,))[0]
    assert caught("fc2", "split", bad, emu, sc)


@pytest.mark.parametrize("mode", list(ve.MODES))
def test_bars_catch_planted_defects(block0, mode):
    d = block0
    # one 64-row M tile of image 0's qkv taken from image 1
    emu, _, sc = ve.linear_ref(d["ln1"], d["B"]["Wqkv"], d["B"]["bqkv"], mode)
    bad = emu.clone()
    bad[0, 64:128] = emu[1, 64:128]
    assert caught("qkv", mode, bad, emu, sc)
    # alpha applied twice to the scores
    lse, _, sc, Pm = ve.scores_ref(d["q"], d["k"], mode)
    assert caught("lse", mode, ve.scores_ref(d["q"], d["k"], mode, alpha=ve.ALPHA ** 2)[0], lse, sc)
    # P.V without its last 5 keys (the K tail of 197 = 3 x 64 + 5)
    emu, _, sc = ve.pv_ref(Pm, d["v"], mode)
    Pt = Pm.clone()
    Pt[..., -5:] = 0
    assert caught("pv", mode, ve.pv_ref(Pt, d["v"], mode)[0], emu, sc)
    # P.V with the next head's V
    assert caught("pv", mode, ve.pv_ref(Pm, d["v"].roll(1, dims=1), mode)[0], emu, sc)
