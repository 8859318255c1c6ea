"""GPU tests of sinnerf_b200.vit (csrc/vit.cu): the DINO ViT-S/16 CLS feature and its input gradient against the
float64 oracle (tests/vit_oracle.py) on SinNeRF's three patch shapes, in contiguous NCHW and in the
'(b p q) c -> b c p q' views of ray-major tensors, in the split and the single-product modes; batching, determinism,
the no-grad pass, the autocast policy, and an end-to-end check through render_rays' training path."""
import pytest
import torch

from sinnerf_b200 import config, synthetic
from sinnerf_b200.nerf import NeRF, Embedding
from sinnerf_b200.rendering import render_rays
from sinnerf_b200.vit import load_dino_weights
from tests import vit_oracle as vo
from tests._common import rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D = torch.float64

SHAPES = [(64, 64), (63, 84), (56, 70)]
LAYOUTS = ["nchw", "rays"]
# (feature, input gradient) rel-L2 bars against float64.  The single-product bars come from a CPU emulation of operand
# rounding (f16 ~1e-3 / 4e-3, bf16 ~1e-2 / 4e-2) plus margin.  Measured on an H100 over the three shapes: split
# <= 9e-6 / 5e-5, f16 <= 1.0e-3 / 2.8e-3, bf16 <= 9.2e-3 / 2.8e-2, so the bars keep a 3-7x margin.
BARS = {"f16x3": (1e-4, 1e-3), "f16": (5e-3, 2e-2), "bf16": (3e-2, 1e-1)}


@pytest.fixture(scope="module")
def sd():
    return synthetic.dino_vits16_state_dict(0)


@pytest.fixture(scope="module")
def ext(sd):
    return load_dino_weights(sd).to(DEV)


def as_layout(x, layout):
    """-> (leaf, view): x (B,3,H,W) as a contiguous leaf, or as the '(b p q) c -> b c p q' view of a ray-major leaf"""
    B, Cc, H, W = x.shape
    if layout == "nchw":
        leaf = x.detach().clone().contiguous().requires_grad_(True)
        return leaf, leaf
    leaf = x.detach().permute(0, 2, 3, 1).reshape(B * H * W, Cc).contiguous().requires_grad_(True)
    return leaf, leaf.view(B, H, W, Cc).permute(0, 3, 1, 2)


def inputs(h, w, seed, B=1):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, h, w, generator=g), torch.randn(384, generator=g, dtype=D)


def oracle(sd, x, wvec):
    x64 = x.detach().to(D).cpu().requires_grad_(True)
    f = vo.cls_feature(sd, x64)
    (f * wvec).sum().backward()
    return f.detach(), x64.grad


@pytest.mark.parametrize("mode", list(BARS))
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("hw", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_parity_vs_float64(ext, sd, hw, layout, mode):
    x, wvec = inputs(*hw, seed=hw[0] + hw[1])
    want_f, want_g = oracle(sd, x, wvec)
    leaf, view = as_layout(x.to(DEV), layout)
    f = ext.cls_feature(view, precision=mode)
    (g,) = torch.autograd.grad((f * wvec.to(DEV, torch.float32)).sum(), [view])
    assert g.stride() == view.stride()
    ef, eg = rel_l2(f.detach().cpu(), want_f), rel_l2(g[0:1].cpu(), want_g)
    print(f"vit parity {mode} {hw} {layout}: feature {ef:.2e} gradient {eg:.2e}")
    bf, bg = BARS[mode]
    assert ef <= bf and eg <= bg, (ef, eg)


def test_batch_only_image0_and_semantic_loss_bitwise(ext):
    x, _ = inputs(63, 84, seed=5, B=3)
    leaf, view = as_layout(x.to(DEV), "rays")
    f = ext.cls_feature(view)
    (g,) = torch.autograd.grad(f.square().sum(), [view])
    assert float(g[0].abs().sum()) > 0 and torch.equal(g[1:], torch.zeros_like(g[1:]))
    # semantic_loss (one batched pass of both patches) == two separate cls_feature calls, bit for bit
    ref = torch.randn(384, generator=torch.Generator().manual_seed(9)).to(DEV)
    c0, _ = inputs(64, 64, seed=6)
    f0, _ = inputs(64, 64, seed=7)
    lc, vc = as_layout(c0.to(DEV), "rays")
    lf, vf = as_layout(f0.to(DEV), "rays")
    loss = ext.semantic_loss(ref, vc, vf)
    gc, gf = torch.autograd.grad(loss, [lc, lf])
    lc2, vc2 = as_layout(c0.to(DEV), "rays")
    lf2, vf2 = as_layout(f0.to(DEV), "rays")
    loss2 = torch.nn.functional.mse_loss(ext.cls_feature(vc2), ref) + torch.nn.functional.mse_loss(ext.cls_feature(vf2), ref)
    gc2, gf2 = torch.autograd.grad(loss2, [lc2, lf2])
    assert torch.equal(loss, loss2) and torch.equal(gc, gc2) and torch.equal(gf, gf2)


@pytest.mark.parametrize("mode", list(BARS))
def test_deterministic(ext, mode):
    x, _ = inputs(56, 70, seed=11)
    out = []
    for _ in range(2):
        leaf, view = as_layout(x.to(DEV), "nchw")
        f = ext.cls_feature(view, precision=mode)
        (g,) = torch.autograd.grad(f.sum(), [view])
        out.append((f, g))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_no_grad_pass_and_split_modes_agree(ext):
    x, _ = inputs(64, 64, seed=12)
    xd = x.to(DEV).requires_grad_(True)
    f = ext.cls_feature(xd)
    with torch.no_grad():
        f_ng = ext.cls_feature(xd)
    assert f_ng.grad_fn is None and torch.equal(f.detach(), f_ng)
    # 'fp32', 'f16x3' and 'bf16x3' all run the fp16 three-product split
    with torch.no_grad():
        assert torch.equal(ext.cls_feature(xd, precision="fp32"), f_ng)
        assert torch.equal(ext.cls_feature(xd, precision="bf16x3"), f_ng)


def test_autocast_policy(ext):
    x, _ = inputs(64, 64, seed=13)
    xd = x.to(DEV)
    with torch.no_grad():
        want16 = ext.cls_feature(xd, precision="f16")
        want = ext.cls_feature(xd, precision="f16x3")
        with torch.autocast("cuda", dtype=torch.float16):
            got16 = ext.cls_feature(xd, precision="autocast")
        got = ext.cls_feature(xd, precision="autocast")
    assert torch.equal(got16, want16) and torch.equal(got, want) and got16.dtype == torch.float32


def test_weight_image_repacked_on_change(sd):
    e = load_dino_weights(sd).to(DEV)
    x = inputs(64, 64, seed=14)[0].to(DEV)
    with torch.no_grad():
        a = e.cls_feature(x)
        img = e.packed(DEV, config.resolve_precision())
        assert e.packed(DEV, config.resolve_precision()) is img
        e.model.blocks[11].mlp.fc2.bias.add_(1.0)
        b = e.cls_feature(x)
    assert not torch.equal(a, b)


def test_end_to_end_training_path(ext, sd):
    """render_rays' training path on a 64x64 side patch: the rendered coarse and fine rgb -> semantic_loss ->
    .backward(), against the same graph with the oracle's float64 semantic loss on the rendered fp32 outputs.
    - The gradients reaching the rendered rgb (what the ViT backward produces) are held to the parity bar, 1e-3.
    - The NeRF parameter gradients are held to 1e-2: the sigma head's are sums that nearly cancel over the patch, so
      the rgb gradients' rounding reaches them amplified.  Measured on an H100: rgb gradients 2.3e-4, sigma.bias
      4.5e-3, while the oracle graph's own run-to-run spread is 9e-7.
    The ViT's parameters get no .grad."""
    models = []
    for seed in (0, 1):
        m = NeRF(use_new_activation=True)
        m.load_state_dict(synthetic.default_init_params(seed))
        models.append(m.to(DEV))
    emb = [Embedding(3, 10), Embedding(3, 4)]
    side = synthetic.patch_rays("lego", 64, 64, 6, seed=2).to(DEV)
    ref = torch.randn(384, generator=torch.Generator().manual_seed(4)).to(DEV)

    def view(out, k):
        return out[k].view(1, 64, 64, 3).permute(0, 3, 1, 2)

    def grads(loss_fn):
        for m in models:
            m.zero_grad(set_to_none=True)
        r = render_rays(models, emb, side, 64, False, 0, 0, 64, 32768, True)
        for k in ("rgb_coarse", "rgb_fine"):
            r[k].retain_grad()
        loss = loss_fn(view(r, "rgb_coarse"), view(r, "rgb_fine"))
        loss.backward()
        return float(loss), [r[k].grad.detach().clone() for k in ("rgb_coarse", "rgb_fine")], \
            [{k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None} for m in models]

    old = config.get_train_storage()
    config.set_train_storage("fp32")
    try:
        lf, rf, gf = grads(lambda c, f: ext.semantic_loss(ref, c, f))
        lo, ro, go = grads(lambda c, f: vo.semantic_loss(sd, ref.double().cpu(), c.double().cpu(), f.double().cpu()))
    finally:
        config.set_train_storage(old)
    assert all(p.grad is None for p in ext.parameters())
    assert abs(lf - lo) <= 1e-4 * abs(lo), (lf, lo)
    rgb_err = max(rel_l2(a, b) for a, b in zip(rf, ro))
    assert rgb_err <= 1e-3, rgb_err
    n, worst = 0, (0.0, "")
    for a, b in zip(gf, go):
        assert a.keys() == b.keys()
        for k in a:
            if float(b[k].norm()) == 0.0:
                continue
            worst = max(worst, (rel_l2(a[k], b[k]), k))
            n += 1
    print(f"vit end to end: rgb-gradient rel-L2 {rgb_err:.2e}; worst parameter-gradient rel-L2 {worst[0]:.2e} "
          f"({worst[1]})")
    assert worst[0] <= 1e-2 and n >= 20, worst
