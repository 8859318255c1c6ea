"""GPU tests of the standalone DiffAugment (sinnerf_b200.discriminator.DiffAugment, csrc/disc.cu diff_aug_*_kernel)
against the float64 oracle (tests/diff_aug_oracle.py) given the same draws -- the call is re-seeded and its
draws replayed through diff_augment_draws -- at every case of tests/golden/diff_aug.npz, in NCHW, channels_first=False
and the '(b p q) c -> b c p q' view of a ray-major tensor; translation at its extreme shifts; other channel counts and
repeated ops; bitwise agreement with the discriminator's fused augmentation in every precision mode; determinism,
the absence of host synchronisation, autocast and the argument checks."""
import numpy as np
import pytest
import torch

from sinnerf_b200 import discriminator as disc
from sinnerf_b200.discriminator import DiffAugment, Discriminator, diff_augment_draws, draw_augment
from tests import diff_aug_oracle as dao
from tests._common import load_npz, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D64 = torch.float64
# rel-L2 against float64: fp32 arithmetic whose longest reduction (contrast's mean, and its gradient's mean) sums
# 3 x 84 x 63 = 15876 terms; both directions are held to 1e-6
BAR = 1e-6
LAYOUTS = ["nchw", "nhwc", "rays"]


def _gate_seed(fire):
    for s in range(1000):
        np.random.seed(s)
        if (np.random.random() >= 0.5) == fire:
            return s
    raise AssertionError


def golden_cases():
    g = load_npz("diff_aug.npz")
    out = []
    for i in range(int(g["n_cases"])):
        pi, H, W, B, fire, *_ = (int(v) for v in g[f"c{i}_meta"])
        if fire:
            out.append((str(g["policies"][pi]), H, W, B))
    return out


def as_layout(x, layout):
    """-> (leaf, the tensor DiffAugment is given, channels_first) for x (B, C, H, W)"""
    B, C, H, W = x.shape
    if layout == "nchw":
        leaf = x.clone().requires_grad_(True)
        return leaf, leaf, True
    leaf = x.permute(0, 2, 3, 1).reshape(B * H * W, C).contiguous().requires_grad_(True)
    if layout == "nhwc":
        return leaf, leaf.view(B, H, W, C), False
    return leaf, leaf.view(B, H, W, C).permute(0, 3, 1, 2), True


def to_nchw(t, channels_first):
    return t if channels_first else t.permute(0, 3, 1, 2)


def run(x_in, policy, channels_first, np_seed, torch_seed):
    np.random.seed(np_seed)
    torch.cuda.manual_seed(torch_seed)
    return DiffAugment(x_in, policy, channels_first)


def replay(policy, shape, np_seed, torch_seed):
    np.random.seed(np_seed)
    torch.cuda.manual_seed(torch_seed)
    return diff_augment_draws(policy, shape, DEV)


def check_against_oracle(x, policy, layout, torch_seed=0, fwd_bar=BAR, grad_bar=BAR):
    leaf, x_in, cf = as_layout(x, layout)
    s = _gate_seed(True)
    y = run(x_in, policy, cf, s, torch_seed)
    draws = replay(policy, tuple(x.shape), s, torch_seed)
    assert y is not x_in and y.is_contiguous() and y.shape == x_in.shape and y.dtype == torch.float32
    xo = x.double().cpu().requires_grad_(True)
    want = dao.diff_augment(xo, [(op, tuple(t.cpu() for t in ts)) for op, ts in draws])
    got = to_nchw(y, cf)
    assert rel_l2(got.detach().cpu(), want.detach()) <= fwd_bar, (policy, layout)
    w = torch.randn(x.shape, generator=torch.Generator().manual_seed(torch_seed)).double()   # fp32 values
    (got * w.to(DEV, torch.float32)).sum().backward()
    (want * w).sum().backward()
    B, C, H, W = x.shape
    gx = leaf.grad if layout == "nchw" else leaf.grad.view(B, H, W, C).permute(0, 3, 1, 2)
    assert leaf.grad.stride() == leaf.stride()
    assert rel_l2(gx.cpu(), xo.grad) <= grad_bar, (policy, layout)
    return got.detach(), want.detach(), gx, xo.grad


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("policy,H,W,B", golden_cases())
def test_oracle_parity(policy, H, W, B, layout):
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H * W + B)).to(DEV)
    got, want, gx, gw = check_against_oracle(x, policy, layout, torch_seed=H + W + B)
    if "color" not in policy:
        # translation and cutout only move and zero values: exact in both directions
        assert torch.equal(got.cpu().double(), want)
        assert torch.equal(gx.cpu().double(), gw)


@pytest.mark.parametrize("policy", ["color,color", "cutout,translation,cutout", "translation,color,translation",
                                    "color,translation,color,cutout"])
@pytest.mark.parametrize("C", [1, 3, 5])
def test_repeated_ops_and_channels(policy, C):
    x = torch.rand(2, C, 24, 30, generator=torch.Generator().manual_seed(C)).to(DEV)
    for layout in LAYOUTS:
        check_against_oracle(x, policy, layout, torch_seed=C)


@pytest.mark.parametrize("H,W", [(64, 64), (63, 84), (7, 9)])
def test_translation_edges(H, W):
    sy, sx = int(H * 0.125 + 0.5), int(W * 0.125 + 0.5)
    ty = torch.tensor([-sy, sy, 0, -sy, sy, 0, sy, -sy, 0], device=DEV)
    tx = torch.tensor([-sx, -sx, -sx, sx, sx, sx, 0, 0, 0], device=DEV)
    B = ty.numel()
    x = (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H)) + 0.5).to(DEV).requires_grad_(True)
    draws = [("translation", (ty, tx))]
    y = disc._DiffAugFn.apply(x, True, draws)
    want = dao.diff_augment(x.detach().cpu().double(), [("translation", (ty.cpu(), tx.cpu()))])
    assert torch.equal(y.detach().cpu().double(), want)
    g = torch.rand(y.shape, generator=torch.Generator().manual_seed(W)).to(DEV) + 0.5
    (gx,) = torch.autograd.grad(y, x, g)
    for b in range(B):
        a, c = int(ty[b]), int(tx[b])
        # output pixel (i, j) reads input (i + a, j + c): input rows [r0, r1) and columns [c0, c1) are read, each by
        # one output pixel; the others are shifted out and get no gradient
        r0, r1, c0, c1 = max(0, a), H + min(0, a), max(0, c), W + min(0, c)
        live = torch.zeros(H, W, dtype=torch.bool, device=DEV)
        live[r0:r1, c0:c1] = True
        assert (gx[b][:, ~live] == 0).all()
        assert torch.equal(gx[b][:, r0:r1, c0:c1], g[b][:, r0 - a:r1 - a, c0 - c:c1 - c])
        # the zero borders: the output rows / columns read from the padding (the input is >= 0.5 elsewhere)
        inside = torch.zeros(H, W, dtype=torch.bool, device=DEV)
        inside[r0 - a:r1 - a, c0 - c:c1 - c] = True
        assert (y[b][:, ~inside] == 0).all() and (y[b][:, inside] >= 0.5).all()


@pytest.mark.parametrize("precision", ["f16x3", "f16", "bf16"])
@pytest.mark.parametrize("imsize,H,W,B", [(64, 64, 64, 2), (-1, 63, 84, 1), (-1, 56, 70, 2)])
def test_agrees_with_discriminator_bitwise(precision, imsize, H, W, B):
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(B)).to(DEV)
    for s in range(1000):   # a numpy seed whose two discriminator gates both apply the augmentation
        np.random.seed(s)
        if np.random.random() > 0.5 and np.random.random() >= 0.5:
            break
    outs = []
    for policy in ("color,cutout", None):
        np.random.seed(0)
        torch.manual_seed(0)
        outs.append(Discriminator(False, policy, imsize=imsize, precision=precision).to(DEV))
    D_aug, D_plain = outs
    np.random.seed(s)
    torch.cuda.manual_seed(7)
    want = D_aug(x)
    np.random.seed(s)
    torch.cuda.manual_seed(7)
    aug = draw_augment("color,cutout", tuple(x.shape), DEV)
    assert aug is not None
    y = disc._DiffAugFn.apply(x, True, [("color", aug[:3]), ("cutout", aug[3:])])
    got = D_plain(y)
    assert torch.equal(got, want)


def test_gate_returns_input_itself():
    x = torch.rand(1, 3, 16, 16, device=DEV)
    np.random.seed(_gate_seed(False))
    assert DiffAugment(x) is x
    np.random.seed(_gate_seed(True))
    assert DiffAugment(x, "") is x


def test_deterministic():
    x = torch.rand(3, 3, 63, 84, generator=torch.Generator().manual_seed(0)).to(DEV)
    w = torch.randn(3, 3, 63, 84, generator=torch.Generator().manual_seed(1)).to(DEV)
    outs = []
    for _ in range(2):
        leaf = x.clone().requires_grad_(True)
        y = run(leaf, "color,translation,cutout", True, _gate_seed(True), 3)
        (y * w).sum().backward()
        outs.append((y.detach(), leaf.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_no_host_sync():
    x = torch.rand(2, 3, 64, 64, device=DEV).requires_grad_(True)
    run(x, "color,translation,cutout", True, _gate_seed(True), 1).sum().backward()   # warm-up (library load, check)
    torch.cuda.synchronize()
    np.random.seed(_gate_seed(True))
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = DiffAugment(x, "color,translation,cutout")
        z = DiffAugment(x.detach().permute(0, 2, 3, 1), "cutout,color", channels_first=False)
        (y.square().sum() + z.sum()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_autocast_does_not_change_the_arithmetic():
    x = torch.rand(2, 3, 56, 70, generator=torch.Generator().manual_seed(2)).to(DEV)
    outs = []
    for ac in (False, True):
        leaf = x.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=ac):
            y = run(leaf, "color,translation,cutout", True, _gate_seed(True), 4)
        assert y.dtype == torch.float32
        (y * 3).sum().backward()
        outs.append((y.detach(), leaf.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_input_checks():
    with pytest.raises(RuntimeError):
        DiffAugment(torch.rand(1, 3, 8, 8))
    with pytest.raises(TypeError):
        DiffAugment(torch.rand(1, 3, 8, 8, device=DEV, dtype=torch.float64))
    with pytest.raises(TypeError):
        DiffAugment(torch.rand(1, 3, 8, 8, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError):
        DiffAugment(torch.rand(3, 8, 8, device=DEV))
    with pytest.raises(ValueError):
        DiffAugment(torch.rand(1, 1, 3, 8, 8, device=DEV))
