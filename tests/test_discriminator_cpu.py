"""CPU tests of sinnerf_b200.discriminator: the float64 oracle (tests/disc_oracle.py) against the reference's own
Discriminator (tests/golden/discriminator.npz, including the number and order of its random draws) and against
torch's nn.Conv2d + spectral_norm + InstanceNorm2d; the drop-in's parameters, buffers and state dict; the refused
configurations and shapes; and the C ABI's argument checks, none of which needs a device."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sinnerf_b200 import _lib
from sinnerf_b200.discriminator import Discriminator, draw_augment, layer_schedule, output_sizes
from tests import disc_oracle as do
from tests._common import load_npz

D64 = torch.float64
CASES = ["b64", "llff", "dtu"]
C_void, C_i64 = ctypes.c_void_p, ctypes.c_int64


@pytest.fixture(scope="module")
def gold():
    return load_npz("discriminator.npz")


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a), dtype=D64), torch.as_tensor(np.asarray(b), dtype=D64)
    return float((a - b).norm() / b.norm())


def build(imsize, seed):
    np.random.seed(seed)
    torch.manual_seed(seed)
    return Discriminator(False, "color,cutout", imsize=imsize)


def state(D):
    convs = D.convs()
    ws = [m.weight_orig.detach().double().clone().requires_grad_(True) for m in convs]
    return ws, [m.weight_u.double().clone() for m in convs], [m.weight_v.double().clone() for m in convs]


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_golden(gold, case):
    g = {k.split("/", 1)[1]: v for k, v in gold.items() if k.startswith(case + "/")}
    imsize, H, W, B, seed = (int(v) for v in g["meta"])
    D = build(imsize, seed)
    ws, us, vs = state(D)
    # the seeded initialisation is the reference's
    for i, w in enumerate(ws):
        flat = w.detach().reshape(-1).numpy()
        assert np.array_equal(flat[g["sample_idx"][i]].astype(np.float32), g["w0_sample"][i])
        assert abs(float(w.detach().norm()) - g["w0_norm"][i]) <= 1e-12 * g["w0_norm"][i]
    assert np.array_equal(torch.cat(us).float().numpy(), g["u0"]) and np.array_equal(torch.cat(vs).float().numpy(), g["v0"])

    gen = torch.Generator().manual_seed(1000 + seed)
    fake, real, fake2 = (torch.rand(B, 3, H, W, generator=gen) for _ in range(3))
    sigmas, fired = [], []

    def call(x):
        nonlocal us, vs
        aug = draw_augment("color,cutout", tuple(x.shape), "cpu")
        fired.append(aug is not None)
        out, us, vs, sig = do.forward(ws, us, vs, x, imsize, True, aug)
        sigmas.append([float(s) for s in sig])
        return out

    xf = fake.double().requires_grad_(True)
    pf = call(xf)
    (-pf.mean()).backward()
    for w in ws:
        w.grad = None
    pr = call(real.double())
    pf2 = call(fake2.double())
    ((F.relu(1 - pr).mean() + F.relu(1 + pf2).mean()) / 2).backward()

    assert fired == list(g["fired"])
    # same number and order of draws: the next values of both generators agree
    assert np.random.random() == float(g["next_np"])
    assert np.array_equal(torch.rand(4).numpy(), g["next_torch"])
    assert rel(pf.detach(), g["out_g"]) <= 1e-5
    assert rel(pr.detach(), g["out_real"]) <= 1e-5 and rel(pf2.detach(), g["out_fake"]) <= 1e-5
    assert rel(xf.grad, g["dx_g"]) <= 1e-5
    assert rel(sigmas, g["sigma"]) <= 1e-6
    assert rel(torch.cat(us), g["u1"]) <= 1e-5 and rel(torch.cat(vs), g["v1"]) <= 1e-5
    for i, w in enumerate(ws):
        assert rel(w.grad.reshape(-1)[torch.as_tensor(g["sample_idx"][i])], g["dw_sample"][i]) <= 1e-4
        assert abs(float(w.grad.norm()) - g["dw_norm"][i]) <= 1e-5 * g["dw_norm"][i]


@pytest.mark.parametrize("imsize,H,W", [(64, 64, 64), (-1, 63, 84), (32, 32, 32), (128, 128, 128), (-1, 20, 26)])
@pytest.mark.parametrize("training", [True, False])
def test_oracle_matches_torch_modules(imsize, H, W, training):
    """torch's spectral_norm hooks, Conv2d and InstanceNorm2d in float64 against the restatement (no augmentation)"""
    D = build(imsize, 3).double().train(training)
    ws, us, vs = state(D)
    x = torch.rand(2, 3, H, W, dtype=D64, generator=torch.Generator().manual_seed(5))
    x1, x2 = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    want = D.main(x1)
    got, us2, vs2, _ = do.forward(ws, us, vs, x2, imsize, training)
    assert want.shape == got.shape == (2, 1, *output_sizes(imsize, H, W)[-1])
    assert rel(got.detach(), want.detach()) <= 1e-12
    for m, u, v in zip(D.convs(), us2, vs2):
        assert rel(u, m.weight_u) <= 1e-12 and rel(v, m.weight_v) <= 1e-12
    gout = torch.randn(want.shape, dtype=D64, generator=torch.Generator().manual_seed(6))
    (want * gout).sum().backward()
    (got * gout).sum().backward()
    assert rel(x2.grad, x1.grad) <= 1e-11
    for m, w in zip(D.convs(), ws):
        assert rel(w.grad, m.weight_orig.grad) <= 1e-11


def test_augment_matches_diffaugment_semantics():
    """the cutout zeroes the clamped window, and the colour maps are affine about the two means"""
    x = torch.rand(2, 3, 9, 12, dtype=D64, generator=torch.Generator().manual_seed(1))
    aug = (torch.tensor([0.5, 0.5]), torch.tensor([0.5, 0.5]), torch.tensor([0.5, 0.5]),
           torch.tensor([0, 9]), torch.tensor([11, 0]))
    y = do.augment(x, aug)      # brightness 0, saturation 1, contrast 1: only the cutout acts
    ch, cw = 5, 6
    mask = torch.ones(2, 1, 9, 12, dtype=D64)
    mask[0, :, 0:ch - ch // 2, 11 - cw // 2:] = 0
    mask[1, :, 9 - ch // 2:, 0:cw - cw // 2] = 0
    assert torch.allclose(y, x * mask, atol=1e-15)


@pytest.mark.parametrize("imsize,n_params,keys", [
    (64, 2763776, [0, 2, 5, 8, 11]), (-1, 2117632, [0, 3, 6]), (32, 2635776, [0, 3, 6, 9]),
    (128, 2795008, [0, 2, 5, 8, 11, 14])])
def test_state_dict_layout(imsize, n_params, keys):
    D = build(imsize, 0)
    assert sum(p.numel() for p in D.parameters()) == n_params
    want = [f"main.{i}.{k}" for i in keys for k in ("weight_orig", "weight_u", "weight_v")]
    assert list(D.state_dict().keys()) == want
    assert [(m.in_channels, m.out_channels, m.bias) for m in D.convs()] == [(a, b, None) for a, b, _ in layer_schedule(imsize)]
    # a Lightning checkpoint's D.* entries load strictly into a fresh module
    ckpt = {"state_dict": {f"D.{k}": v.clone() for k, v in D.state_dict().items()}}
    E = Discriminator(False, "color,cutout", imsize=imsize)
    E.load_state_dict({k[2:]: v for k, v in ckpt["state_dict"].items() if k.startswith("D.")}, strict=True)
    for a, b in zip(D.state_dict().values(), E.state_dict().values()):
        assert torch.equal(a, b)


def test_refused_configurations():
    with pytest.raises(NotImplementedError):
        Discriminator(True, "color,cutout")
    with pytest.raises(NotImplementedError):
        Discriminator(False, "color,cutout", ndf=32)
    with pytest.raises(NotImplementedError):
        Discriminator(False, "color,translation,cutout")
    Discriminator(False, None)
    Discriminator(False, "")


@pytest.mark.parametrize("imsize,H,W", [(64, 8, 8), (-1, 4, 4), (-1, 3, 40), (-1, 8, 8), (32, 2, 2), (128, 16, 16)])
def test_shapes_the_reference_cannot_run(imsize, H, W):
    D = build(imsize, 0).double()
    with pytest.raises((ValueError, RuntimeError)):
        D.main(torch.rand(1, 3, H, W, dtype=D64))
    with pytest.raises(ValueError):
        output_sizes(imsize, H, W)
    assert _lib.load().snb_disc_workspace_bytes(imsize, 1, H, W, 1) == 0


def test_cpu_tensors_raise():
    D = Discriminator(False, "color,cutout")
    with pytest.raises(RuntimeError, match="CUDA"):
        D(torch.rand(1, 3, 64, 64))


def test_cabi_argument_checks():
    lib = _lib.load()
    assert lib.snb_disc_workspace_bytes(64, 0, 64, 64, 0) == 0
    assert lib.snb_disc_workspace_bytes(64, 2, 64, 64, 1) > lib.snb_disc_workspace_bytes(64, 2, 64, 64, 0) > \
        lib.snb_disc_workspace_bytes(64, 1, 64, 64, 0) > 0
    L = _lib.DISC_MAX_LAYERS
    nul = (C_void * L)()
    st = (C_i64 * 4)(1, 1, 1, 1)
    assert lib.snb_disc_forward(64, 99, 1, nul, nul, nul, None, st, 1, 64, 64, None, None, None, None) == -3
    assert lib.snb_disc_forward(64, 1, 1, nul, nul, nul, None, st, 1, 64, 64, None, None, None, None) == -1
    assert lib.snb_disc_forward(64, 1, 1, nul, nul, nul, None, st, 0, 64, 64, None, None, None, None) == -1
    assert lib.snb_disc_forward(-1, 1, 1, nul, nul, nul, None, st, 1, 8, 8, None, None, None, None) == -1
    fake = (C_void * L)(*([16] * L))
    assert lib.snb_disc_forward(64, 1, 1, fake, fake, fake, None, st, 1, 64, 64, None, None, None, None) == -1
    assert b"null input" in lib.snb_last_error()
    aug = _lib.SnbDiscAug(16, None, None, None, None)
    assert lib.snb_disc_forward(64, 1, 1, fake, fake, fake, 16, st, 1, 64, 64, aug, 16, 16, None) == -1
    assert b"DiffAugment" in lib.snb_last_error()
    assert lib.snb_disc_backward(64, 7, nul, 1, 64, 64, None, None, None, nul, None, None) == -3
    assert lib.snb_disc_backward(64, 1, fake, 1, 64, 64, None, None, None, nul, None, None) == -1
    assert lib.snb_disc_backward(64, 1, fake, 1, 64, 64, 16, 16, None, nul, 16, None) == -1
    assert lib.snb_disc_backward(64, 1, fake, 1, 64, 64, 16, None, None, None, 16, None) == -1

