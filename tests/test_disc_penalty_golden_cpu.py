"""CPU test: the float64 restatement of the discriminator (tests/disc_oracle.py) under SinNeRF's compute_grad2
double backward equals the reference module's (tests/golden/disc_penalty.npz, from make_disc_penalty_golden.py) at
float64 round-off, on every branch, B = 1 and 2, with the augmentation gates firing or not.  The GPU tests of
forward_with_penalty hold the kernels to this restatement."""
import os

import numpy as np
import pytest
import torch

from sinnerf_b200.discriminator import Discriminator
from tests import disc_oracle as do
from tests.golden.make_disc_penalty_golden import BRANCHES, case_name, inputs

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "disc_penalty.npz")
CASES = [(imsize, H, W, B, fire) for imsize, H, W in BRANCHES for B in (1, 2) for fire in (True, False)]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b)))


@pytest.mark.parametrize("imsize,H,W,B,fire", CASES)
def test_restatement_matches_reference(golden, imsize, H, W, B, fire):
    name = case_name(imsize, H, W, B, fire)
    seed = int(golden[f"{name}/meta"][5])
    torch.manual_seed(seed)
    D = Discriminator(False, "color,cutout", imsize=imsize)
    convs = D.convs()
    ws = [m.weight_orig.detach().double().clone().requires_grad_(True) for m in convs]
    us, vs = [m.weight_u.double() for m in convs], [m.weight_v.double() for m in convs]
    x, c = inputs(seed, B, H, W)
    x.requires_grad_(True)
    draws = golden[f"{name}/draws"]
    aug = tuple(torch.from_numpy(d) for d in draws) if fire else None
    out, *_ = do.forward(ws, us, vs, x, imsize, True, aug)
    (g,) = torch.autograd.grad(out.sum(), x, create_graph=True)
    reg = g.pow(2).view(B, -1).sum(1)
    (reg * c).sum().backward()
    assert rel(reg.detach().numpy(), golden[f"{name}/reg"]) <= 1e-12
    assert rel(x.grad.reshape(-1).numpy()[golden[f"{name}/dx_idx"]], golden[f"{name}/dx_sample"]) <= 1e-10
    assert abs(float(x.grad.norm()) / float(golden[f"{name}/dx_norm"]) - 1) <= 1e-12
    for i, w in enumerate(ws):
        got = w.grad.reshape(-1).numpy()[golden[f"{name}/sample_idx"][i]]
        assert rel(got, golden[f"{name}/dw_sample"][i]) <= 1e-10, i
        assert abs(float(w.grad.norm()) / float(golden[f"{name}/dw_norm"][i]) - 1) <= 1e-12, i
