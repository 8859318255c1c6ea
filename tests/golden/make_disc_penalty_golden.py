#!/usr/bin/env python
"""Generate tests/golden/disc_penalty.npz by running the REFERENCE's own Discriminator (models/discriminator.py,
with models/diff_aug.py) in float64 on the CPU under SinNeRF's compute_grad2 (models/sinnerf.py:227-239).

Run where a reference checkout is available (the GPU test machines need none):

    python tests/golden/make_disc_penalty_golden.py /path/to/reference

Per case (imsize 64 at 64x64, -1 at 63x84 and 56x70, 32 at 32x32, 128 at 128x128; B = 1 and 2; the augmentation
gates firing or not), in training mode: torch.manual_seed(seed) builds Discriminator(False, 'color,cutout',
imsize=...) and casts it to float64; x (from torch.Generator(2000 + seed)) is made to require grad; under
np.random.seed(gate seed) and torch.manual_seed(seed + 1) one call d_out = D(x), then
g = autograd.grad(d_out.sum(), x, create_graph=True), reg = (g^2).view(B, -1).sum(1), and a backward of
sum(c reg) for per-image weights c (from the same generator).  Stored: the DiffAugment draws the call made (so the
restatement can replay them), reg, and a seeded sample and the norm of the input gradient and of every weight_orig
gradient.  The weights and inputs are not stored: they regenerate from the seeds.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
BRANCHES = [(64, 64, 64), (-1, 63, 84), (-1, 56, 70), (32, 32, 32), (128, 128, 128)]
N_SAMPLE = 64


def gate_seed(fire):
    """first numpy seed whose two gate draws apply (fire) or skip the augmentation"""
    for s in range(1000):
        np.random.seed(s)
        a, b = np.random.random(), np.random.random()
        if (a > 0.5 and b >= 0.5) == fire:
            return s
    raise AssertionError


def case_name(imsize, H, W, B, fire):
    return f"i{imsize}_{H}x{W}_b{B}_{'aug' if fire else 'plain'}"


def inputs(seed, B, H, W):
    g = torch.Generator().manual_seed(2000 + seed)
    x = torch.rand(B, 3, H, W, generator=g, dtype=torch.float64)
    c = torch.rand(B, generator=g, dtype=torch.float64) + 0.5
    return x, c


def run_case(Disc, imsize, H, W, B, fire, seed):
    torch.manual_seed(seed)
    D = Disc(False, "color,cutout", imsize=imsize).double()
    convs = [m for m in D.main if isinstance(m, torch.nn.Conv2d)]
    x, c = inputs(seed, B, H, W)
    x.requires_grad_(True)
    draws = []
    rand, randint = torch.rand, torch.randint

    def rec_rand(*a, **k):
        t = rand(*a, **k)
        draws.append(t.reshape(-1).double().numpy().copy())
        return t

    def rec_randint(*a, **k):
        t = randint(*a, **k)
        draws.append(t.reshape(-1).double().numpy().copy())
        return t

    np.random.seed(gate_seed(fire))
    torch.manual_seed(seed + 1)
    torch.rand, torch.randint = rec_rand, rec_randint
    try:
        d_out = D(x)
    finally:
        torch.rand, torch.randint = rand, randint
    assert (len(draws) == 5) == fire, len(draws)
    (g,) = torch.autograd.grad(d_out.sum(), x, create_graph=True)
    reg = g.pow(2).view(B, -1).sum(1)
    (reg * c).sum().backward()
    rng = np.random.default_rng(7)
    idx = [rng.integers(0, m.weight_orig.numel(), N_SAMPLE) for m in convs]
    out = {
        "draws": np.stack(draws) if fire else np.zeros((0, B)),
        "reg": reg.detach().numpy(),
        "dx_idx": (dxi := rng.integers(0, x.numel(), 4 * N_SAMPLE)),
        "dx_sample": x.grad.reshape(-1).numpy()[dxi],
        "dx_norm": np.array(float(x.grad.norm())),
        "sample_idx": np.stack(idx),
        "dw_sample": np.stack([m.weight_orig.grad.reshape(-1).numpy()[i] for m, i in zip(convs, idx)]),
        "dw_norm": np.array([float(m.weight_orig.grad.norm()) for m in convs]),
    }
    return out


def main():
    if len(sys.argv) < 2:
        sys.exit("usage: python tests/golden/make_disc_penalty_golden.py /path/to/reference")
    sys.path.insert(0, sys.argv[1])
    from models.discriminator import Discriminator
    data = {}
    for k, (imsize, H, W) in enumerate(BRANCHES):
        for B in (1, 2):
            for fire in (True, False):
                seed = 10 * k + B
                name = case_name(imsize, H, W, B, fire)
                for key, v in run_case(Discriminator, imsize, H, W, B, fire, seed).items():
                    data[f"{name}/{key}"] = v
                data[f"{name}/meta"] = np.array([imsize, H, W, B, int(fire), seed])
                print(name, "reg", data[f"{name}/reg"])
    path = os.path.join(HERE, "disc_penalty.npz")
    np.savez_compressed(path, **data)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
