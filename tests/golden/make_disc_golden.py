#!/usr/bin/env python
"""Generate tests/golden/discriminator.npz by running the REFERENCE's own Discriminator (models/discriminator.py,
with models/diff_aug.py) on the CPU.

Run where a reference checkout is available (the GPU test machines need none):

    python tests/golden/make_disc_golden.py /path/to/reference

Per case (imsize 64 at 64x64 with B = 2, imsize -1 at 63x84 and at 56x70 with B = 1), under np.random.seed(s) and
torch.manual_seed(s) in training mode: build Discriminator(False, 'color,cutout', imsize=...); one generator-step
call D(fake) with -mean backward to the input; then a discriminator-step pair D(real), D(fake2.detach()) with the
hinge loss backward to the weights.  The inputs come from a separate torch.Generator(1000 + s), so they are not
stored.  Stored: every np.random.random() value the calls drew (to show which calls augmented), the outputs, the
input gradient, each call's sigma per layer (u . W v from the post-call buffers), the initial and the final u / v,
a seeded sample and the norm of every initial weight and of every weight gradient, and the next np.random.random()
and torch.rand(4) after the sequence.  The weights are not stored: they regenerate from the seed.  Each case's seed
is the first from its start whose three calls include one that augments and one that does not.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [("b64", 64, 64, 64, 2, 0), ("llff", -1, 63, 84, 1, 10), ("dtu", -1, 56, 70, 1, 20)]
N_SAMPLE = 64


def _sigma(m):
    w = m.weight_orig.detach().double().reshape(m.weight_orig.shape[0], -1)
    return float(torch.dot(m.weight_u.double(), w @ m.weight_v.double()))


def run_case(Disc, imsize, H, W, B, seed):
    gates = []
    orig = np.random.random

    def rec(*a):
        v = orig(*a)
        gates.append(v)
        return v

    np.random.seed(seed)
    torch.manual_seed(seed)
    D = Disc(False, "color,cutout", imsize=imsize)
    convs = [m for m in D.main if isinstance(m, torch.nn.Conv2d)]
    out = {"u0": np.concatenate([m.weight_u.numpy() for m in convs]).astype(np.float32),
           "v0": np.concatenate([m.weight_v.numpy() for m in convs]).astype(np.float32)}
    rng = np.random.default_rng(7)
    idx = [rng.integers(0, m.weight_orig.numel(), N_SAMPLE) for m in convs]
    out["sample_idx"] = np.stack(idx)
    out["w0_sample"] = np.stack([m.weight_orig.detach().reshape(-1).numpy()[i] for m, i in zip(convs, idx)])
    out["w0_norm"] = np.array([float(m.weight_orig.detach().double().norm()) for m in convs])
    g = torch.Generator().manual_seed(1000 + seed)
    fake, real, fake2 = (torch.rand(B, 3, H, W, generator=g) for _ in range(3))
    np.random.random = rec
    try:
        calls = []
        xf = fake.clone().requires_grad_(True)
        pf = D(xf)
        calls.append(len(gates))
        sig_g = [_sigma(m) for m in convs]
        (-pf.mean()).backward()
        D.zero_grad(set_to_none=True)
        pr = D(real)
        calls.append(len(gates))
        sig_r = [_sigma(m) for m in convs]
        pf2 = D(fake2.detach())
        calls.append(len(gates))
        sig_f = [_sigma(m) for m in convs]
        ((F.relu(1 - pr).mean() + F.relu(1 + pf2).mean()) / 2).backward()
    finally:
        np.random.random = orig
    fired = []
    lo = 0
    for hi in calls:
        v = gates[lo:hi]
        fired.append(len(v) == 2 and v[0] > 0.5 and v[1] >= 0.5)
        lo = hi
    out.update({
        "gates": np.array(gates), "gate_ends": np.array(calls), "fired": np.array(fired),
        "out_g": pf.detach().numpy(), "dx_g": xf.grad.numpy(), "out_real": pr.detach().numpy(),
        "out_fake": pf2.detach().numpy(), "sigma": np.array([sig_g, sig_r, sig_f]),
        "u1": np.concatenate([m.weight_u.numpy() for m in convs]).astype(np.float32),
        "v1": np.concatenate([m.weight_v.numpy() for m in convs]).astype(np.float32),
        "dw_sample": np.stack([m.weight_orig.grad.reshape(-1).numpy()[i] for m, i in zip(convs, idx)]),
        "dw_norm": np.array([float(m.weight_orig.grad.double().norm()) for m in convs]),
        "next_np": np.array(np.random.random()), "next_torch": torch.rand(4).numpy(),
    })
    return out, fired


def main():
    if len(sys.argv) < 2:
        sys.exit("usage: python tests/golden/make_disc_golden.py /path/to/reference")
    ref = sys.argv[1]
    sys.path.insert(0, ref)
    from models.discriminator import Discriminator
    data = {}
    for name, imsize, H, W, B, start in CASES:
        for seed in range(start, start + 100):
            out, fired = run_case(Discriminator, imsize, H, W, B, seed)
            if any(fired) and not all(fired):
                break
        else:
            raise RuntimeError(f"{name}: no seed in range gives a mixed sequence")
        print(f"{name}: seed {seed}, augmentation fired per call {fired}")
        data[f"{name}/meta"] = np.array([imsize, H, W, B, seed])
        for k, v in out.items():
            data[f"{name}/{k}"] = v
    path = os.path.join(HERE, "discriminator.npz")
    np.savez_compressed(path, **data)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
