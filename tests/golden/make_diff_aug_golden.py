#!/usr/bin/env python
"""Generate tests/golden/diff_aug.npz by running the REFERENCE's own DiffAugment (models/diff_aug.py) on the CPU.

Run where a reference checkout is available (the GPU test machines need none):

    python tests/golden/make_diff_aug_golden.py /path/to/reference

Cases: every policy of POLICIES at every shape of SHAPES, B = 1 and 3, once with a numpy seed whose gate draw skips
the augmentation and once with one whose gate applies it.  Each case seeds np.random and torch, draws its (B, 3, H, W)
input from a separate torch.Generator(input_seed) (the input is not stored, only its seed), and calls
DiffAugment(x, policy) in fp32 as training does, recording every np.random.random(), torch.rand and torch.randint
value the call drew, then the next np.random.random() and torch.rand(4) after it.  The reference's code is then run
again on x in float64 with the recorded draws replayed (torch.rand draws in fp32 and casts, so a float64 run would
otherwise draw other values): that output is the one stored, so a float64 restatement can be held to it at 1e-12.
Stored per applied case: each image and channel's float64 output sum, and the float64 output at every element for
images of at most 1024 elements, else at 512 fixed positions (flat indices stored), plus the fp32 output there.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
POLICIES = ["color", "translation", "cutout", "color,cutout", "color,translation,cutout", "translation,cutout",
            "cutout,color"]
SHAPES = [(64, 64), (63, 84), (56, 70), (7, 9)]
BATCHES = [1, 3]
N_SAMPLE = 512


def gate_seed(fire, start):
    """first numpy seed from start whose first draw applies (fire) or skips DiffAugment (np.random.random() < 0.5)"""
    for s in range(start, start + 1000):
        np.random.seed(s)
        if (np.random.random() >= 0.5) == fire:
            return s
    raise AssertionError


def run(diff_aug, x, policy, np_seed, torch_seed, replay=None):
    """DiffAugment(x, policy) under the seeds -> (out, recorded draws, np draws, (next np value, next torch.rand(4)));
    replay: draws to hand back instead of drawing (cast to the requested dtype)"""
    rand, randint, npr = torch.rand, torch.randint, np.random.random
    rec, nps = [], []

    def rec_rand(*a, **k):
        if replay is not None:
            return replay.pop(0).to(k.get("dtype", torch.float32))
        v = rand(*a, **k)
        rec.append(v.clone())
        return v

    def rec_randint(*a, **k):
        if replay is not None:
            return replay.pop(0).clone()
        v = randint(*a, **k)
        rec.append(v.clone())
        return v

    def rec_np(*a):
        v = npr(*a)
        nps.append(v)
        return v

    np.random.seed(np_seed)
    torch.manual_seed(torch_seed)
    torch.rand, torch.randint, np.random.random = rec_rand, rec_randint, rec_np
    try:
        out = diff_aug.DiffAugment(x, policy)
    finally:
        torch.rand, torch.randint, np.random.random = rand, randint, npr
    after = (np.random.random(), torch.rand(4))
    return out, rec, nps, after


def main(ref):
    sys.path.insert(0, ref)
    from models import diff_aug

    data = {"policies": np.array(POLICIES)}
    i = 0
    for pi, policy in enumerate(POLICIES):
        for (H, W) in SHAPES:
            for B in BATCHES:
                for fire in (False, True):
                    np_seed = gate_seed(fire, 100 * i)
                    torch_seed, input_seed = 1000 + i, 2000 + i
                    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(input_seed))
                    out, rec, nps, after = run(diff_aug, x, policy, np_seed, torch_seed)
                    assert (out is x) != fire
                    k = f"c{i}_"
                    data[k + "meta"] = np.array([pi, H, W, B, int(fire), np_seed, torch_seed, input_seed])
                    data[k + "np_draws"] = np.array(nps)
                    data[k + "after_np"] = np.array(after[0])
                    data[k + "after_torch"] = after[1].numpy()
                    data[k + "n_draws"] = np.array(len(rec))
                    for j, t in enumerate(rec):
                        data[k + f"draw{j}"] = t.reshape(B).numpy()
                    if fire:
                        out64, _, _, _ = run(diff_aug, x.double(), policy, np_seed, torch_seed, replay=list(rec))
                        if "color" not in policy:
                            assert torch.equal(out64, out.double())
                        numel = 3 * H * W
                        idx = (np.arange(B * numel) if numel <= 1024 else
                               np.sort(np.random.default_rng(i).choice(B * numel, N_SAMPLE, replace=False)))
                        data[k + "idx"] = idx
                        data[k + "out64"] = out64.reshape(-1).numpy()[idx]
                        data[k + "out32"] = out.reshape(-1).numpy()[idx]
                        data[k + "sum64"] = out64.sum((2, 3)).numpy()
                    i += 1
    data["n_cases"] = np.array(i)
    path = os.path.join(HERE, "diff_aug.npz")
    np.savez_compressed(path, **data)
    print(path, i, "cases")


if __name__ == "__main__":
    if len(sys.argv) < 2:
        sys.exit("usage: python tests/golden/make_diff_aug_golden.py /path/to/reference")
    main(sys.argv[1])
