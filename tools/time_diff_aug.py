#!/usr/bin/env python
"""CUDA-event times of the standalone DiffAugment (sinnerf_b200.discriminator.DiffAugment) against the oracle
(tests/diff_aug_oracle.py) run as fp32 PyTorch on the same GPU -- the reference's augmentation ops:

  1. one call, forward and forward + input gradient, policies 'color,cutout' (the default) and
     'color,translation,cutout', at the recipes' patch shapes 64x64, 63x84 and 56x70, B = 1 and 2, on the
     '(b p q) c -> b c p q' view of a ray-major tensor that requires grad;
  2. the dloss='relavistic' generator step's D(DiffAugment(real_patch)) with the library's Discriminator
     (policy 'color,cutout', imsize 64 / -1), forward and the weight gradients of its mean, with either augmentation.
Every timed call augments: the draws are made with the reference's calls (diff_augment_draws' per-op draws, on the
device) but without the gate, which would skip half the calls on either side.  Implementations alternate within each
round; min and median over rounds.  The card's name, power limit and SM clocks are read in the same run.

    python tools/time_diff_aug.py [--calls 200] [--rounds 7]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sinnerf_b200 import discriminator as disc  # noqa: E402
from tests import diff_aug_oracle as oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=200, help="calls per timed window")
ap.add_argument("--rounds", type=int, default=7)
args = ap.parse_args()
dev = torch.device("cuda:0")


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, n):
    """{name: (min, median)} ms per call; implementations alternate within a round"""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, f in fns.items():
            ts[k].append(timed(f, n))
    return {k: (min(v), statistics.median(v)) for k, v in ts.items()}


def fmt(r):
    return " | ".join(f"{k} min {v[0]:.4f} med {v[1]:.4f}" for k, v in r.items())


def draws(policy, shape):
    B, _, H, W = shape
    return [(p, disc._DRAWS[p](B, H, W, dev)) for p in policy.split(",")]


def fused(x, policy):
    return disc._DiffAugFn.apply(x, True, draws(policy, tuple(x.shape)))


def reference(x, policy):
    return oracle.diff_augment(x, draws(policy, tuple(x.shape)))


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                      "-i", "0"], capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi name, power.limit, clocks.sm, clocks.max.sm: {smi}")
torch.manual_seed(0)
g = torch.Generator().manual_seed(0)
impls = {"reference fp32 torch": reference, "fused": fused}

# ---- 1. one call
for policy in ("color,cutout", "color,translation,cutout"):
    for H, W in ((64, 64), (63, 84), (56, 70)):
        for B in (1, 2):
            rays = torch.rand(B * H * W, 3, generator=g).to(dev).requires_grad_(True)
            x = rays.view(B, H, W, 3).permute(0, 3, 1, 2)
            w = torch.rand(B, 3, H, W, generator=g).to(dev)
            fwd = {k: (lambda f=f: f(x.detach(), policy)) for k, f in impls.items()}
            bwd = {k: (lambda f=f: (f(x, policy) * w).sum().backward()) for k, f in impls.items()}
            print(f"{policy:24s} {H}x{W} B={B} forward, ms/call: {fmt(alternate(fwd, args.calls))}")
            print(f"{policy:24s} {H}x{W} B={B} forward + input grad, ms/call: {fmt(alternate(bwd, args.calls))}")

# ---- 2. the relavistic generator step's D(DiffAugment(real_patch))
for imsize, (H, W) in ((64, (64, 64)), (-1, (63, 84)), (-1, (56, 70))):
    D = disc.Discriminator(False, "color,cutout", imsize=imsize).to(dev)
    real = torch.rand(1, 3, H, W, generator=g).to(dev)
    step = {k: (lambda f=f: D(f(real, "color,cutout")).mean().backward()) for k, f in impls.items()}
    print(f"relavistic D(DiffAugment(real)) {H}x{W} B=1 forward + weight grads, ms/call: "
          f"{fmt(alternate(step, args.calls // 4))}")
