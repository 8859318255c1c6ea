#!/usr/bin/env python
"""CUDA-event times of the wgan_gp discriminator step on the GPU: Discriminator.forward_with_penalty (csrc/disc.cu)
against the oracle (tests/disc_oracle.py) run as fp32 PyTorch on the same GPU through
torch.autograd.grad(create_graph=True), with cuDNN and TF32 off, then on.  One step is the real call with its
penalty, the fake call, compute_loss(fake, 0) + compute_loss(real, 1) + 10 reg.mean() and the backward to the
weights, at the recipes' patch shapes with B = 1: 64x64 (blender, imsize 64), 63x84 (LLFF) and 56x70 (DTU)
(imsize -1).  Every call makes its own DiffAugment draws from the global generators, as in training.
Implementations alternate within each round; min and median over rounds.  The card's name, power limit and SM clocks
are read in the same run.

    python tools/time_disc_penalty.py [--steps 50] [--rounds 7]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sinnerf_b200.discriminator import Discriminator, draw_augment  # noqa: E402
from tests import disc_oracle as oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=50, help="steps per timed window")
ap.add_argument("--rounds", type=int, default=7)
args = ap.parse_args()
dev = torch.device("cuda:0")


def fast_torch(on):
    torch.backends.cuda.matmul.allow_tf32 = on
    torch.backends.cudnn.allow_tf32 = on
    torch.backends.cudnn.enabled = on


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, n):
    """{name: (min, median)} ms per step; each entry is (cudnn + tf32 flag, fn); implementations alternate in a round"""
    for on, f in fns.values():
        fast_torch(on)
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, (on, f) in fns.items():
            fast_torch(on)
            ts[k].append(timed(f, n))
    fast_torch(True)
    return {k: (min(v), statistics.median(v)) for k, v in ts.items()}


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                      "-i", "0"], capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi name, power.limit, clocks.sm, clocks.max.sm: {smi}")
np.random.seed(0)
torch.manual_seed(0)
g = torch.Generator().manual_seed(0)


class OracleD:
    """the oracle as an fp32 PyTorch module: its own u / v state, draws made like the drop-in's"""

    def __init__(self, D):
        self.imsize = D.imsize
        self.ws = [m.weight_orig.detach().clone().requires_grad_(True) for m in D.convs()]
        self.us = [m.weight_u.clone() for m in D.convs()]
        self.vs = [m.weight_v.clone() for m in D.convs()]

    def __call__(self, x):
        aug = draw_augment("color,cutout", tuple(x.shape), x.device)
        out, self.us, self.vs, _ = oracle.forward(self.ws, self.us, self.vs, x, self.imsize, True, aug)
        return out

    def forward_with_penalty(self, x):
        x = x.detach().requires_grad_(True)
        out = self(x)
        (gx,) = torch.autograd.grad(out.sum(), x, create_graph=True)
        return out, gx.pow(2).flatten(1).sum(1)


for name, imsize, (H, W) in (("blender", 64, (64, 64)), ("llff", -1, (63, 84)), ("dtu", -1, (56, 70))):
    D = Discriminator(False, "color,cutout", imsize=imsize).to(dev)
    O = OracleD(D)
    real = torch.rand(1, 3, H, W, generator=g).to(dev)
    fake = torch.rand(1, 3, H, W, generator=g).to(dev)

    def step(m):
        def f():
            pred_real, reg_real = m.forward_with_penalty(real)
            pred_fake = m(fake)
            # compute_loss(fake, 0) + compute_loss(real, 1) + 10 compute_grad2(real).mean()
            loss_d = -pred_fake.mean() + pred_real.mean() + 10 * reg_real.mean()
            loss_d.backward()
        return f
    r = alternate({"oracle fp32": (False, step(O)), "oracle cudnn+tf32": (True, step(O)), "fused": (False, step(D))},
                  args.steps)
    print(f"{name:8s} {H}x{W} wgan_gp D step (2 calls, penalty, weight grads), ms/step: " +
          " | ".join(f"{k} min {v[0]:.3f} med {v[1]:.3f}" for k, v in r.items()))
