#!/usr/bin/env python
"""CUDA-event times of opt_d's step -- get_optimizer(hparams, [D], rate=0.2) -- fused (one snb_optim_step_tensors
launch) against the optimiser it replaces, on the discriminator's weight_orig tensors at imsize 64 (5 tensors,
2.76 M parameters) and -1 (3 tensors, 2.12 M):

  adam    torch.optim.Adam as get_optimizer builds it (default foreach path on CUDA)
  sgd     torch.optim.SGD, momentum 0.9 (default foreach path)
  radam / ranger   the reference's rules (oracle/optim_oracle.py: one ATen kernel per operation and tensor)

The gradients come from one real discriminator step (hinge loss on two 2-image batches).  Fused and replaced are timed
in alternated rounds of --steps steps each; min and median over --rounds rounds of the mean step time (CUDA events
around back-to-back step() calls: whichever of the host and the device is slower sets it).  A separate torch.profiler
pass then gives the device side alone: the kernels per step and their summed duration.

    python tools/time_disc_optim.py [--steps 50] [--rounds 11]
"""
import argparse
import copy
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from oracle import optim_oracle  # noqa: E402
from sinnerf_b200.discriminator import Discriminator  # noqa: E402
from sinnerf_b200.optim import get_optimizer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=50, help="optimiser steps per timed round")
ap.add_argument("--rounds", type=int, default=11)
args = ap.parse_args()
dev = torch.device("cuda:0")
LR, RATE = 5e-4, 0.2


class HParams:
    lr, momentum, weight_decay = LR, 0.9, 0.0

    def __init__(self, optimizer):
        self.optimizer = optimizer


REPLACED = {   # the optimiser the reference's get_optimizer builds over D.parameters() (utils/__init__.py:10-31)
    "adam": lambda ps: torch.optim.Adam(ps, lr=LR * RATE, eps=1e-8),
    "sgd": lambda ps: torch.optim.SGD(ps, lr=LR * RATE, momentum=0.9),
    "radam": lambda ps: optim_oracle.RAdam(ps, lr=LR * RATE, eps=1e-8),
    "ranger": lambda ps: optim_oracle.Ranger(ps, lr=LR * RATE, eps=1e-8),
}
SHAPES = {64: (64, 64), -1: (63, 84)}


def discriminator_with_grads(imsize):
    torch.manual_seed(0)
    np.random.seed(0)
    d = Discriminator(False, "color,cutout", imsize=imsize).to(dev)
    H, W = SHAPES[imsize]
    real, fake = torch.rand(2, 3, H, W, device=dev), torch.rand(2, 3, H, W, device=dev)
    (F.relu(1 - d(real)).mean() + F.relu(1 + d(fake)).mean()).backward()
    return d


def round_ms(opt, n):
    """Mean ms per step of n back-to-back steps (CUDA events)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        opt.step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_us(opt, n=20):
    """(kernels per step, summed kernel microseconds per step) over n steps under torch.profiler."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            opt.step()
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(ks) / n, sum(e.time_range.elapsed_us() for e in ks) / n


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi: {gpu}")
print(f"opt_d step, ms per step: min / median over {args.rounds} alternated rounds of {args.steps} steps")
for imsize in (64, -1):
    base = discriminator_with_grads(imsize)
    n_params = sum(p.numel() for p in base.parameters())
    for rule, make_replaced in REPLACED.items():
        opts = {}
        for impl in ("fused", "replaced"):
            d = copy.deepcopy(base)
            for p, q in zip(d.parameters(), base.parameters()):
                p.grad = q.grad.clone()
            opts[impl] = get_optimizer(HParams(rule), [d], rate=RATE) if impl == "fused" else \
                make_replaced(list(d.parameters()))
            for _ in range(3):                     # warm-up: state creation, first launches
                opts[impl].step()
        torch.cuda.synchronize()
        times = {"fused": [], "replaced": []}
        for r in range(args.rounds):
            order = ("fused", "replaced") if r % 2 == 0 else ("replaced", "fused")
            for impl in order:
                times[impl].append(round_ms(opts[impl], args.steps))
        cells = []
        for impl in ("fused", "replaced"):
            t = sorted(times[impl])
            cells.append(f"{impl} {t[0]:.4f} / {t[len(t) // 2]:.4f}")
        ratio = sorted(times["replaced"])[len(times["replaced"]) // 2] / sorted(times["fused"])[len(times["fused"]) // 2]
        dev_side = []
        for impl in ("fused", "replaced"):
            k, us = kernel_us(opts[impl])
            dev_side.append(f"{impl} {k:.0f} kernels {us:.1f} us")
        print(f"  imsize {imsize:3d} ({len(list(base.parameters()))} tensors, {n_params / 1e6:.2f} M)  {rule:6s}  "
              f"{cells[0]}   {cells[1]}   (median ratio {ratio:.1f}x)   device: {dev_side[0]}, {dev_side[1]}")
