#!/usr/bin/env python
"""CUDA-event times of the optimiser step, fused against the optimiser it replaces (torch.optim.Adam on its default
foreach path; oracle/optim_oracle.py: the reference's SGD / RAdam / Ranger restated with torch ops, one ATen kernel per
operation and tensor):

  1. one optimiser step over both NeRFs (48 tensors, 1.19 M parameters).  The fused step includes the re-pack of the
     weight images; the replaced step leaves them stale, and the next forward re-packs them (counted in 2.);
  2. the tools/time_train.py training step (4 x 4096 rays, 64 + 64 samples, forward + backward) followed by the step.

    python tools/time_optim.py [--steps 50] [--iters 5] [--rays 4096] [--calls 4]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import optim_oracle  # noqa: E402
from sinnerf_b200 import synthetic  # noqa: E402
from sinnerf_b200.nerf import NeRF, Embedding  # noqa: E402
from sinnerf_b200.optim import FusedAdam, FusedRAdam, FusedRanger, FusedSGD  # noqa: E402
from sinnerf_b200.rendering import render_rays  # noqa: E402
from sinnerf_b200.synthetic import default_init_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=50, help="optimiser steps per timed window (part 1)")
ap.add_argument("--iters", type=int, default=5, help="timed training steps per optimiser (part 2)")
ap.add_argument("--rays", type=int, default=4096)
ap.add_argument("--calls", type=int, default=4)
args = ap.parse_args()
dev = torch.device("cuda:0")
LR, WD = 5e-4, 0.0

# name -> (fused, replaced) constructors with get_optimizer's arguments (reference utils/__init__.py:15-27)
OPTIMIZERS = {
    "adam": (lambda ms: FusedAdam(ms, lr=LR, eps=1e-8, weight_decay=WD),
             lambda ps: torch.optim.Adam(ps, lr=LR, eps=1e-8, weight_decay=WD)),
    "sgd": (lambda ms: FusedSGD(ms, lr=LR, momentum=0.9, weight_decay=WD),
            lambda ps: optim_oracle.SGD(ps, lr=LR, momentum=0.9, weight_decay=WD)),
    "radam": (lambda ms: FusedRAdam(ms, lr=LR, eps=1e-8, weight_decay=WD),
              lambda ps: optim_oracle.RAdam(ps, lr=LR, eps=1e-8, weight_decay=WD)),
    "ranger": (lambda ms: FusedRanger(ms, lr=LR, eps=1e-8, weight_decay=WD),
               lambda ps: optim_oracle.Ranger(ps, lr=LR, eps=1e-8, weight_decay=WD)),
}


def fresh_models():
    ms = []
    for seed in (0, 1):
        m = NeRF(use_new_activation=True)
        m.load_state_dict(default_init_params(seed))
        ms.append(m.to(dev))
    return ms


def timed(fn, n):
    """ms per call: CUDA events around n calls, after 3 warm-up calls."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi: {gpu}")

# ---- 1. the optimiser step alone (synthetic gradients of the training step's magnitude)
print(f"\n1. one optimiser step over both models (mean of {args.steps} steps)")
g = torch.Generator(device=dev).manual_seed(0)
for name, (make_fused, make_replaced) in OPTIMIZERS.items():
    row = []
    for impl in ("fused", "replaced"):
        ms = fresh_models()
        for p in (p for m in ms for p in m.parameters()):
            p.grad = torch.randn(p.shape, device=dev, generator=g) * 1e-3
        opt = make_fused(ms) if impl == "fused" else make_replaced([p for m in ms for p in m.parameters()])
        row.append(timed(opt.step, args.steps))
    print(f"  {name:7s} fused {row[0]:7.3f} ms   replaced {row[1]:7.3f} ms   ({row[1] / row[0]:.1f}x)")

# ---- 2. the training step of tools/time_train.py followed by the optimiser step
print(f"\n2. training step ({args.calls} x {args.rays} rays, 64+64 samples, fwd + bwd) + optimiser step "
      f"(min of {args.iters})")
emb = [Embedding(3, 10), Embedding(3, 4)]
batches = [synthetic.random_rays("lego", args.rays, seed=i).to(dev) for i in range(args.calls)]
target = torch.rand(args.rays, 3, device=dev)


def train_step(models, opt):
    for m in models:
        m.zero_grad(set_to_none=True)
    loss = 0.0
    for r in batches:
        out = render_rays(models, emb, r, 64, False, 1.0, 1.0, 64, 32768, True)
        loss = loss + ((out["rgb_coarse"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean() \
            + 0.1 * out["depth_fine"].mean()
    loss.backward()
    opt.step()


rows = []
for name, (make_fused, make_replaced) in OPTIMIZERS.items():
    rows.append((name, "fused", make_fused))
    rows.append((name, "replaced", lambda ms, mk=make_replaced: mk([p for m in ms for p in m.parameters()])))
for name, impl, make in rows:
    ms = fresh_models()
    opt = make(ms)
    train_step(ms, opt)
    torch.cuda.synchronize()
    ts = []
    for _ in range(args.iters):
        ts.append(timed(lambda: train_step(ms, opt), 1))
    print(f"  {name:7s} {impl:6s} {min(ts):7.2f} ms   (median {sorted(ts)[len(ts) // 2]:.2f})")
