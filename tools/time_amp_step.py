#!/usr/bin/env python
"""Time GradScaler-native stepping of the fused optimisers against the plain path (`amp_scaling=False`: GradScaler's
own unscale pass, then a host read of found_inf before every step).

1. Host time `scaler.step(opt)` blocks with ~200 ms of GPU work queued ahead of it (FusedAdam over the two NeRF
   models, and over a Discriminator).
2. The configs[4]-shaped training step of tools/time_train.py (four render_rays calls of 4096 rays, 64 + 64 samples,
   perturb 1, noise_std 1) under fp16 autocast with set_precision('autocast') and a GradScaler, stepped by FusedAdam;
   with a discriminator, also the adversarial part of a SinNeRF step: the first batch's rgb_fine as a 64x64 patch
   into D (dis_weight 0.01) and a hinge discriminator step stepped by opt_d.  Wall time per step over --steps steps
   ending in a synchronise; the two paths alternate within each round; min and median over --rounds rounds.

    python tools/time_amp_step.py [--rounds 7] [--steps 10]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import sinnerf_b200  # noqa: E402
from sinnerf_b200 import synthetic  # noqa: E402
from sinnerf_b200.discriminator import Discriminator  # noqa: E402
from sinnerf_b200.nerf import Embedding, NeRF  # noqa: E402
from sinnerf_b200.optim import FusedAdam  # noqa: E402
from sinnerf_b200.rendering import render_rays  # noqa: E402
from sinnerf_b200.synthetic import default_init_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=10)
args = ap.parse_args()
dev = torch.device("cuda:0")
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi name, power.limit, clocks.max.sm: {smi}")
sinnerf_b200.set_precision("autocast")


def nerfs():
    ms = []
    for seed in (0, 1):
        m = NeRF(use_new_activation=True)
        m.load_state_dict(default_init_params(seed))
        ms.append(m.to(dev))
    return ms


def disc():
    torch.manual_seed(0)
    return Discriminator(False, "color,cutout", imsize=64).to(dev)


def sleep_cycles(seconds):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    torch.cuda._sleep(10 ** 7)
    end.record()
    end.synchronize()
    return int(seconds * 10 ** 7 / (start.elapsed_time(end) * 1e-3))


# ---------------------------------------------------------------- 1. host time of scaler.step behind queued work
SLEEP = sleep_cycles(0.2)
print("\n1. host ms of scaler.step(opt) with ~200 ms of GPU work queued (min / median of 5)")
for name, make in (("FusedAdam, two NeRF models", nerfs), ("FusedAdam, Discriminator imsize 64", lambda: [disc()])):
    for amp_scaling in (False, True):
        models = make()
        opt = FusedAdam(models, amp_scaling=amp_scaling)
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
        ps = [p for group in opt.param_groups for p in group["params"]]
        ts = []
        for i in range(7):
            for p in ps:
                p.grad = scaler.scale(torch.full_like(p, 1e-3))
            torch.cuda.synchronize()
            torch.cuda._sleep(SLEEP)
            t0 = time.perf_counter()
            scaler.step(opt)
            t1 = time.perf_counter()
            scaler.update()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append((t1 - t0) * 1e3)
        path = "GradScaler-native" if amp_scaling else "plain (amp_scaling=False)"
        print(f"   {name:36s} {path:26s} {min(ts):8.3f} / {statistics.median(ts):8.3f}")

# ---------------------------------------------------------------- 2. the configs[4]-shaped step
emb = [Embedding(3, 10), Embedding(3, 4)]
batches = [synthetic.random_rays("lego", 4096, seed=i).to(dev) for i in range(4)]
target = torch.rand(4096, 3, device=dev)
real = torch.rand(1, 3, 64, 64, device=dev)


class Trainer:
    def __init__(self, amp_scaling, with_d):
        self.models = nerfs()
        self.opt = FusedAdam(self.models, lr=5e-4, amp_scaling=amp_scaling)
        self.d = disc() if with_d else None
        self.opt_d = FusedAdam([self.d], lr=1e-4, amp_scaling=amp_scaling) if with_d else None
        self.scaler = torch.amp.GradScaler("cuda")

    def step(self):
        self.opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            outs = [render_rays(self.models, emb, r, 64, False, 1.0, 1.0, 64, 32768, True) for r in batches]
            loss = 0.0
            for out in outs:
                loss = loss + ((out["rgb_coarse"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean() \
                    + 0.1 * out["depth_fine"].mean()
            if self.d is not None:
                fake = outs[0]["rgb_fine"].float().view(64, 64, 3).permute(2, 0, 1)[None].contiguous()
                loss = loss - 0.01 * self.d(fake).mean()
        self.scaler.scale(loss).backward()
        self.scaler.step(self.opt)
        if self.d is not None:
            self.opt_d.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.float16):
                loss_d = F.relu(1 - self.d(real)).mean() + F.relu(1 + self.d(fake.detach())).mean()
            self.scaler.scale(loss_d).backward()
            self.scaler.step(self.opt_d)
        self.scaler.update()


print(f"\n2. configs[4]-shaped fp16-autocast training step + GradScaler + FusedAdam, ms per step "
      f"(min / median of {args.rounds} rounds of {args.steps} steps)")
for with_d in (False, True):
    trainers = {amp: Trainer(amp, with_d) for amp in (False, True)}
    for t in trainers.values():
        for _ in range(3):
            t.step()
    torch.cuda.synchronize()
    times = {amp: [] for amp in trainers}
    for _ in range(args.rounds):
        for amp, t in trainers.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                t.step()
            torch.cuda.synchronize()
            times[amp].append((time.perf_counter() - t0) * 1e3 / args.steps)
    label = "with a discriminator step" if with_d else "NeRF only"
    for amp in trainers:
        path = "GradScaler-native" if amp else "plain (amp_scaling=False)"
        print(f"   {label:26s} {path:26s} {min(times[amp]):8.2f} / {statistics.median(times[amp]):8.2f}")
