#!/usr/bin/env python
"""Time the sigma-only training pass: a BASELINE.json configs[4]-shaped step (4 x 4096 rays, 64 + 64 samples,
perturb = noise_std = 1, forward + backward) with and without test_time, and the sigma-only coarse pass alone
(render_rays(test_time=True)'s coarse field pass + weights-only compositing, forward + backward), with CUDA events.
Prints the card's name and power limit beside the numbers.

    python tools/time_sigma_train.py [--rays 4096] [--calls 4] [--iters 10]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sinnerf_b200 import _lib, config, synthetic  # noqa: E402
from sinnerf_b200.nerf import Embedding, NeRF  # noqa: E402
from sinnerf_b200.rendering import _SigmaPass, _linspace01, render_rays  # noqa: E402
from sinnerf_b200.synthetic import default_init_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rays", type=int, default=4096)
ap.add_argument("--calls", type=int, default=4)
ap.add_argument("--iters", type=int, default=10)
args = ap.parse_args()
dev = torch.device("cuda:0")
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi: {gpu} | precision {config.get_precision()}, "
      f"train storage {config.get_train_storage()}")
models = []
for seed in (0, 1):
    m = NeRF(use_new_activation=True)
    m.load_state_dict(default_init_params(seed))
    models.append(m.to(dev))
emb = [Embedding(3, 10), Embedding(3, 4)]
batches = [synthetic.random_rays("lego", args.rays, seed=i).to(dev) for i in range(args.calls)]
target = torch.rand(args.rays, 3, device=dev)


def step(test_time):
    for m in models:
        m.zero_grad(set_to_none=True)
    loss = 0.0
    for r in batches:
        out = render_rays(models, emb, r, 64, False, 1.0, 1.0, 64, 32768, True, test_time=test_time)
        loss = loss + ((out["rgb_fine"] - target) ** 2).mean() + 0.1 * out["depth_fine"].mean() \
            + 0.01 * out["opacity_coarse"].sum(1).mean()
        if not test_time:
            loss = loss + ((out["rgb_coarse"] - target) ** 2).mean()
    loss.backward()


# the coarse sigma-only pass alone: fixed stratified depths, the same field + compositing forward and backward
prec = _lib.precision_id(config.get_precision())
zs = []
for r in batches:
    t = _linspace01(64, dev)
    zs.append((r[:, 6:7] * (1 - t) + r[:, 7:8] * t).contiguous())
noise = [torch.randn(args.rays, 64, device=dev) for _ in batches]


def coarse_alone():
    models[0].zero_grad(set_to_none=True)
    loss = 0.0
    for r, z, nz in zip(batches, zs, noise):
        w = _SigmaPass.apply(models[0], prec, r, z, nz, 1.0, True, *models[0]._param_list())
        loss = loss + w.sum(1).mean()
    loss.backward()


def timed(fn, *a):
    fn(*a)
    torch.cuda.synchronize()
    ts = []
    for _ in range(args.iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*a)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[0], ts[len(ts) // 2]


n = args.rays * args.calls
# alternate the two steps so drift of the shared machine hits both alike
res = {"full": [], "test_time": []}
for _ in range(2):
    res["full"].append(timed(step, False))
    res["test_time"].append(timed(step, True))
for k, v in res.items():
    best = min(x[0] for x in v)
    med = sorted(x[1] for x in v)[len(v) // 2]
    print(f"train step {k:>9}: {args.calls} x {args.rays} rays, 64+64, fwd+bwd  min {best:.2f} ms  median {med:.2f} ms")
best, med = timed(coarse_alone)
print(f"sigma-only coarse pass alone: {args.calls} x {args.rays} rays x 64 samples, fwd+bwd  min {best:.2f} ms  "
      f"median {med:.2f} ms  ({n * 64 / best / 1e3:.1f} M points/s)")
print(f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
