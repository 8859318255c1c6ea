#!/usr/bin/env python
"""CUDA-event times of sinnerf_b200.warp.forward_warp at the shapes the reference datasets warp, with seeded synthetic
depth (about 40 % holes, so the contended hole group is in the timing):

  400x400, 1 pose,    last     blender rot3d, once per training sample (DataLoader worker)
  400x400, 125 poses, last     blender rot3d at construction (--angle 20: 5^3 poses)
  504x378, 41 poses,  zbuffer  LLFF at construction (one per pose of the scene)
  640x512, 3 poses,   zbuffer  DTU at construction (one per source view)

Reports ms per call and per pose, and the algorithmic bytes -- 4 B depth read + 17 B of outputs per pixel and pose,
+ 12 B image gather per hit -- over the time, against the H100 SXM's 3.35 TB/s.  The numpy oracle's time
(tests/warp_oracle.py, one CPU thread of whatever host runs this) is an informational row, not the reference.

    python tools/time_warp.py [--rounds 7] [--iters 20]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sinnerf_b200.warp import forward_warp, warp_matrices  # noqa: E402
from tests import warp_oracle  # noqa: E402
from tests.warp_scenes import proj, random_poses, scene  # noqa: E402

SHAPES = [("rot3d per sample", 400, 400, 1, "last"), ("rot3d construction", 400, 400, 125, "last"),
          ("LLFF construction", 378, 504, 41, "zbuffer"), ("DTU construction", 512, 640, 3, "zbuffer")]
HBM_BYTES_PER_S = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--iters", type=int, default=20, help="calls per timed window")
args = ap.parse_args()
dev = torch.device("cuda:0")
assert torch.cuda.is_available(), "tools/time_warp.py needs a GPU"
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.TimeoutExpired):
    card = torch.cuda.get_device_name(0) + ", power limit unknown"
print(f"# {card}")
print("| case | H x W | poses | occlusion | ms / call (min, median) | ms / pose | GB/s (share of 3.35 TB/s) | "
      "numpy oracle ms / pose |")
print("|---|---|---|---|---|---|---|---|")
for name, H, W, P, occ in SHAPES:
    image, depth = scene(H, W, seed=H + P, holes=0.4)
    src = random_poses(H, W, P, seed=P)
    src_arg = src[0] if P == 1 else src
    im, d = torch.from_numpy(image).to(dev), torch.from_numpy(depth).to(dev)
    fn = lambda: forward_warp(im, d, proj(H, W), src_arg, occlusion=occ)   # noqa: E731
    out = fn()
    torch.cuda.synchronize()
    hits = int(out[2].sum())
    times = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / args.iters)
    t_min, t_med = min(times), statistics.median(times)
    nbytes = P * H * W * (4 + 17) + 12 * hits
    gbs = nbytes / (t_min * 1e-3) / 1e9
    M = warp_matrices(proj(H, W), src[:1])
    t0 = time.perf_counter()
    warp_oracle.forward_warp(image, depth, M, occ)
    t_cpu = (time.perf_counter() - t0) * 1e3
    print(f"| {name} | {H} x {W} | {P} | {occ} | {t_min:.3f}, {t_med:.3f} | {t_min / P:.4f} | "
          f"{gbs:.0f} ({gbs * 1e9 / HBM_BYTES_PER_S:.1%}) | {t_cpu:.1f} |")
