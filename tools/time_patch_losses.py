#!/usr/bin/env python
"""CUDA-event times of the patch losses (sinnerf_b200.losses) against the fp32 restatement of kornia 0.6.3
(tests/patch_loss_oracle.py, the same ATen ops kornia dispatches, run on the GPU in fp32 with TF32 off):

  1. one call, forward + backward, of inverse_depth_smoothness_loss(depth, rgb) and of ssim_loss(rgb, target, 11) and
     ssim_loss(depth, depth_gt, 11) at the recipes' patch shapes, on the '(b p q) c -> b c p q' views of ray-major
     tensors: 64x64 (blender), 63x84 (LLFF), 56x70 (DTU);
  2. the tools/time_train.py training step (4 x 4096 rays, 64 + 64 samples, perturb 1, noise 1, forward + backward)
     whose first two ray sets are 64x64 patches, plus the reference step's patch terms on them: the four smoothness
     calls (models/sinnerf.py:370-373, 395-398) and l2_ssim's ssim_loss on the rgb and the depth patch.
     Oracle and fused losses alternate; min and median over rounds.

    python tools/time_patch_losses.py [--calls 200] [--rounds 7] [--steps 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sinnerf_b200 import losses as fused  # noqa: E402
from sinnerf_b200 import synthetic  # noqa: E402
from sinnerf_b200.nerf import NeRF, Embedding  # noqa: E402
from sinnerf_b200.rendering import render_rays  # noqa: E402
from tests import patch_loss_oracle as oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=200, help="calls per timed window (part 1)")
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=5, help="training steps per timed window (part 2)")
args = ap.parse_args()
dev = torch.device("cuda:0")
torch.backends.cudnn.allow_tf32 = False
IMPLS = {"oracle": (oracle.inverse_depth_smoothness_loss, oracle.ssim_loss),
         "fused": (fused.inverse_depth_smoothness_loss, fused.ssim_loss)}


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, n):
    """{name: (min, median)} ms per call over args.rounds rounds, the implementations alternating within each round."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, f in fns.items():
            ts[k].append(timed(f, n))
    return {k: (min(v), statistics.median(v)) for k, v in ts.items()}


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi: {gpu}")

# ---- 1. one call, forward + backward
g = torch.Generator().manual_seed(0)
for name, (H, W) in (("blender", (64, 64)), ("llff", (63, 84)), ("dtu", (56, 70))):
    n = H * W
    rgb = torch.rand(n, 3, generator=g).to(dev).requires_grad_(True)
    dep = (torch.rand(n, generator=g) * 4 + 2).to(dev).requires_grad_(True)
    tgt = torch.rand(1, 3, H, W, generator=g).to(dev)
    dgt = (torch.rand(1, 1, H, W, generator=g) * 4 + 2).to(dev)
    img, idep = rgb.view(1, H, W, 3).permute(0, 3, 1, 2), dep.view(1, H, W, 1).permute(0, 3, 1, 2)
    for loss_name, make in (("smoothness", lambda s, q: s(idep, img)), ("ssim rgb", lambda s, q: q(img, tgt, 11)),
                            ("ssim depth", lambda s, q: q(idep, dgt, 11))):
        fns = {k: (lambda s=s, q=q: make(s, q).backward()) for k, (s, q) in IMPLS.items()}
        r = alternate(fns, args.calls)
        print(f"{name:8s} {H}x{W} {loss_name:11s} fwd+bwd ms/call  oracle min {r['oracle'][0]:.4f} med {r['oracle'][1]:.4f}"
              f" | fused min {r['fused'][0]:.4f} med {r['fused'][1]:.4f}")

# ---- 2. training step + patch terms
models = []
for seed in (0, 1):
    m = NeRF(use_new_activation=True)
    m.load_state_dict(synthetic.default_init_params(seed))
    models.append(m.to(dev))
emb = [Embedding(3, 10), Embedding(3, 4)]
batches = [synthetic.patch_rays("lego", 64, 64, 6, seed=i).to(dev) for i in range(2)] + \
          [synthetic.random_rays("lego", 4096, seed=i).to(dev) for i in range(2, 4)]
target = torch.rand(4096, 3, device=dev)
tgt_patch, dgt_patch = target.view(1, 64, 64, 3).permute(0, 3, 1, 2), torch.rand(1, 1, 64, 64, device=dev) * 4 + 2


def step(impl):
    smooth, ssim = IMPLS[impl] if impl else (None, None)
    for m in models:
        m.zero_grad(set_to_none=True)
    loss = 0.0
    outs = [render_rays(models, emb, r, 64, False, 1.0, 1.0, 64, 32768, True) for r in batches]
    for out in outs:
        loss = loss + ((out["rgb_coarse"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean() \
            + 0.1 * out["depth_fine"].mean()
    if impl:
        rgb = [o["rgb_fine"].view(1, 64, 64, 3).permute(0, 3, 1, 2) for o in outs[:2]]
        df = [o["depth_fine"].view(1, 64, 64, 1).permute(0, 3, 1, 2) for o in outs[:2]]
        dc = [o["depth_coarse"].view(1, 64, 64, 1).permute(0, 3, 1, 2) for o in outs[:2]]
        loss = loss + smooth(df[0], rgb[0]) + smooth(dc[0], rgb[0]) + smooth(dc[1], rgb[1]) + smooth(df[1], rgb[1]) \
            + ssim(rgb[0], tgt_patch, 11) + ssim(df[0], dgt_patch, 11)
    loss.backward()


r = alternate({"none": lambda: step(None), "oracle": lambda: step("oracle"), "fused": lambda: step("fused")}, args.steps)
print(f"train step 4 x 4096 rays fwd+bwd, ms/step: without patch terms min {r['none'][0]:.2f} med {r['none'][1]:.2f} | "
      f"oracle patch terms min {r['oracle'][0]:.2f} med {r['oracle'][1]:.2f} | "
      f"fused patch terms min {r['fused'][0]:.2f} med {r['fused'][1]:.2f}")
