#!/usr/bin/env python
"""CUDA-event times of the semantic loss (sinnerf_b200.vit) against the oracle (tests/vit_oracle.py) run as fp32
PyTorch on the same GPU, with TF32 off and on, on synthetic DINO ViT-S/16 weights:

  1. the ref_ refresh: one forward of a 64x64 patch under no_grad;
  2. semantic_loss(ref, coarse, fine) forward + backward at the recipes' patch shapes, on the '(b p q) c -> b c p q'
     views of ray-major tensors: 64x64 (blender), 63x84 (LLFF), 56x70 (DTU);
  3. the tools/time_train.py training step (4 x 4096 rays, 64 + 64 samples, perturb 1, noise 1, forward + backward)
     whose second ray set is a 64x64 side patch, with and without the semantic term on its coarse and fine rgb.
Implementations alternate within each round; min and median over rounds.  The card's name, power limit and SM clocks
are read in the same run.

    python tools/time_vit.py [--calls 50] [--rounds 7] [--steps 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from sinnerf_b200 import synthetic  # noqa: E402
from sinnerf_b200.nerf import NeRF, Embedding  # noqa: E402
from sinnerf_b200.rendering import render_rays  # noqa: E402
from sinnerf_b200.vit import load_dino_weights  # noqa: E402
from tests import vit_oracle as oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=50, help="calls per timed window (parts 1, 2)")
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=5, help="training steps per timed window (part 3)")
args = ap.parse_args()
dev = torch.device("cuda:0")

sd = synthetic.dino_vits16_state_dict(0)
sd_dev = {k: v.to(dev) for k, v in sd.items()}
ext = load_dino_weights(sd).to(dev)


def tf32(on):
    torch.backends.cuda.matmul.allow_tf32 = on
    torch.backends.cudnn.allow_tf32 = on


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, n):
    """{name: (min, median)} ms per call; each entry is (tf32 flag, fn); implementations alternate within a round"""
    for on, f in fns.values():
        tf32(on)
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, (on, f) in fns.items():
            tf32(on)
            ts[k].append(timed(f, n))
    tf32(False)
    return {k: (min(v), statistics.median(v)) for k, v in ts.items()}


def fmt(r):
    return " | ".join(f"{k} min {v[0]:.3f} med {v[1]:.3f}" for k, v in r.items())


smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                      "-i", "0"], capture_output=True, text=True).stdout.strip()
print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi name, power.limit, clocks.sm, clocks.max.sm: {smi}")

g = torch.Generator().manual_seed(0)
ref = torch.randn(384, generator=g).to(dev)

# ---- 1. ref_ refresh (forward only, no_grad)
real = torch.rand(1, 3, 64, 64, generator=g).to(dev)


def ref_fused():
    with torch.no_grad():
        ext.cls_feature(real)


def ref_oracle():
    with torch.no_grad():
        oracle.cls_feature(sd_dev, real)


r = alternate({"oracle fp32": (False, ref_oracle), "oracle tf32": (True, ref_oracle), "fused": (False, ref_fused)},
              args.calls)
print(f"ref_ forward 64x64, ms/call: {fmt(r)}")

# ---- 2. semantic_loss forward + backward, both patches
for name, (H, W) in (("blender", (64, 64)), ("llff", (63, 84)), ("dtu", (56, 70))):
    rays = [torch.rand(H * W, 3, generator=g).to(dev).requires_grad_(True) for _ in range(2)]
    views = [t.view(1, H, W, 3).permute(0, 3, 1, 2) for t in rays]
    fns = {"oracle fp32": (False, lambda: oracle.semantic_loss(sd_dev, ref, *views).backward()),
           "oracle tf32": (True, lambda: oracle.semantic_loss(sd_dev, ref, *views).backward()),
           "fused": (False, lambda: ext.semantic_loss(ref, *views).backward())}
    r = alternate(fns, args.calls)
    print(f"{name:8s} {H}x{W} semantic_loss fwd+bwd, ms/call: {fmt(r)}")

# ---- 3. training step with and without the semantic term
models = []
for seed in (0, 1):
    m = NeRF(use_new_activation=True)
    m.load_state_dict(synthetic.default_init_params(seed))
    models.append(m.to(dev))
emb = [Embedding(3, 10), Embedding(3, 4)]
batches = [synthetic.random_rays("lego", 4096, seed=0).to(dev), synthetic.patch_rays("lego", 64, 64, 6, seed=1).to(dev)] + \
          [synthetic.random_rays("lego", 4096, seed=i).to(dev) for i in range(2, 4)]
target = torch.rand(4096, 3, device=dev)


def step(impl):
    for m in models:
        m.zero_grad(set_to_none=True)
    loss = 0.0
    outs = [render_rays(models, emb, r, 64, False, 1.0, 1.0, 64, 32768, True) for r in batches]
    for out in outs:
        loss = loss + ((out["rgb_coarse"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean() \
            + 0.1 * out["depth_fine"].mean()
    if impl:
        c, f = (outs[1][k].view(1, 64, 64, 3).permute(0, 3, 1, 2) for k in ("rgb_coarse", "rgb_fine"))
        sem = ext.semantic_loss(ref, c, f) if impl == "fused" else oracle.semantic_loss(sd_dev, ref, c, f)
        loss = loss + 10.0 * sem
    loss.backward()


r = alternate({"none": (False, lambda: step(None)), "oracle fp32": (False, lambda: step("oracle")),
               "oracle tf32": (True, lambda: step("oracle")), "fused": (False, lambda: step("fused"))}, args.steps)
print(f"train step 4 x 4096 rays fwd+bwd, ms/step (none = without the semantic term): {fmt(r)}")
