#!/usr/bin/env python
"""CUDA-event times of the adversarial-loss discriminator (sinnerf_b200.discriminator) against the oracle
(tests/disc_oracle.py) run as fp32 PyTorch on the same GPU, with cuDNN and TF32 off, then on:

  1. a generator-step call: D(fake) forward + the input gradient of -mean;
  2. a discriminator-step pair: D(real), D(fake.detach()), the hinge loss and the weight gradients;
     both at the recipes' patch shapes with B = 1: 64x64 (blender, imsize 64), 63x84 (LLFF) and 56x70 (DTU)
     (imsize -1);
  3. the tools/time_train.py training step (4 x 4096 rays, 64 + 64 samples, perturb 1, noise 1, forward + backward)
     whose second ray set is a 64x64 side patch, with and without 0.01 x the hinge generator loss on its fine rgb.
Every call makes its own DiffAugment draws from the global generators, as in training (about one call in four
augments).
Implementations alternate within each round; min and median over rounds.  The card's name, power limit and SM clocks
are read in the same run.

    python tools/time_discriminator.py [--calls 50] [--rounds 7] [--steps 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from sinnerf_b200 import synthetic  # noqa: E402
from sinnerf_b200.discriminator import Discriminator, draw_augment  # noqa: E402
from sinnerf_b200.nerf import NeRF, Embedding  # noqa: E402
from sinnerf_b200.rendering import render_rays  # noqa: E402
from tests import disc_oracle as oracle  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=50, help="calls per timed window (parts 1, 2)")
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=5, help="training steps per timed window (part 3)")
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
    """{name: (min, median)} ms per call; each entry is (cudnn + tf32 flag, fn); implementations alternate in a round"""
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


def fmt(r):
    return " | ".join(f"{k} min {v[0]:.3f} med {v[1]:.3f}" for k, v in r.items())


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


for name, imsize, (H, W) in (("blender", 64, (64, 64)), ("llff", -1, (63, 84)), ("dtu", -1, (56, 70))):
    D = Discriminator(False, "color,cutout", imsize=imsize).to(dev)
    O = OracleD(D)
    rays = torch.rand(H * W, 3, generator=g).to(dev).requires_grad_(True)
    fake = rays.view(1, H, W, 3).permute(0, 3, 1, 2)
    real = torch.rand(1, 3, H, W, generator=g).to(dev)

    def gs(m):
        return lambda: (-m(fake).mean()).backward()

    def ds(m):
        def f():
            pr, pf = m(real), m(fake.detach())
            ((F.relu(1 - pr).mean() + F.relu(1 + pf).mean()) / 2).backward()
        return f
    r = alternate({"oracle fp32": (False, gs(O)), "oracle cudnn+tf32": (True, gs(O)), "fused": (False, gs(D))},
                  args.calls)
    print(f"{name:8s} {H}x{W} G-step call fwd + input grad, ms/call: {fmt(r)}")
    r = alternate({"oracle fp32": (False, ds(O)), "oracle cudnn+tf32": (True, ds(O)), "fused": (False, ds(D))},
                  args.calls)
    print(f"{name:8s} {H}x{W} D-step pair fwd x2 + weight grads, ms/pair: {fmt(r)}")

# ---- 3. training step with and without the adversarial generator term
models = []
for seed in (0, 1):
    m = NeRF(use_new_activation=True)
    m.load_state_dict(synthetic.default_init_params(seed))
    models.append(m.to(dev))
emb = [Embedding(3, 10), Embedding(3, 4)]
batches = [synthetic.random_rays("lego", 4096, seed=0).to(dev), synthetic.patch_rays("lego", 64, 64, 6, seed=1).to(dev)] + \
          [synthetic.random_rays("lego", 4096, seed=i).to(dev) for i in range(2, 4)]
target = torch.rand(4096, 3, device=dev)
D = Discriminator(False, "color,cutout", imsize=64).to(dev)
O = OracleD(D)


def step(impl):
    for m in models:
        m.zero_grad(set_to_none=True)
    loss = 0.0
    outs = [render_rays(models, emb, r, 64, False, 1.0, 1.0, 64, 32768, True) for r in batches]
    for out in outs:
        loss = loss + ((out["rgb_coarse"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean() \
            + 0.1 * out["depth_fine"].mean()
    if impl:
        f = outs[1]["rgb_fine"].view(1, 64, 64, 3).permute(0, 3, 1, 2)
        loss = loss + 0.01 * -(D(f) if impl == "fused" else O(f)).mean()
    loss.backward()


r = alternate({"none": (False, lambda: step(None)), "oracle fp32": (False, lambda: step("oracle")),
               "oracle cudnn+tf32": (True, lambda: step("oracle")), "fused": (False, lambda: step("fused"))},
              args.steps)
print(f"train step 4 x 4096 rays fwd+bwd, ms/step (none = without the adversarial term): {fmt(r)}")
