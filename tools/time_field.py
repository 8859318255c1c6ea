#!/usr/bin/env python
"""Time the field kernel alone (fine-pass shape) for one precision; used for profiling runs.

    python tools/time_field.py [--precision f16x3] [--rays 160000] [--samples 128] [--iters 5] [--sigma-only]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sinnerf_b200.synthetic import default_init_params  # noqa: E402  (seeded default-init weights)
from sinnerf_b200 import _lib, synthetic  # noqa: E402
from sinnerf_b200.nerf import NeRF  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--precision", default="f16x3")
ap.add_argument("--rays", type=int, default=160000)
ap.add_argument("--samples", type=int, default=128)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--sigma-only", action="store_true")
ap.add_argument("--dump", default="", help="save the output tensor here (A/B comparison of builds)")
args = ap.parse_args()

dev = torch.device("cuda:0")
torch.manual_seed(0)
lib = _lib.load()
prec = _lib.precision_id(args.precision)
m = NeRF(use_new_activation=True)
m.load_state_dict(default_init_params(1))
m = m.to(dev)
img = m.packed_weights(prec)
rays = synthetic.frame_rays("lego", seed=0)[:args.rays].to(dev)
n, S = rays.shape[0], args.samples
z = (torch.linspace(2, 6, S, device=dev)[None, :] + torch.rand(n, 1, device=dev) * 0.01).contiguous()
raw = torch.empty(n, S, 1 if args.sigma_only else 4, device=dev)


def run():
    _lib.check(lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, int(args.sigma_only),
                                     _lib.ptr(raw), _lib.stream_ptr(dev)), "snb_field_forward")


for _ in range(2):
    run()
torch.cuda.synchronize()
ts = []
for _ in range(args.iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ms = min(ts)
flops = 2 * (982528 // 2 if args.sigma_only else 593408) * n * S
sms = torch.cuda.get_device_properties(0).multi_processor_count
print(f"precision={args.precision} rays={n} S={S} "
      f"ms={ms:.3f} (median {sorted(ts)[len(ts) // 2]:.3f})  {flops / ms / 1e9:.1f} TFLOP/s algorithmic  "
      f"{n * S / 128 / sms :.0f} tiles/SM  {ms * 1e3 / (n * S / 128 / sms):.2f} us/tile")
if args.dump:
    torch.save(raw.cpu(), args.dump)
