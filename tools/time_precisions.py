#!/usr/bin/env python
"""Time the tensor-core precision modes against each other in one run, and measure each one's error.

    python tools/time_precisions.py [--modes f16x3,bf16,f16] [--rounds 7] [--json out.json]

Per mode, alternated round by round with CUDA events (median over the rounds):
  * field: the fine-pass field kernel alone, 160 000 rays x 128 samples (seeded default-init weights);
  * patch: BASELINE configs[2]'s render, the 63x84 stride-4 LLFF-shape patch (5 292 rays, 64+64), no grad;
  * train: the configs[4]-shaped training step, render_rays_multi over 4 x 4096 rays (64+64, perturb 1, noise 1, the
    losses evaluated in the compositing kernels), backward and a FusedAdam step with its re-pack.
Error: rel-L2 of each mode's render of the configs[2] patch with the trained room.ckpt weights (tests/golden) against
the fp32 oracle (oracle/render_oracle.py, run on the GPU in fp32).  The card's name and power limit are printed with
the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import render_oracle as orc  # noqa: E402
from sinnerf_b200 import _lib, synthetic  # noqa: E402
from sinnerf_b200.nerf import Embedding, NeRF  # noqa: E402
from sinnerf_b200.optim import FusedAdam  # noqa: E402
from sinnerf_b200.rendering import RayLosses, render_rays, render_rays_multi  # noqa: E402
from sinnerf_b200.synthetic import default_init_params  # noqa: E402
from tests._common import rel_l2, room_params  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--modes", default="f16x3,bf16,f16")
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--json", default="", help="also write the result here")
args = ap.parse_args()
modes = args.modes.split(",")
dev = torch.device("cuda:0")
lib = _lib.load()
emb = [Embedding(3, 10), Embedding(3, 4)]


def card():
    name = torch.cuda.get_device_name(dev)
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return f"{name}, power limit / max SM clock: {q}"


def models_from(params):
    ms = []
    for p in params:
        m = NeRF(use_new_activation=True)
        m.load_state_dict(p)
        ms.append(m.to(dev))
    return ms


# ---------------------------------------------------------------------------------------------------- workloads
def field_workload(mode):
    prec = _lib.precision_id(mode)
    m = models_from([default_init_params(1)])[0]
    img = m.packed_weights(prec)
    rays = synthetic.frame_rays("lego", seed=0)[:160000].to(dev)
    n, S = rays.shape[0], 128
    z = (torch.linspace(2, 6, S, device=dev)[None, :] + torch.rand(n, 1, device=dev) * 0.01).contiguous()
    raw = torch.empty(n, S, 4, device=dev)

    def run():
        _lib.check(lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, 0, _lib.ptr(raw),
                                         _lib.stream_ptr(dev)), "snb_field_forward")
    return run, 1


def patch_workload(mode):
    models = models_from([default_init_params(0), default_init_params(1)])
    rays = synthetic.patch_rays("llff", 63, 84, 4, seed=0).to(dev)

    def run():
        with torch.no_grad():
            render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, False, precision=mode)
    return run, 20


def train_workload(mode):
    models = models_from([default_init_params(0), default_init_params(1)])
    n_rays = 4096
    batches = [synthetic.random_rays("lego", n_rays, seed=100 + i).to(dev) for i in range(4)]
    g = torch.Generator().manual_seed(0)
    trgb = torch.rand(n_rays, 3, generator=g).to(dev)
    tdep = (torch.rand(n_rays, generator=g) * 4 + 2).to(dev)
    ext = [(torch.randn(n_rays, 3, generator=g) / n_rays).to(dev) for _ in range(2)]
    specs = [RayLosses(trgb, tdep), None, None, RayLosses(None, tdep)]
    opt = FusedAdam(models, lr=5e-4, precision=mode)

    def run():
        opt.zero_grad(set_to_none=True)
        res = render_rays_multi(models, emb, batches, 64, False, 1.0, 1.0, 64, 32768, True, precision=mode,
                                batch_losses=specs)
        loss = res[0]["loss_rgb"] + 0.1 * res[0]["loss_depth"]
        for k, w in zip((1, 2), ext):
            loss = loss + (res[k]["rgb_fine"] * w).sum() + (res[k]["rgb_coarse"] * w).sum()
        loss.backward()
        opt.step()
    return run, 3


WORKLOADS = {"field": field_workload, "patch": patch_workload, "train": train_workload}


def time_all():
    runs = {(w, m): make(m) for w, make in WORKLOADS.items() for m in modes}
    for run, reps in runs.values():      # warm-up: module loads, image packs, allocator
        for _ in range(2):
            run()
    torch.cuda.synchronize()
    ts = {key: [] for key in runs}
    for _ in range(args.rounds):
        for key, (run, reps) in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            ts[key].append(e0.elapsed_time(e1) / reps)
    return {w: {m: {"median_ms": statistics.median(ts[(w, m)]), "min_ms": min(ts[(w, m)])} for m in modes}
            for w in WORKLOADS}


# ---------------------------------------------------------------------------------------------------- error
def errors():
    pc, pf = room_params("coarse"), room_params("fine")
    rays = synthetic.patch_rays("llff", 63, 84, 4, seed=0).to(dev)
    with torch.no_grad():
        ref = orc.render_rays({k: v.to(dev) for k, v in pc.items()}, {k: v.to(dev) for k, v in pf.items()}, rays,
                              N_samples=64, N_importance=64, perturb=0, noise_std=0)
        models = models_from([pc, pf])
        out = {}
        for mode in modes:
            got = render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, False, precision=mode)
            out[mode] = {k: rel_l2(got[k].cpu(), ref[k].cpu()) for k in ("rgb_fine", "depth_fine", "opacity_fine")}
    return out


torch.backends.cuda.matmul.allow_tf32 = False     # the fp32 oracle stays fp32 on the GPU
result = {"card": card(), "modes": modes, "rounds": args.rounds, "time": time_all(), "rel_l2_vs_fp32_oracle": errors()}
print(f"card: {result['card']}")
print(f"{'mode':>6} | field 160k x 128 (ms) | patch 5292 rays (ms) | train 4 x 4096 (ms) | rgb_fine | depth_fine | opacity_fine")
for m in modes:
    tm, er = result["time"], result["rel_l2_vs_fp32_oracle"][m]
    print(f"{m:>6} | {tm['field'][m]['median_ms']:21.2f} | {tm['patch'][m]['median_ms']:20.3f} | "
          f"{tm['train'][m]['median_ms']:19.2f} | {er['rgb_fine']:.2e} | {er['depth_fine']:.2e} | {er['opacity_fine']:.2e}")
print(json.dumps(result))
if args.json:
    with open(args.json, "w") as fh:
        json.dump(result, fh, indent=1)
