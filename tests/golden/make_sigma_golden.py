#!/usr/bin/env python
"""Generate tests/golden/sigma_train.npz by running the REFERENCE's sigma-only passes under autograd.

Run in the build container only (needs /root/reference; the GPU box has none):

    python tests/golden/make_sigma_golden.py

With the reference's trained checkpoint (ckpts/room.ckpt), on CPU/fp32, through the reference's own
``models/rendering.py`` and ``models/nerf.py`` (unmodified, from /root/reference):
  det   render_rays(test_time=True, N_importance=64), perturb = noise_std = 0
  rand  the same with perturb = noise_std = 1 and the four random tensors replayed from a seed
  pts   eval_points(points, models, embeddings) (models/rendering.py:64-123)
Each loss is a fixed seeded linear functional of the outputs; the reference's autograd gradients of every parameter
tensor are stored as a seeded sample of the tensor plus its norm, as in reference_live.npz.  A tensor the pass never
reaches (no .grad in the reference) has no entry.  Nothing here is used at run time by the product;
tests/test_sigma_golden_cpu.py holds the oracle to this file and tests/test_gpu_sigma_train.py the CUDA path.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import Embedding, load_room, np_, replay_rng, room_models  # noqa: E402  (reference modules)
from models.rendering import eval_points, render_rays  # noqa: E402  (reference)

from sinnerf_b200 import synthetic  # noqa: E402

GRAD_SAMPLE = 512
TT_KEYS = ("opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")


def grad_sample_index(numel, k=GRAD_SAMPLE):
    """Fixed, seeded sample of flat indices of a tensor (all of them when it is small)."""
    if numel <= k:
        return torch.arange(numel)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(numel))[:k].sort().values


def store_grads(out, prefix, model):
    for name, prm in model.named_parameters():
        if prm.grad is None:
            continue
        g = prm.grad.detach().flatten()
        idx = grad_sample_index(g.numel())
        out[f"{prefix}_grad_{name}_idx"] = np_(idx).astype(np.int32)
        out[f"{prefix}_grad_{name}_val"] = np_(g[idx])
        out[f"{prefix}_grad_{name}_norm"] = np.array(float(g.double().norm()))


def main():
    torch.set_num_threads(8)
    room = load_room()
    out = {}
    rays = synthetic.random_rays("llff", 48, seed=61)
    emb = [Embedding(3, 10), Embedding(3, 4)]
    for case, (perturb, noise_std, seed) in (("det", (0.0, 0.0, 71)), ("rand", (1.0, 1.0, 72))):
        models = [m.train() for m in room_models(room)]
        torch.manual_seed(seed)
        res = render_rays(models, emb, rays, 64, False, perturb, noise_std, 64, 1024 * 32, False, test_time=True)
        assert set(res) == set(TT_KEYS), sorted(res)
        rng = replay_rng(seed, rays.shape[0], 64, 64, perturb)
        g = torch.Generator().manual_seed(seed + 100)
        proj = {k: torch.randn(res[k].shape, generator=g) for k in TT_KEYS}
        sum((res[k] * proj[k]).sum() for k in TT_KEYS).backward()
        out[f"{case}_rays"] = np_(rays)
        for k, v in rng.items():
            out[f"{case}_rng_{k}"] = np_(v)
        for k in TT_KEYS:
            out[f"{case}_out_{k}"] = np_(res[k])
            out[f"{case}_proj_{k}"] = np_(proj[k])
        store_grads(out, f"{case}_coarse", models[0])
        store_grads(out, f"{case}_fine", models[1])
    models = [m.train() for m in room_models(room)]
    g = torch.Generator().manual_seed(73)
    pts = (torch.rand(1000, 3, generator=g) * 2 - 1) * 1.5
    sigma = eval_points(pts, models, [Embedding(3, 10), Embedding(3, 4)])
    proj = torch.randn(sigma.shape, generator=g)
    (sigma * proj).sum().backward()
    out["pts"], out["pts_sigma"], out["pts_proj"] = np_(pts), np_(sigma), np_(proj)
    store_grads(out, "pts_fine", models[1])
    assert all(p.grad is None for p in models[0].parameters())
    path = os.path.join(HERE, "sigma_train.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
