"""Seeded synthetic rays of the shapes the reference's datasets emit.

There are no datasets on the build or GPU boxes, so benchmarks and parity tests
use camera-model rays (pixel grid -> pinhole direction -> small random rotation),
not Gaussian noise, so the positional-encoding arguments have realistic size.
Ray rows are ``[ox, oy, oz, dx, dy, dz, near, far]`` and directions are *not*
normalised, as in the reference (datasets/ray_utils.py:73-120).

Shapes (SURVEY.md section 8d):
  lego  400x400, f = 0.5*800/tan(0.5*0.6911)*(400/800), near 2 far 6, white_back
        (datasets/blender_ray_patch_1image_rot3d.py:177,201-211)
  llff  504x378, f = 410, near 1.2, far 7.6, no white_back; patch = 63x84 stride 4
        (datasets/llff_ray_patch_1image_proj.py:351,396-403,625-630)
  dtu   640x512, d = [(i-cx)/fx, (j-cy)/fy, 1], near 2.125 far 4.525, white_back
        (datasets/dtu_proj.py:17-34,290,312,396-398)
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict

import torch


@dataclass(frozen=True)
class FrameShape:
    name: str
    width: int
    height: int
    focal: float
    near: float
    far: float
    white_back: bool
    opencv: bool  # True: +z forward, y down (DTU); False: -z forward, y up (blender/LLFF)


SHAPES = {
    "lego": FrameShape("lego", 400, 400, 0.5 * 800 / math.tan(0.5 * 0.6911) * (400 / 800), 2.0, 6.0, True, False),
    "llff": FrameShape("llff", 504, 378, 410.0, 1.2, 7.6, False, False),
    "dtu": FrameShape("dtu", 640, 512, 2892.33 * (640 / 1600), 2.125, 4.525, True, True),
}


def _small_rotation(gen: torch.Generator) -> torch.Tensor:
    """Rodrigues rotation about a random axis by <= ~11 degrees."""
    axis = torch.randn(3, generator=gen, dtype=torch.float64)
    axis = axis / axis.norm()
    ang = (torch.rand((), generator=gen, dtype=torch.float64) - 0.5) * 0.4
    kx, ky, kz = axis.tolist()
    K = torch.tensor([[0, -kz, ky], [kz, 0, -kx], [-ky, kx, 0]], dtype=torch.float64)
    R = torch.eye(3, dtype=torch.float64) + math.sin(ang) * K + (1 - math.cos(ang)) * (K @ K)
    return R.to(torch.float32)


def frame_rays(shape: str, seed: int = 0, rows=None, cols=None) -> torch.Tensor:
    """(H*W, 8) fp32 rays of a whole frame (or of the given row/col index sets), row-major
    over (row, col) like the reference's flattened (H, W) grids."""
    fs = SHAPES[shape]
    gen = torch.Generator().manual_seed(seed)
    R = _small_rotation(gen)
    origin = torch.tensor([0.0, 0.0, 4.0 if not fs.opencv else -3.3]) + (torch.rand(3, generator=gen) - 0.5) * 0.2
    jj = torch.arange(fs.height, dtype=torch.float32) if rows is None else rows.to(torch.float32)
    ii = torch.arange(fs.width, dtype=torch.float32) if cols is None else cols.to(torch.float32)
    j, i = torch.meshgrid(jj, ii, indexing="ij")
    if fs.opencv:
        d = torch.stack([(i - fs.width / 2) / fs.focal, (j - fs.height / 2) / fs.focal, torch.ones_like(i)], -1)
    else:
        d = torch.stack([(i - fs.width / 2) / fs.focal, -(j - fs.height / 2) / fs.focal, -torch.ones_like(i)], -1)
    d = d.reshape(-1, 3) @ R.t()
    n = d.shape[0]
    rays = torch.empty(n, 8, dtype=torch.float32)
    rays[:, 0:3] = origin + (torch.rand(n, 3, generator=gen) - 0.5) * 0.0  # one camera centre per frame
    rays[:, 3:6] = d
    rays[:, 6] = fs.near
    rays[:, 7] = fs.far
    return rays


def patch_rays(shape: str, patch_h: int, patch_w: int, stride: int, seed: int = 0) -> torch.Tensor:
    """Strided patch of a frame, as the *_ray_patch_* datasets cut it
    (datasets/llff_ray_patch_1image_proj.py:625-646)."""
    fs = SHAPES[shape]
    gen = torch.Generator().manual_seed(seed + 7919)
    span_h, span_w = (patch_h - 1) * stride + 1, (patch_w - 1) * stride + 1
    top = int(torch.randint(0, fs.height - span_h + 1, (1,), generator=gen))
    left = int(torch.randint(0, fs.width - span_w + 1, (1,), generator=gen))
    rows = torch.arange(top, top + span_h, stride)
    cols = torch.arange(left, left + span_w, stride)
    return frame_rays(shape, seed, rows, cols)


def random_rays(shape: str, n: int, seed: int = 0) -> torch.Tensor:
    """n rays at random pixels of a frame (the 4096-ray random sets of a training step)."""
    fs = SHAPES[shape]
    allr = frame_rays(shape, seed)
    gen = torch.Generator().manual_seed(seed + 104729)
    idx = torch.randint(0, fs.width * fs.height, (n,), generator=gen)
    return allr[idx].contiguous()


def default_init_params(seed: int) -> Dict[str, torch.Tensor]:
    """State dict of `torch.manual_seed(seed); NeRF(use_new_activation=True)` -- the seeded default-init weights the bench
    and the measurement tools render with (the modules are created in the reference's order, models/nerf.py:66-103, so
    these are the reference's numbers; tests/test_oracle_golden.py holds them equal to the oracle's own copy).  The global
    RNG state is left untouched."""
    from .nerf import NeRF
    state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    sd = {k: v.detach().clone() for k, v in NeRF(use_new_activation=True).state_dict().items()}
    torch.random.set_rng_state(state)
    return sd


def dino_vits16_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for DINO ViT-S/16's weights (the released file is not in the repository), with the keys and
    shapes of dino_deitsmall16_pretrain.pth.  LayerNorm gains and biases and every Linear bias are non-trivial, and the
    qkv weights (N(0, (1.5/sqrt(384))^2)) give attention logits with a per-layer standard deviation of a few units, so
    softmax is neither uniform nor one-hot.  Much larger qkv weights make the 12-block stack chaotic: rounding the
    operands to bf16 alone then moves the CLS feature by tens of percent.  The global RNG state is untouched."""
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    d, m = 384, 1536
    sd = {"cls_token": n(1, 1, d, std=0.5), "pos_embed": n(1, 197, d, std=0.5),
          "patch_embed.proj.weight": n(d, 3, 16, 16, std=1.0 / math.sqrt(768)), "patch_embed.proj.bias": n(d, std=0.1)}
    for b in range(12):
        p = f"blocks.{b}."
        sd[p + "norm1.weight"] = 1.0 + n(d, std=0.2)
        sd[p + "norm1.bias"] = n(d, std=0.1)
        sd[p + "attn.qkv.weight"] = n(3 * d, d, std=1.5 / math.sqrt(d))
        sd[p + "attn.qkv.bias"] = n(3 * d, std=0.1)
        sd[p + "attn.proj.weight"] = n(d, d, std=0.5 / math.sqrt(d))
        sd[p + "attn.proj.bias"] = n(d, std=0.05)
        sd[p + "norm2.weight"] = 1.0 + n(d, std=0.2)
        sd[p + "norm2.bias"] = n(d, std=0.1)
        sd[p + "mlp.fc1.weight"] = n(m, d, std=1.0 / math.sqrt(d))
        sd[p + "mlp.fc1.bias"] = n(m, std=0.1)
        sd[p + "mlp.fc2.weight"] = n(d, m, std=0.5 / math.sqrt(m))
        sd[p + "mlp.fc2.bias"] = n(d, std=0.05)
    sd["norm.weight"] = 1.0 + n(d, std=0.2)
    sd["norm.bias"] = n(d, std=0.1)
    return sd
