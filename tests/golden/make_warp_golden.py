#!/usr/bin/env python
"""Generate tests/golden/warp.npz by running the REFERENCE's four forward-warp functions.

Run where a reference checkout is available (the GPU test machines need none):

    python tests/golden/make_warp_golden.py [/path/to/reference]

Calls, unmodified, the datasets' own
    llff_ray_patch_1image_proj.forward_warp     (painter loop, fp32 projection with + 1e-9)
    dtu_proj.warp_img_proj_numpy                (painter loop, fp64 projection through BLAS, no + 1e-9)
    blender_ray_patch_1image_rot3d.forward_warp (numpy scatter, floor, + 1e-9)
    blender_ray_patch_1image_proj.forward_warp  (numpy scatter, no + 1e-9, also returns depth_mask)
on seeded synthetic views -- a tilted plane with a box occluder in front and about 20 % holes (depth 0) -- and
stores, per case, the inputs, the reference's outputs and its per-source coordinates x_src, y_src, depth_src.
LLFF and DTU run at 64x48 (a swapped clamp axis would show); the blender variants at 40x40, since they name the axes
the other way round and only square frames make them agree.  Poses: a small rotation; a large one that puts points
off-frame and behind the camera; for LLFF and rot3d the reference pose itself (the LLFF dataset warps into every pose
of the scene, the reference's included, and rot3d's construction grid contains the zero rotation; the DTU and
blender-proj functions raise there, since their hole pixels divide 0 by Z == 0); and for LLFF a sideways
translation that puts the reference centre, where every hole pixel lands, exactly on the source camera's principal
plane (Z == 0).

For DTU the function returns no coordinates, so they are recomputed here with the same numpy operations in the same
order; the script checks that they reproduce the reference's output through tests/warp_oracle.resolve.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import warp_oracle  # noqa: E402


def reference_datasets(ref):
    """The four dataset modules, loaded as a package of their own (the real datasets/__init__ imports them all)."""
    pkg = types.ModuleType("refdatasets")
    pkg.__path__ = [os.path.join(ref, "datasets")]
    sys.modules["refdatasets"] = pkg
    mods = {}
    for name in ("llff_ray_patch_1image_proj", "dtu_proj", "blender_ray_patch_1image_rot3d",
                 "blender_ray_patch_1image_proj"):
        spec = importlib.util.spec_from_file_location(f"refdatasets.{name}", os.path.join(ref, "datasets", f"{name}.py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    mods["blender_ray_patch_1image_proj"].torch = _TorchWithArrayLikes()
    return mods


class _TorchWithArrayLikes:
    """torch, except that ones_like / zeros_like of a numpy array are numpy arrays.  blender_ray_patch_1image_proj
    .forward_warp calls torch.ones_like on the numpy array np.zeros_like returned, which current torch refuses; with
    this its depth_mask is the numpy scatter of ones, like its rgb and depth."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def ones_like(a, *args, **kw):
        return np.ones_like(a) if isinstance(a, np.ndarray) else torch.ones_like(a, *args, **kw)

    @staticmethod
    def zeros_like(a, *args, **kw):
        return np.zeros_like(a) if isinstance(a, np.ndarray) else torch.zeros_like(a, *args, **kw)


def scene(h, w, seed):
    """Reference view: rgb (h, w, 3) in (0, 1], depth (h, w): plane 2.6-3.4, box at ~1.8, ~20 % holes."""
    g = np.random.default_rng(seed)
    r, c = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    depth = 3.0 + 0.4 * (c / w) - 0.3 * (r / h)
    box = (np.abs(r - h / 2) < h / 5) & (np.abs(c - w / 2) < w / 6)
    depth[box] = 1.8 + 0.05 * (c[box] / w)
    depth[g.random((h, w)) < 0.2] = 0.0
    rgb = g.uniform(0.02, 1.0, (h, w, 3))
    return rgb.astype(np.float32), depth.astype(np.float32)


def intrinsics(h, w):
    return np.array([[1.1 * w, 0, w / 2], [0, 1.1 * w, h / 2], [0, 0, 1]], dtype=np.float32)


def rot(ax, deg):
    t = np.deg2rad(deg)
    c, s = np.cos(t), np.sin(t)
    i, j = [(1, 2), (2, 0), (0, 1)][ax]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def c2w(R, T):
    m = np.eye(4)
    m[:3, :3], m[:3, 3] = R, T
    return m


REF_C2W = c2w(np.eye(3), [0.0, 0.0, 0.0])
POSES = {   # source c2w: camera rotated about its own centre, or moved
    "small": c2w(rot(0, 3.0) @ rot(1, -5.0) @ rot(2, 2.0), [0.05, -0.03, 0.02]),
    "large": c2w(rot(1, 75.0) @ rot(0, 10.0), [0.2, 0.1, -0.3]),
    "sideways": c2w(np.eye(3), [0.5, 0.0, 0.0]),
    "identity": REF_C2W,
}
CASES = [   # variant, occlusion, (h, w), poses
    ("llff", "zbuffer", (48, 64), ("small", "large", "sideways", "identity")),
    ("dtu", "zbuffer", (48, 64), ("small", "large")),
    ("rot3d", "last", (40, 40), ("small", "large", "identity")),
    ("bproj", "last", (40, 40), ("small", "large")),
]


def full_proj(K, E):
    P = np.eye(4)
    P[:3, :3] = K
    return P @ E


def run_torch_variant(mod, rgb, depth, K, E_ref, E_src):
    data = torch.from_numpy(rgb).permute(2, 0, 1)[None]
    d = torch.from_numpy(depth)[None]
    Kt, Er, Es = (torch.from_numpy(x) for x in (K, E_ref, E_src))
    out = mod.forward_warp(data, d, Kt, Er, Kt, Es)
    x, y, z = mod.project_with_depth(d, Kt, Er, Kt, Es)
    extra = {"ref_mask": np.asarray(out[2], dtype=np.float32)} if len(out) == 3 else {}
    return (np.asarray(out[0], np.float32), np.asarray(out[1], np.float32), x.numpy().reshape(-1),
            y.numpy().reshape(-1), z.numpy().reshape(-1), extra)


def dtu_coordinates(depth, ref_proj, src_proj):
    """warp_img_proj_numpy's projection, step for step: homogeneous (c d, r d, d, 1), inv(ref) then src, fp64."""
    h, w = depth.shape
    cc, rr = np.meshgrid(np.arange(w), np.arange(h))
    pts = np.vstack((cc.reshape(-1), rr.reshape(-1), np.ones(h * w, dtype=np.int64)))
    pts = np.vstack((pts * depth.reshape(-1), np.ones(h * w, dtype=np.int64)))
    pts = np.matmul(src_proj, np.matmul(np.linalg.inv(ref_proj), pts))
    z = pts[2].astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        pts /= pts[2]
    return pts[0].astype(np.float32), pts[1].astype(np.float32), z


def reference_targets(x, y, h, w):
    """The integer pixel every reference variant indexes: clip, then truncate (== floor once clipped to >= 0)."""
    ok = ~np.isnan(x) & ~np.isnan(y)
    col = np.clip(np.where(ok, x, 0), 0, w - 1).astype(np.int64)
    row = np.clip(np.where(ok, y, 0), 0, h - 1).astype(np.int64)
    return np.where(ok, row * w + col, -1)


def main(ref):
    mods = reference_datasets(ref)
    convert = mods["llff_ray_patch_1image_proj"].convert
    out = {}
    for ci, (variant, occlusion, (h, w), poses) in enumerate(CASES):
        rgb, depth = scene(h, w, seed=ci)
        K = intrinsics(h, w)
        E_ref = convert(REF_C2W).astype(np.float32)
        out[f"{variant}/image"], out[f"{variant}/depth"] = rgb, depth
        out[f"{variant}/K"], out[f"{variant}/E_ref"] = K, E_ref
        for pose in poses:
            E_src = convert(POSES[pose]).astype(np.float32)
            key = f"{variant}/{pose}"
            extra = {}
            if variant == "dtu":
                ref_proj = full_proj(K, E_ref).astype(np.float32)
                src_proj = full_proj(K, E_src).astype(np.float32)
                new, new_depth = mods["dtu_proj"].warp_img_proj_numpy(rgb, depth, ref_proj, src_proj)
                x, y, z = dtu_coordinates(depth, ref_proj, src_proj)
            else:
                mod = mods["llff_ray_patch_1image_proj" if variant == "llff" else
                           "blender_ray_patch_1image_rot3d" if variant == "rot3d" else "blender_ray_patch_1image_proj"]
                new, new_depth, x, y, z, extra = run_torch_variant(mod, rgb, depth, K, E_ref, E_src)
            out[f"{key}/E_src"] = E_src
            out[f"{key}/ref_rgb"], out[f"{key}/ref_depth"] = np.asarray(new, np.float32), np.asarray(new_depth, np.float32)
            out[f"{key}/x_src"], out[f"{key}/y_src"], out[f"{key}/depth_src"] = x, y, z
            for k, v in extra.items():
                out[f"{key}/{k}"] = v
            # the reference's own targets through the oracle's occlusion rule reproduce its output
            got = warp_oracle.resolve(reference_targets(x, y, h, w), z, rgb, occlusion)
            assert np.array_equal(got[0], out[f"{key}/ref_rgb"]) and np.array_equal(got[1], out[f"{key}/ref_depth"]), key
            assert "ref_mask" not in extra or np.array_equal(got[2], extra["ref_mask"] != 0), key
            holes_z = z.reshape(h, w)[depth == 0]
            print(f"{key}: {h}x{w} {occlusion}, hit {int(got[2].sum())}, Z<0 {int((z < 0).sum())}, "
                  f"hole-group Z {float(holes_z[0]):+g}")
    path = os.path.join(HERE, "warp.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
