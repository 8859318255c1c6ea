"""Forward warp of the reference view into unseen views through its depth: the geometry pseudo-labels SinNeRF's
datasets build, executed by libsinnerf_b200's sm_90a kernels (csrc/warp.cu) with every pose of a batch in one launch.

    from sinnerf_b200.warp import forward_warp
    rgb, depth, hit = forward_warp(image, depth_ref, ref_proj, src_proj, occlusion="zbuffer")

One function serves the reference's four variants:
    occlusion="zbuffer"  nearest depth wins (the painter loops of datasets/llff_ray_patch_1image_proj.py:144-166 and
                         datasets/dtu_proj.py:236-273)
    occlusion="last"     the last source in raster order wins (the numpy scatters of the two blender datasets;
                         `hit` is blender_ray_patch_1image_proj's depth_mask)

The projection is fp64 with every product and sum rounded on its own, so the result is defined to the bit
(DESIGN.md section 4.4): x' = X / Z, with 1e-9 in place of Z where Z == 0.  Two documented differences from the
reference: it projects in fp32 (LLFF, blender) or through BLAS in fp64 (DTU), so a source within its rounding of a
pixel boundary can land one pixel away.  That includes the pixels of poses that keep integer coordinates, such as the
reference pose itself: this warp lands them exactly on their own pixel, the reference shifts about half of them by
one.  And the blender-proj and DTU variants divide without the `+ 1e-9`, which matters only at Z == 0, where they
index with NaN.
Sources with a non-finite depth or a NaN coordinate are skipped.  The labels are data: there is no autograd.
fp32 CUDA tensors only: there is no CPU path.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

__all__ = ["forward_warp", "warp_matrices"]

# device workspace per launch (keys and slots, 12 B per target pixel per pose in "zbuffer" mode); larger batches are
# warped in chunks of poses
WORKSPACE_BUDGET = 256 << 20


def _as_f64(m) -> np.ndarray:
    if isinstance(m, torch.Tensor):
        m = m.detach().cpu().double().numpy()
    return np.asarray(m, dtype=np.float64)


def warp_matrices(ref_proj, src_proj) -> np.ndarray:
    """(P, 3, 4) fp64: the top three rows of src_proj @ inv(ref_proj), composed on the host in fp64 as
    I + (src_proj - ref_proj) @ inv(ref_proj), so the reference camera itself gives exactly the identity.
    ref_proj (4, 4); src_proj (4, 4) or (P, 4, 4); tensors or arrays.  A singular ref_proj is ValueError."""
    ref = _as_f64(ref_proj)
    src = _as_f64(src_proj)
    if ref.shape != (4, 4):
        raise ValueError(f"forward_warp: ref_proj must be (4, 4) (got {ref.shape})")
    if src.ndim == 2:
        src = src[None]
    if src.ndim != 3 or src.shape[1:] != (4, 4) or src.shape[0] < 1:
        raise ValueError(f"forward_warp: src_proj must be (4, 4) or (P, 4, 4) with P >= 1 (got {tuple(src.shape)})")
    try:
        inv = np.linalg.inv(ref)
    except np.linalg.LinAlgError as e:
        raise ValueError(f"forward_warp: ref_proj is singular ({e})") from None
    if not np.all(np.isfinite(inv)):
        raise ValueError("forward_warp: ref_proj is singular (its inverse is not finite)")
    # I + (src - ref) inv(ref), not src inv(ref): the same matrix, but a source camera equal to the reference gives
    # exactly the identity (and a pure move exactly I plus a translation column), so its pixels keep their exact
    # integer coordinates instead of landing a rounding error below them
    return np.ascontiguousarray((np.eye(4) + np.matmul(src - ref, inv))[:, :3, :])


def forward_warp(image: torch.Tensor, depth_ref: torch.Tensor, ref_proj, src_proj, *, occlusion: str = "zbuffer"):
    """Warp `image` (H, W, 3) with depth `depth_ref` (H, W), both fp32 CUDA, from the camera with full projection
    `ref_proj` (4, 4) into the cameras `src_proj` ((4, 4) or (P, 4, 4)); a full projection is [[K, 0], [0, 1]] @ E with
    E the 4x4 world-to-camera matrix.  Returns (rgb, depth, hit): rgb (P, H, W, 3) -- (H, W, 3) when src_proj is a
    single 4x4 --, depth (P, H, W) fp32 and hit (P, H, W) bool, on the image's device; pixels nothing landed on are 0.
    Errors: a CPU tensor is RuntimeError, a dtype other than fp32 TypeError, shapes / occlusion / a singular ref_proj
    ValueError."""
    what = "forward_warp"
    if occlusion not in _lib.WARP_OCCLUSION:
        raise ValueError(f"{what}: occlusion must be one of {sorted(_lib.WARP_OCCLUSION)} (got {occlusion!r})")
    for t, name in ((image, "image"), (depth_ref, "depth_ref")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{what}: {name} is not a torch.Tensor (got {type(t)})")
    if image.dim() != 3 or image.shape[2] != 3:
        raise ValueError(f"{what}: image must be (H, W, 3) (got {tuple(image.shape)})")
    H, W = image.shape[:2]
    if tuple(depth_ref.shape) != (H, W):
        raise ValueError(f"{what}: depth_ref must be (H, W) = {(H, W)} (got {tuple(depth_ref.shape)})")
    if H < 1 or W < 1 or H * W >= 1 << 31:
        raise ValueError(f"{what}: needs H, W >= 1 and H*W < 2^31 (got {H} x {W})")
    single = (src_proj.dim() if isinstance(src_proj, torch.Tensor) else np.ndim(src_proj)) == 2
    mats = warp_matrices(ref_proj, src_proj)
    for t, name in ((image, "image"), (depth_ref, "depth_ref")):
        if t.dtype != torch.float32:
            raise TypeError(f"{what}: {name} must be float32 (got {t.dtype})")
    _lib.require_device(image, what)
    if depth_ref.device != image.device:
        raise RuntimeError(f"{what}: image and depth_ref must be on the same device (got {image.device} and "
                           f"{depth_ref.device})")

    lib = _lib.load()
    dev = image.device
    occ = _lib.WARP_OCCLUSION[occlusion]
    P = mats.shape[0]
    image, depth_ref = image.contiguous(), depth_ref.contiguous()
    rgb = torch.empty((P, H, W, 3), device=dev, dtype=torch.float32)
    depth = torch.empty((P, H, W), device=dev, dtype=torch.float32)
    hit = torch.empty((P, H, W), device=dev, dtype=torch.bool)
    with torch.cuda.device(dev):
        stream = _lib.stream_ptr(dev)
        mats_d = torch.from_numpy(mats).to(dev)
        chunk = max(1, WORKSPACE_BUDGET // lib.snb_forward_warp_workspace_bytes(1, H, W, occ))
        ws = torch.empty(lib.snb_forward_warp_workspace_bytes(min(chunk, P), H, W, occ), device=dev, dtype=torch.uint8)
        for p0 in range(0, P, chunk):
            n = min(chunk, P - p0)
            _lib.check(lib.snb_forward_warp(_lib.ptr(image), _lib.ptr(depth_ref), H, W, _lib.ptr(mats_d[p0]), n, occ,
                                            _lib.ptr(rgb[p0]), _lib.ptr(depth[p0]), _lib.ptr(hit[p0]), _lib.ptr(ws),
                                            stream), "snb_forward_warp")
    if single:
        return rgb[0], depth[0], hit[0]
    return rgb, depth, hit
