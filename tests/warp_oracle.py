"""numpy restatement of the forward warp (sinnerf_b200.warp, csrc/warp.cu) on the CPU, the oracle its kernels are
checked against bit for bit.  Two pieces, so each can be pinned separately against the reference datasets:

    project(M, depth)                        -> targets, zf      the contract's fp64 projection
    resolve(targets, zf, image, occlusion)   -> rgb, depth, hit  the occlusion rule

project uses elementwise ufuncs only (numpy never contracts a multiply and an add into an FMA; matmul could block
the sums differently).  resolve is vectorised (a lexsort by target, then key); `painter_loop` / `scatter_loop` are
the reference's sequential loops, kept as the definition resolve is tested against."""
from __future__ import annotations

import numpy as np


def coordinates(M: np.ndarray, depth: np.ndarray):
    """M (3, 4) fp64, depth (H, W) fp32 -> x', y' (H*W,) fp64, zf (H*W,) fp32 = float(Z), and ok (H*W,) bool: false
    for a source the warp skips (non-finite depth or a NaN coordinate)."""
    H, W = depth.shape
    d = depth.astype(np.float64).reshape(-1)
    r, c = np.divmod(np.arange(H * W, dtype=np.int64), W)
    u, v = c.astype(np.float64) * d, r.astype(np.float64) * d
    X, Y, Z = (((M[k, 0] * u + M[k, 1] * v) + M[k, 2] * d) + M[k, 3] for k in range(3))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        zd = np.where(Z != 0, Z, 1e-9)
        x, y = X / zd, Y / zd
        zf = Z.astype(np.float32)
    return x, y, zf, np.isfinite(d) & ~np.isnan(x) & ~np.isnan(y)


def project(M: np.ndarray, depth: np.ndarray):
    """M (3, 4) fp64, depth (H, W) fp32 -> targets (H*W,) int64 flat row*W + col, -1 for a skipped source, and
    zf (H*W,) fp32."""
    H, W = depth.shape
    x, y, zf, ok = coordinates(M, depth)
    col = np.clip(np.floor(np.where(ok, x, 0.0)), 0, W - 1).astype(np.int64)
    row = np.clip(np.floor(np.where(ok, y, 0.0)), 0, H - 1).astype(np.int64)
    return np.where(ok, row * W + col, -1), zf


def resolve(targets: np.ndarray, zf: np.ndarray, image: np.ndarray, occlusion: str):
    """targets (N,) int64 into image's H*W pixels (-1 = skipped), zf (N,) fp32, image (H, W, 3): source i is pixel i of
    the image.  -> rgb (H, W, 3), depth (H, W) fp32, hit (H, W) bool.

    "zbuffer": with L the last source index with zf == 0 on a target (-1 if none), the winner is the argmin of zf over
    the sources with index > L or zf < 0, ties to the lowest index; if that set is empty, the winner is L.  This is
    what the painter loop (`painter_loop`) keeps: its `s == 0` test accepts whatever follows a stored zero.
    "last": the winner is the largest index."""
    H, W = image.shape[:2]
    n = H * W
    src = image.reshape(-1, 3)
    idx = np.arange(len(targets), dtype=np.int64)
    valid = targets >= 0
    win = np.full(n, -1, dtype=np.int64)
    if occlusion == "last":
        np.maximum.at(win, targets[valid], idx[valid])
    elif occlusion == "zbuffer":
        last_zero = np.full(n, -1, dtype=np.int64)
        z0 = valid & (zf == 0)
        np.maximum.at(last_zero, targets[z0], idx[z0])
        cand = valid.copy()
        cand[valid] = (idx[valid] > last_zero[targets[valid]]) | (zf[valid] < 0)
        ci, ct, cz = idx[cand], targets[cand], zf[cand]
        order = np.lexsort((ci, cz, ct))           # by target, then zf, then index
        ct, ci = ct[order], ci[order]
        first = np.ones(len(ct), dtype=bool)
        first[1:] = ct[1:] != ct[:-1]
        win = last_zero.copy()
        win[ct[first]] = ci[first]
    else:
        raise ValueError(occlusion)
    hit = win >= 0
    rgb = np.zeros((n, 3), dtype=np.float32)
    depth = np.zeros(n, dtype=np.float32)
    rgb[hit] = src[win[hit]]
    depth[hit] = zf[win[hit]]
    return rgb.reshape(H, W, 3), depth.reshape(H, W), hit.reshape(H, W)


def forward_warp(image: np.ndarray, depth: np.ndarray, mats: np.ndarray, occlusion: str):
    """image (H, W, 3), depth (H, W) fp32, mats (P, 3, 4) fp64 (sinnerf_b200.warp.warp_matrices) -> the stacked
    (P, H, W, 3) rgb, (P, H, W) depth and (P, H, W) hit of resolve(project(M, depth)) per pose."""
    outs = [resolve(*project(M, depth), image, occlusion) for M in mats]
    return tuple(np.stack(o) for o in zip(*outs))


def painter_loop(targets, zf, image):
    """The LLFF / DTU datasets' painter loop, literally: keep source i when the stored depth is 0 or greater than its."""
    H, W = image.shape[:2]
    src = image.reshape(-1, 3)
    rgb, depth, hit = np.zeros((H * W, 3), np.float32), np.zeros(H * W, np.float32), np.zeros(H * W, bool)
    for i, t in enumerate(targets):
        if t >= 0 and (depth[t] == 0 or depth[t] > zf[i]):
            depth[t], rgb[t], hit[t] = zf[i], src[i], True
    return rgb.reshape(H, W, 3), depth.reshape(H, W), hit.reshape(H, W)


def scatter_loop(targets, zf, image):
    """The blender datasets' scatter, one source at a time in raster order: the last writer stays."""
    H, W = image.shape[:2]
    src = image.reshape(-1, 3)
    rgb, depth, hit = np.zeros((H * W, 3), np.float32), np.zeros(H * W, np.float32), np.zeros(H * W, bool)
    for i, t in enumerate(targets):
        if t >= 0:
            depth[t], rgb[t], hit[t] = zf[i], src[i], True
    return rgb.reshape(H, W, 3), depth.reshape(H, W), hit.reshape(H, W)
