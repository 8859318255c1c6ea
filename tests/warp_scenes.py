"""Seeded synthetic views and cameras for the forward-warp tests and tools/time_warp.py: a tilted plane with a box
occluder in front and a fraction of holes (depth 0), seen by pinhole cameras in the datasets' convention."""
import numpy as np


def rot(ax, deg):
    t = np.deg2rad(deg)
    c, s = np.cos(t), np.sin(t)
    i, j = [(1, 2), (2, 0), (0, 1)][ax]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def proj(H, W, R=np.eye(3), T=(0.0, 0.0, 0.0)):
    """[[K, 0], [0, 1]] @ E for a camera with rotation R and centre T, E = the datasets' convert(c2w)."""
    K = np.eye(4)
    K[0, 0] = K[1, 1] = 1.1 * max(H, W)
    K[0, 2], K[1, 2] = W / 2, H / 2
    flip = np.diag([1.0, -1.0, -1.0])
    E = np.eye(4)
    E[:3, :3] = flip @ R.T
    E[:3, 3] = -flip @ R.T @ np.asarray(T)
    return K @ E


def random_poses(H, W, n, seed, max_deg=20.0):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        a = g.uniform(-max_deg, max_deg, 3)
        out.append(proj(H, W, rot(0, a[0]) @ rot(1, a[1]) @ rot(2, a[2]), g.uniform(-0.3, 0.3, 3)))
    return np.stack(out)


def scene(H, W, seed, holes=0.2):
    g = np.random.default_rng(seed)
    r, c = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    depth = 3.0 + 0.4 * c / max(W, 1) - 0.3 * r / max(H, 1) + 0.01 * g.standard_normal((H, W))
    box = (np.abs(r - H / 2) < H / 5) & (np.abs(c - W / 2) < W / 6)
    depth[box] = 1.8 + 0.1 * g.random(box.sum())
    depth[g.random((H, W)) < holes] = 0.0
    return g.random((H, W, 3)).astype(np.float32), depth.astype(np.float32)
