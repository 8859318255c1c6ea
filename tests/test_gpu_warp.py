"""sinnerf_b200.warp.forward_warp on the H100 against the numpy oracle (tests/warp_oracle.py), bit for bit: rgb,
depth (including the sign of a zero) and hit, in both occlusion modes."""
import os

import numpy as np
import pytest
import torch

from sinnerf_b200 import warp
from sinnerf_b200.warp import forward_warp, warp_matrices
from tests import warp_oracle as wo
from tests.warp_scenes import proj, random_poses, rot, scene

pytestmark = pytest.mark.gpu
MODES = ("zbuffer", "last")


def check(image, depth, ref_proj, src_proj, occlusion, **kw):
    """forward_warp on the GPU == the oracle, bit for bit; returns the GPU result."""
    dev = torch.device("cuda")
    got = forward_warp(torch.from_numpy(image).to(dev), torch.from_numpy(depth).to(dev), ref_proj, src_proj,
                       occlusion=occlusion, **kw)
    torch.cuda.synchronize()
    want = wo.forward_warp(image, depth, warp_matrices(ref_proj, src_proj), occlusion)
    single = np.ndim(src_proj) == 2
    for g, w, name in zip(got, want, ("rgb", "depth", "hit")):
        assert g.device.type == "cuda"
        g = g.cpu().numpy()
        w = w[0] if single else w
        assert g.shape == w.shape and g.dtype == w.dtype, name
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), \
            f"{name}: {int((g != w).reshape(g.shape[0], -1).any(-1).sum()) if g.ndim > 2 else -1} poses differ"
    return got


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "warp.npz")))


@pytest.mark.parametrize("variant,pose,occlusion", [
    ("llff", "small", "zbuffer"), ("llff", "large", "zbuffer"), ("llff", "sideways", "zbuffer"),
    ("llff", "identity", "zbuffer"), ("dtu", "small", "zbuffer"), ("dtu", "large", "zbuffer"), ("rot3d", "small", "last"),
    ("rot3d", "large", "last"), ("rot3d", "identity", "last"), ("bproj", "small", "last"), ("bproj", "large", "last")])
def test_golden_inputs(golden, variant, pose, occlusion):
    K, E_ref, E_src = golden[f"{variant}/K"], golden[f"{variant}/E_ref"], golden[f"{variant}/{pose}/E_src"]
    full = lambda E: np.block([[K.astype(np.float64), np.zeros((3, 1))], [np.zeros((1, 3)), np.ones((1, 1))]]) @ E
    for occ in (occlusion,) + tuple(m for m in MODES if m != occlusion):   # the other rule on the same geometry too
        check(golden[f"{variant}/image"], golden[f"{variant}/depth"], full(E_ref), full(E_src), occ)


@pytest.mark.parametrize("H,W", [(400, 400), (378, 504)])
@pytest.mark.parametrize("occlusion", MODES)
def test_random_geometry(H, W, occlusion):
    image, depth = scene(H, W, seed=H)
    check(image, depth, proj(H, W), random_poses(H, W, 4, seed=W), occlusion)


@pytest.mark.parametrize("occlusion", MODES)
def test_full_poses_800(occlusion):
    image, depth = scene(800, 800, seed=8, holes=0.4)
    check(image, depth, proj(800, 800), random_poses(800, 800, 5, seed=9), occlusion)


@pytest.mark.parametrize("H,W", [(37, 53), (1, 1), (1, 61), (29, 1)])
@pytest.mark.parametrize("occlusion", MODES)
def test_odd_sizes(H, W, occlusion):
    image, depth = scene(H, W, seed=H * 100 + W)
    check(image, depth, proj(H, W), random_poses(H, W, 3, seed=W), occlusion)
    rgb, dep, hit = check(image, depth, proj(H, W), random_poses(H, W, 1, seed=1)[0], occlusion)
    assert rgb.shape == (H, W, 3) and dep.shape == (H, W) and hit.shape == (H, W)


@pytest.mark.parametrize("occlusion", MODES)
def test_all_holes(occlusion):
    """Every source lands on one pixel (the reference centre): the most contended target possible."""
    image, _ = scene(256, 320, seed=3)
    depth = np.zeros((256, 320), np.float32)
    rgb, dep, hit = check(image, depth, proj(256, 320), random_poses(256, 320, 3, seed=4), occlusion)
    assert int(hit.sum()) == 3
    want = 0 if occlusion == "zbuffer" else 256 * 320 - 1          # lowest index wins a tie; the scatter keeps the last
    assert torch.equal(rgb[hit].cpu(), torch.from_numpy(image.reshape(-1, 3)[[want] * 3]))


@pytest.mark.parametrize("occlusion", MODES)
def test_negative_z(occlusion):
    """A camera turned 75 degrees: part of the scene is behind it (zf < 0 competes in zbuffer mode)."""
    H, W = 120, 160
    image, depth = scene(H, W, seed=5)
    src = np.stack([proj(H, W, rot(1, a) @ rot(0, 10.0), (0.2, 0.1, -0.3)) for a in (75.0, -80.0, 100.0)])
    _, dep, hit = check(image, depth, proj(H, W), src, occlusion)
    assert bool((dep[hit] < 0).any())


@pytest.mark.parametrize("occlusion", MODES)
def test_z_zero_class(occlusion):
    """A pure sideways move: the hole group lands at Z == 0 exactly and resets the painter loop."""
    H, W = 96, 128
    image, depth = scene(H, W, seed=6, holes=0.3)
    src = np.stack([proj(H, W, np.eye(3), (t, 0.0, 0.0)) for t in (0.5, -0.25, 1.0)])
    assert np.all(warp_matrices(proj(H, W), src)[:, 2, 3] == 0)
    check(image, depth, proj(H, W), src, occlusion)


@pytest.mark.parametrize("H,W", [(400, 400), (378, 504)])
@pytest.mark.parametrize("occlusion", MODES)
def test_identity_pose_returns_the_image(H, W, occlusion):
    """The reference camera itself (in the LLFF pose list and the rot3d grid): every pixel with depth lands on itself,
    exactly, so the warp gives the image back (pixel (0, 0), where the hole group lands, aside)."""
    image, depth = scene(H, W, seed=19)
    rgb, dep, hit = check(image, depth, proj(H, W), proj(H, W), occlusion)
    keep = depth != 0
    keep[0, 0] = False
    keep_d = torch.from_numpy(keep).cuda()
    assert torch.equal(rgb[keep_d].cpu(), torch.from_numpy(image[keep]))
    assert torch.equal(dep[keep_d].cpu(), torch.from_numpy(depth[keep])) and bool(hit[keep_d].all())


@pytest.mark.parametrize("occlusion", MODES)
def test_non_finite_depths_are_skipped(occlusion):
    H, W = 64, 80
    image, depth = scene(H, W, seed=7)
    g = np.random.default_rng(7)
    for bad in (np.nan, np.inf, -np.inf):
        depth[g.random((H, W)) < 0.05] = bad
    check(image, depth, proj(H, W), random_poses(H, W, 3, seed=7), occlusion)


def test_batch_equals_single_calls():
    H, W = 40, 40
    image, depth = scene(H, W, seed=11, holes=0.4)
    src = random_poses(H, W, 125, seed=12)
    dev = torch.device("cuda")
    im, d = torch.from_numpy(image).to(dev), torch.from_numpy(depth).to(dev)
    for occ in MODES:
        batch = forward_warp(im, d, proj(H, W), src, occlusion=occ)
        for p in range(len(src)):
            single = forward_warp(im, d, proj(H, W), src[p], occlusion=occ)
            for b, s in zip(batch, single):
                assert torch.equal(b[p], s)


def test_chunked_batch_equals_single_calls(monkeypatch):
    """A budget of 3.5 poses' workspace: 10 poses go in four launches."""
    H, W = 64, 48
    image, depth = scene(H, W, seed=13, holes=0.4)
    src = random_poses(H, W, 10, seed=14)
    dev = torch.device("cuda")
    im, d = torch.from_numpy(image).to(dev), torch.from_numpy(depth).to(dev)
    singles = {occ: [forward_warp(im, d, proj(H, W), s, occlusion=occ) for s in src] for occ in MODES}
    monkeypatch.setattr(warp, "WORKSPACE_BUDGET", int(3.5 * H * W * 12))
    for occ in MODES:
        batch = check(image, depth, proj(H, W), src, occ)
        for p, single in enumerate(singles[occ]):
            for b, s in zip(batch, single):
                assert torch.equal(b[p], s)


def test_non_default_stream():
    H, W = 200, 256
    image, depth = scene(H, W, seed=15)
    src = random_poses(H, W, 6, seed=16)
    dev = torch.device("cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        im, d = torch.from_numpy(image).to(dev, non_blocking=False), torch.from_numpy(depth).to(dev)
        rgb, dep, hit = forward_warp(im, d, proj(H, W), src, occlusion="zbuffer")
        rgb2, dep2, hit2 = (t.cpu() for t in (rgb, dep, hit))
    want = wo.forward_warp(image, depth, warp_matrices(proj(H, W), src), "zbuffer")
    for g, w in zip((rgb2, dep2, hit2), want):
        assert np.array_equal(g.numpy().view(np.uint8), w.view(np.uint8))


def test_repeatable():
    H, W = 378, 504
    image, depth = scene(H, W, seed=17, holes=0.4)
    dev = torch.device("cuda")
    im, d = torch.from_numpy(image).to(dev), torch.from_numpy(depth).to(dev)
    src = random_poses(H, W, 8, seed=18)
    a = forward_warp(im, d, proj(H, W), src)
    b = forward_warp(im, d, proj(H, W), src)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
