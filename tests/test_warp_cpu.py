"""CPU tests of the forward warp: the numpy oracle (tests/warp_oracle.py) against the reference datasets' own warps
(tests/golden/warp.npz, written by tests/golden/make_warp_golden.py), the occlusion rule against the literal loops,
and the argument checks of sinnerf_b200.warp and the C ABI.  The kernels are checked against the oracle bit for bit
on the H100 by tests/test_gpu_warp.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from sinnerf_b200 import _lib, build
from sinnerf_b200.warp import forward_warp, warp_matrices
from tests import warp_oracle as wo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "warp.npz")
# variant -> occlusion, poses (tests/golden/make_warp_golden.py CASES)
VARIANTS = {"llff": ("zbuffer", ("small", "large", "sideways", "identity")), "dtu": ("zbuffer", ("small", "large")),
            "rot3d": ("last", ("small", "large", "identity")), "bproj": ("last", ("small", "large"))}
# poses that keep pixel coordinates exact integers: the identity (both), and a pure sideways move (every row)
INTEGER_POSES = ("sideways", "identity")
CASES = [(v, p) for v, (_, poses) in VARIANTS.items() for p in poses]
BOUNDARY_PX = 1e-3


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def full_proj(K, E, dtype=np.float64):
    P = np.eye(4)
    P[:3, :3] = K
    return (P @ E.astype(np.float64)).astype(dtype)


def case(g, variant, pose):
    """inputs, the reference's outputs, the reference's integer targets and fp32 depths, and the contract's M."""
    image, depth = g[f"{variant}/image"], g[f"{variant}/depth"]
    H, W = depth.shape
    K, E_ref, E_src = g[f"{variant}/K"], g[f"{variant}/E_ref"], g[f"{variant}/{pose}/E_src"]
    x, y, z = (g[f"{variant}/{pose}/{k}"] for k in ("x_src", "y_src", "depth_src"))
    ok = ~np.isnan(x) & ~np.isnan(y)
    col = np.clip(np.where(ok, x, 0), 0, W - 1).astype(np.int64)
    row = np.clip(np.where(ok, y, 0), 0, H - 1).astype(np.int64)
    targets = np.where(ok, row * W + col, -1)
    # DTU hands its projections over in fp32 (dtu_proj.py:522-523); LLFF / blender callers compose K and E
    dt = np.float32 if variant == "dtu" else np.float64
    M = warp_matrices(full_proj(K, E_ref, dt), full_proj(K, E_src, dt))[0]
    ref = (g[f"{variant}/{pose}/ref_rgb"], g[f"{variant}/{pose}/ref_depth"], g.get(f"{variant}/{pose}/ref_mask"))
    return image, depth, targets, z, M, ref


@pytest.mark.parametrize("variant,pose", CASES)
def test_resolve_reproduces_reference(golden, variant, pose):
    """The occlusion rule on the reference's own targets and fp32 depths gives the reference's output bit for bit:
    ties, holes, negative depths, Z == 0 (llff/sideways) and the last-writer order."""
    image, depth, targets, z, _, (ref_rgb, ref_depth, ref_mask) = case(golden, variant, pose)
    rgb, dep, hit = wo.resolve(targets, z, image, VARIANTS[variant][0])
    assert np.array_equal(rgb, ref_rgb)
    assert np.array_equal(dep.view(np.uint32), ref_depth.view(np.uint32))
    if ref_mask is not None:
        assert np.array_equal(hit, ref_mask != 0)


def test_golden_covers_the_special_classes(golden):
    _, _, _, z, M, _ = case(golden, "llff", "sideways")
    assert M[2, 3] == 0.0                     # every hole pixel lands at Z == 0 exactly
    assert (golden["llff/depth"] == 0).mean() > 0.15
    for v in ("llff", "dtu", "rot3d", "bproj"):
        assert (golden[f"{v}/large/depth_src"] < 0).sum() > 100      # behind the source camera


@pytest.mark.parametrize("occlusion", ["zbuffer", "last"])
def test_resolve_equals_loop_exhaustive(occlusion):
    """Every sequence of up to 4 sources on one target over {-2, -1, -0, +0, 1, 2, 3} (2800 sequences): the rule is
    the loop's result for all short runs."""
    import itertools
    vals = np.array([-2, -1, -0.0, 0.0, 1, 2, 3], np.float32)
    loop = wo.painter_loop if occlusion == "zbuffer" else wo.scatter_loop
    image = np.arange(12, dtype=np.float32).reshape(1, 4, 3) + 1
    for n in range(1, 5):
        for combo in itertools.product(range(len(vals)), repeat=n):
            zf = vals[list(combo)]
            targets = np.zeros(n, dtype=np.int64)
            got, want = wo.resolve(targets, zf, image[:, :n], occlusion), loop(targets, zf, image[:, :n])
            for a, b in zip(got, want):
                assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), zf


def _random_case(g, n, n_targets):
    zf = g.choice(np.array([-2, -1, -0.0, 0.0, 1, 2, 3], np.float32), n)
    targets = g.integers(-1, n_targets, n)
    image = g.random((1, n, 3)).astype(np.float32)
    return targets, zf, image


@pytest.mark.parametrize("occlusion", ["zbuffer", "last"])
def test_resolve_equals_loop(occlusion):
    """The vectorised rule equals the reference's sequential loop, on sequences over {-2, -1, -0, +0, 1, 2, 3} with
    ties, single-source targets and skipped sources."""
    g = np.random.default_rng(5)
    loop = wo.painter_loop if occlusion == "zbuffer" else wo.scatter_loop
    for trial in range(20000):
        n = int(g.integers(1, 24))
        targets, zf, image = _random_case(g, n, int(g.integers(1, n + 1)))
        targets = np.minimum(targets, n - 1)
        got, want = wo.resolve(targets, zf, image, occlusion), loop(targets, zf, image)
        for a, b in zip(got, want):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), (trial, targets, zf)


def test_resolve_keeps_sign_of_zero():
    image = np.arange(6, dtype=np.float32).reshape(1, 2, 3)
    _, dep, hit = wo.resolve(np.array([0, 0]), np.array([0.0, -0.0], np.float32), image, "zbuffer")
    assert hit[0, 0] and np.signbit(dep[0, 0])


def _boundary(x, y, H, W):
    """Sources whose coordinate lies within BOUNDARY_PX of a pixel boundary that changes the clamped target."""
    def near(t, n):
        k = np.round(t)
        return (np.abs(t - k) < BOUNDARY_PX) & (k >= 1) & (k <= n - 1)
    return near(x, W) | near(y, H)


@pytest.mark.parametrize("variant,pose", CASES)
def test_project_against_reference_coordinates(golden, variant, pose):
    """The fp64 projection picks the reference's pixel for every source except those within 1e-3 px of a pixel
    boundary in the oracle's own coordinate; those are under 1 % of the sources."""
    image, depth, targets, z, M, _ = case(golden, variant, pose)
    got, zf = wo.project(M, depth)
    x, y, _, _ = wo.coordinates(M, depth)
    differ = got != targets
    boundary = _boundary(x, y, *depth.shape)
    assert not (differ & ~boundary).any(), np.nonzero(differ & ~boundary)
    print(f"{variant}/{pose}: {int(differ.sum())} sources land elsewhere, {int(boundary.sum())} of {x.size} within "
          f"{BOUNDARY_PX} px of a boundary")
    if pose in INTEGER_POSES:
        # The fp64 projection puts these sources exactly on their integer coordinate; the reference's fp32 projection
        # puts about half of them a few ulps below it (up to 8e-6 px), and its floor then moves them one pixel.  So
        # every source is a boundary source here, and the ones that land elsewhere are the reference's rounding.
        H, W = depth.shape
        r, c = np.divmod(np.arange(H * W), W)
        valid = depth.reshape(-1) != 0
        assert np.array_equal(y[valid], r[valid].astype(np.float64))
        if pose == "identity":
            assert np.array_equal(x[valid], c[valid].astype(np.float64))
        xr, yr = golden[f"{variant}/{pose}/x_src"], golden[f"{variant}/{pose}/y_src"]
        assert np.all(np.abs(yr - y)[differ & valid] < 1e-4) and np.all(np.abs(xr - x)[differ & valid] < 1e-4)
    else:
        assert boundary.sum() < 0.01 * x.size
    fin = np.isfinite(z) & (z != 0)
    assert np.allclose(zf[fin], z[fin], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("variant,pose", CASES)
def test_oracle_against_reference(golden, variant, pose):
    """End to end: every output pixel where the oracle and the reference disagree is touched by a boundary source;
    elsewhere the rgb and hit are equal and the depths agree to fp32 rounding of the reference's projection."""
    image, depth, targets, z, M, (ref_rgb, ref_depth, ref_mask) = case(golden, variant, pose)
    H, W = depth.shape
    rgb, dep, hit = wo.forward_warp(image, depth, M[None], VARIANTS[variant][0])
    x, y, _, _ = wo.coordinates(M, depth)
    got_t, _ = wo.project(M, depth)
    b = _boundary(x, y, H, W)
    touched = np.zeros(H * W, bool)
    touched[got_t[b & (got_t >= 0)]] = True
    touched[targets[b & (targets >= 0)]] = True
    touched = touched.reshape(H, W)
    bad = (rgb[0] != ref_rgb).any(-1)      # image colours are >= 0.02: rgb also tells hit from miss
    assert not (bad & ~touched).any()
    print(f"{variant}/{pose}: {int(bad.sum())} of {H * W} pixels differ from the reference, {int(touched.sum())} "
          "touched by boundary sources")
    same = ~touched
    assert np.allclose(dep[0][same], ref_depth[same], rtol=1e-5, atol=1e-6)
    if ref_mask is not None:
        assert np.array_equal(hit[0][same], ref_mask[same] != 0)


def test_identity_pose_returns_the_image(golden):
    """Warping into the reference camera itself gives back the image at every pixel with depth (pixel (0, 0), where
    the hole group lands, aside)."""
    for variant in ("llff", "rot3d"):
        image, depth, _, _, M, _ = case(golden, variant, "identity")
        assert np.array_equal(M, np.eye(4)[:3])
        for occ in ("zbuffer", "last"):
            rgb, dep, hit = wo.forward_warp(image, depth, M[None], occ)
            keep = depth != 0
            keep[0, 0] = False
            assert np.array_equal(rgb[0][keep], image[keep]) and np.array_equal(dep[0][keep], depth[keep])
            assert hit[0][keep].all()


# ---- argument checks, all raised before the library is needed ---------------------------------------------------

def _args(H=4, W=5, **kw):
    a = dict(image=torch.zeros(H, W, 3), depth_ref=torch.ones(H, W), ref_proj=torch.eye(4), src_proj=torch.eye(4))
    a.update(kw)
    return a


@pytest.mark.parametrize("bad", [
    dict(image=torch.zeros(4, 5)), dict(image=torch.zeros(4, 5, 4)), dict(depth_ref=torch.ones(5, 4)),
    dict(depth_ref=torch.ones(4, 5, 1)), dict(ref_proj=torch.eye(3)), dict(src_proj=torch.eye(3)),
    dict(src_proj=torch.zeros(0, 4, 4)), dict(src_proj=torch.eye(4)[None, None]), dict(image=torch.zeros(0, 5, 3),
                                                                                       depth_ref=torch.ones(0, 5)),
    dict(ref_proj=torch.zeros(4, 4)), dict(ref_proj=torch.diag(torch.tensor([1.0, 1.0, 0.0, 1.0]))),
])
def test_value_errors(bad):
    with pytest.raises(ValueError):
        a = _args(**bad)
        forward_warp(a["image"], a["depth_ref"], a["ref_proj"], a["src_proj"])


def test_occlusion_mode_is_checked():
    a = _args()
    for occ in ("painter", "", None, "ZBUFFER"):
        with pytest.raises(ValueError):
            forward_warp(a["image"], a["depth_ref"], a["ref_proj"], a["src_proj"], occlusion=occ)


@pytest.mark.parametrize("bad", [dict(image=torch.zeros(4, 5, 3, dtype=torch.float64)),
                                 dict(depth_ref=torch.ones(4, 5, dtype=torch.float16)),
                                 dict(image=np.zeros((4, 5, 3), np.float32))])
def test_type_errors(bad):
    a = _args(**bad)
    with pytest.raises(TypeError):
        forward_warp(a["image"], a["depth_ref"], a["ref_proj"], a["src_proj"])


def test_cpu_tensors_are_refused():
    a = _args()
    with pytest.raises(RuntimeError, match="CUDA"):
        forward_warp(a["image"], a["depth_ref"], a["ref_proj"], a["src_proj"], occlusion="last")


def test_warp_matrices():
    g = np.random.default_rng(0)
    ref = np.eye(4) + 0.1 * g.standard_normal((4, 4))
    src = np.eye(4) + 0.1 * g.standard_normal((3, 4, 4))
    M = warp_matrices(torch.from_numpy(ref).float(), src)
    assert M.shape == (3, 3, 4) and M.dtype == np.float64 and M.flags.c_contiguous
    want = src @ np.linalg.inv(ref.astype(np.float32).astype(np.float64))
    assert np.allclose(M, want[:, :3], rtol=0, atol=1e-12)
    assert np.array_equal(warp_matrices(ref, src[1]), warp_matrices(ref, src)[1:2])
    # the unmoved camera is exactly the identity, and a pure move changes only the translation column
    K = np.array([[70.4, 0, 32, 0], [0, 70.4, 24, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32).astype(np.float64)
    E = np.diag([1.0, -1.0, -1.0, 1.0])
    moved = E.copy()
    moved[:3, 3] = (-0.5, 0.25, 0.0)
    assert np.array_equal(warp_matrices(K @ E, K @ E)[0], np.eye(4)[:3])
    assert np.array_equal(warp_matrices(K @ E, K @ moved)[0][:, :3], np.eye(3))


# ---- C ABI ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_workspace_bytes(lib):
    assert lib.snb_forward_warp_workspace_bytes(3, 40, 50, 0) == 3 * 40 * 50 * 12
    assert lib.snb_forward_warp_workspace_bytes(3, 40, 50, 1) == 3 * 40 * 50 * 4
    for bad in ((0, 4, 4, 0), (1, 0, 4, 0), (1, 4, 4, 2), (1, 1 << 16, 1 << 15, 1)):
        assert lib.snb_forward_warp_workspace_bytes(*bad) == 0


def test_cabi_argument_errors(lib):
    p = C.c_void_p(16)

    def call(**kw):
        a = dict(image=p, depth=p, height=4, width=4, mats=p, n_poses=1, occlusion=0, rgb=p, dep=p, hit=p, ws=p)
        a.update(kw)
        return lib.snb_forward_warp(*a.values(), None)

    for kw in (dict(image=None), dict(depth=None), dict(mats=None), dict(rgb=None), dict(dep=None), dict(hit=None),
               dict(ws=None), dict(n_poses=0), dict(occlusion=-1), dict(height=0), dict(height=1 << 16, width=1 << 15)):
        assert call(**kw) == -1, kw
        assert lib.snb_last_error()
