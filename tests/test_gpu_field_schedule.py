"""The fused field kernel's result for a point must not depend on where the point sits in a 128-point tile or on
which tile of a CTA's sequence holds it.  The kernel hands the shared activation buffer from one layer's epilogue to
the next layer's wgmmas in 32-column blocks while other wgmmas are still in flight; a hand-over race shows up as rows
whose output changes when the same points are shifted to other tile offsets."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S = 33            # samples per ray: a ray's points straddle tile boundaries at every offset
N_RAYS = 1600     # 52 800 points = 413 tiles, several per CTA
TENSOR_MODES = ["f16x3", "bf16x3", "bf16"]


def tensor_modes():
    """The tensor-core precision modes this build has (the fp32 mode runs the SIMT kernel)."""
    from sinnerf_b200 import _lib
    lib = _lib.load()
    return [m for m, i in _lib.PRECISIONS.items() if m != "fp32" and lib.snb_packed_weights_bytes(i) > 0]


def packed_image(precision):
    if precision not in tensor_modes():
        pytest.skip(f"precision mode {precision} is not built")
    from sinnerf_b200 import _lib
    from sinnerf_b200.nerf import NeRF
    from sinnerf_b200.synthetic import default_init_params
    m = NeRF(use_new_activation=True)
    m.load_state_dict(default_init_params(1))
    return m.to(DEV).packed_weights(_lib.precision_id(precision))


def assert_rows_equal(shared, base, what):
    bad = (shared.view(torch.int32) != base.view(torch.int32)).reshape(-1, base.shape[-1]).any(dim=1)   # per point
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} points differ, first at {int(bad.nonzero()[0])}"


def field_forward(lib, img, prec, rays, z, sigma_only):
    from sinnerf_b200 import _lib
    n = rays.shape[0]
    raw = torch.full((n, S, 1 if sigma_only else 4), float("nan"), device=DEV)
    _lib.check(lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, int(sigma_only),
                                     _lib.ptr(raw), _lib.stream_ptr(torch.device(DEV))), "snb_field_forward")
    torch.cuda.synchronize()
    return raw


@pytest.mark.parametrize("precision", TENSOR_MODES)
@pytest.mark.parametrize("sigma_only", [False, True])
def test_field_rows_independent_of_tile_offset(precision, sigma_only):
    from sinnerf_b200 import _lib, synthetic
    lib = _lib.load()
    prec = _lib.precision_id(precision)
    img = packed_image(precision)
    rays_all = synthetic.frame_rays("lego", seed=0)[:N_RAYS + 127].to(DEV).contiguous()
    g = torch.Generator(device=DEV).manual_seed(7)
    z_all = (torch.linspace(2, 6, S, device=DEV)[None, :] +
             torch.rand(N_RAYS + 127, S, device=DEV, generator=g) * 0.1).contiguous()
    rays, z = rays_all[127:], z_all[127:]
    base = field_forward(lib, img, prec, rays.contiguous(), z.contiguous(), sigma_only)
    assert torch.isfinite(base).all()
    for k in (1, 37, 127):   # k extra rays in front shift every point by 33 k rows modulo the 128-row tile
        out = field_forward(lib, img, prec, rays_all[127 - k:].contiguous(), z_all[127 - k:].contiguous(), sigma_only)
        assert_rows_equal(out[k:], base, f"{precision} sigma_only={sigma_only} k={k}")


@pytest.mark.parametrize("precision", TENSOR_MODES)
@pytest.mark.parametrize("sigma_only", [False, True])
def test_embedded_rows_independent_of_tile_offset(precision, sigma_only):
    """The same for the embedded entry (NeRF.forward on encoded rows), which runs the same consumer schedule."""
    from sinnerf_b200 import _lib
    lib = _lib.load()
    prec = _lib.precision_id(precision)
    img = packed_image(precision)
    n, cin = N_RAYS * S, 63 + 27
    g = torch.Generator(device=DEV).manual_seed(11)
    x_all = (torch.rand(n + 127, cin, device=DEV, generator=g) * 2 - 1).contiguous()

    def run(x):
        out = torch.full((x.shape[0], 1 if sigma_only else 4), float("nan"), device=DEV)
        _lib.check(lib.snb_mlp_forward(_lib.ptr(img), prec, _lib.ptr(x), cin, x.shape[0], int(sigma_only),
                                       _lib.ptr(out), _lib.stream_ptr(torch.device(DEV))), "snb_mlp_forward")
        torch.cuda.synchronize()
        return out

    base = run(x_all[127:].contiguous())
    assert torch.isfinite(base).all()
    for k in (1, 37, 127):
        assert_rows_equal(run(x_all[127 - k:].contiguous())[k:], base, f"{precision} sigma_only={sigma_only} k={k}")
