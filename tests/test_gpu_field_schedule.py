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
    if base.dtype == torch.float32:   # compare the bits
        shared, base = shared.view(torch.int32), base.view(torch.int32)
    bad = (shared != base).reshape(-1, base.shape[-1]).any(dim=1)   # per point
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} points differ, first at {int(bad.nonzero()[0])}"


def field_forward(lib, img, prec, rays, z, sigma_only):
    from sinnerf_b200 import _lib
    n = rays.shape[0]
    raw = torch.full((n, S, 1 if sigma_only else 4), float("nan"), device=DEV)
    _lib.check(lib.snb_field_forward(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S, int(sigma_only),
                                     _lib.ptr(raw), _lib.stream_ptr(torch.device(DEV))), "snb_field_forward")
    torch.cuda.synchronize()
    return raw


# act16 sections in order (csrc/act16.cuh): enc, dir, h1..h8, g as fp16 T32 tensors, then the mask words
A16_SECTIONS = [("enc", 64), ("dir", 32)] + [(f"h{l + 1}", 256) for l in range(8)] + [("g", 128)]


def act16_planes(act16, P):
    """The act16 buffer of P points decoded row-major: {section: (Ppad, F) int16, the fp16 bit patterns} and 'mask':
    (8, Ppad, 256) bool, [l, p, c] the stored ReLU bit of h_{l+1}[p][c].
    Byte offset of the 16-byte cell (p, f8) of a (Ppad, F) tensor: ((p >> 5) * (F >> 3) + f8) * 512 + (p & 31) * 16;
    mask word w of layer l, point p at ((l * 8 + w) * Ppad + p), bit c for feature 32 w + c."""
    ppad = (P + 127) // 128 * 128
    out, off = {}, 0
    for name, F in A16_SECTIONS:
        n = ppad * F * 2
        out[name] = act16[off:off + n].view(torch.int16).reshape(ppad // 32, F // 8, 32, 8).permute(0, 2, 1, 3).reshape(ppad, F)
        off += n
    words = act16[off:off + 8 * 8 * ppad * 4].view(torch.int32).reshape(8, 8, ppad)
    bits = (words[..., None] >> torch.arange(32, device=act16.device, dtype=torch.int32)) & 1
    out["mask"] = bits.permute(0, 2, 1, 3).reshape(8, ppad, 256).bool()
    return out


def train_forward(lib, img, prec, rays, z, sigma_only, storage, fill=0xAB):
    """One training forward of n rays x S samples: storage 'fp32' runs snb_field_forward_train[_sigma], 'fp16'
    snb_field_forward_train16[_sigma] on an act16 buffer filled with `fill` bytes.  -> {name: tensor whose first axis
    is the point}: 'raw' (P, 4) or sigma (P, 1), 'enc', 'h1'..'h8' and, unless sigma_only, 'dir' and 'g' -- fp32 rows
    or act16 fp16 bit patterns -- and for 'fp16' 'mask' (P, 8, 256); plus 'act16' itself, undecoded."""
    from sinnerf_b200 import _lib
    n = rays.shape[0]
    S_ = z.shape[1]
    P = n * S_
    st = _lib.stream_ptr(torch.device(DEV))
    raw = torch.full((P, 1 if sigma_only else 4), float("nan"), device=DEV)
    out = {"raw": raw}
    if storage == "fp32":
        save = {k: torch.full(shape, float("nan"), device=DEV)
                for k, shape in (("enc", (P, 64)), ("dir", (P, 32)), ("h", (8, P, 256)), ("g", (P, 128)))}
        if sigma_only:
            rc = lib.snb_field_forward_train_sigma(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S_, _lib.ptr(raw),
                                                   _lib.ptr(save["enc"]), _lib.ptr(save["h"]), st)
        else:
            rc = lib.snb_field_forward_train(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S_, _lib.ptr(raw),
                                             _lib.ptr(save["enc"]), _lib.ptr(save["dir"]), _lib.ptr(save["h"]),
                                             _lib.ptr(save["g"]), st)
        _lib.check(rc, f"training forward fp32 sigma_only={sigma_only}")
        torch.cuda.synchronize()
        out["enc"] = save["enc"]
        out.update({f"h{l + 1}": save["h"][l] for l in range(8)})
        if not sigma_only:
            out["dir"], out["g"] = save["dir"], save["g"]
        return out
    act16 = torch.full((lib.snb_act16_bytes(P),), fill, dtype=torch.uint8, device=DEV)
    entry = lib.snb_field_forward_train16_sigma if sigma_only else lib.snb_field_forward_train16
    _lib.check(entry(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), n, S_, _lib.ptr(raw), _lib.ptr(act16), st),
               f"training forward fp16 sigma_only={sigma_only}")
    torch.cuda.synchronize()
    planes = act16_planes(act16, P)
    for name, _ in A16_SECTIONS:
        if not (sigma_only and name in ("dir", "g")):
            out[name] = planes[name][:P]
    out["mask"] = planes["mask"][:, :P].permute(1, 0, 2)
    out["act16"] = act16
    return out


# (sigma_only, storage) of the fused entries: storage None is the inference kernel (snb_field_forward), 'fp32' / 'fp16'
# the training forwards keeping fp32 rows / act16 (the ids of the inference entries are the plain sigma_only flags)
ENTRIES = [pytest.param(False, None, id="False"), pytest.param(True, None, id="True"),
           pytest.param(False, "fp32", id="train"), pytest.param(True, "fp32", id="train_sigma"),
           pytest.param(False, "fp16", id="train16"), pytest.param(True, "fp16", id="train16_sigma")]


@pytest.mark.parametrize("precision", TENSOR_MODES)
@pytest.mark.parametrize("sigma_only,storage", ENTRIES)
def test_field_rows_independent_of_tile_offset(precision, sigma_only, storage):
    """The fused (rays, z) entries: every output row, and for the training forwards every saved row (fp32 rows, act16
    cells and ReLU mask bits), is the same bits with the points shifted by 33 k rows (k = 1, 37, 127) in the tiles."""
    from sinnerf_b200 import _lib, synthetic
    lib = _lib.load()
    prec = _lib.precision_id(precision)
    img = packed_image(precision)
    rays_all = synthetic.frame_rays("lego", seed=0)[:N_RAYS + 127].to(DEV).contiguous()
    g = torch.Generator(device=DEV).manual_seed(7)
    z_all = (torch.linspace(2, 6, S, device=DEV)[None, :] +
             torch.rand(N_RAYS + 127, S, device=DEV, generator=g) * 0.1).contiguous()

    def run(k):
        r, zz = rays_all[127 - k:].contiguous(), z_all[127 - k:].contiguous()
        if storage is None:
            return {"raw": field_forward(lib, img, prec, r, zz, sigma_only).reshape(-1, 1 if sigma_only else 4)}
        out = train_forward(lib, img, prec, r, zz, sigma_only, storage)
        out.pop("act16", None)
        return out

    base = run(0)
    assert torch.isfinite(base["raw"]).all()
    for k in (1, 37, 127):   # k extra rays in front shift every point by 33 k rows modulo the 128-row tile
        out = run(k)
        assert out.keys() == base.keys()
        for name, want in base.items():
            assert_rows_equal(out[name][S * k:], want, f"{precision} sigma_only={sigma_only} storage={storage} k={k} {name}")
        del out


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


@pytest.mark.parametrize("precision", TENSOR_MODES)
def test_train16_saves_the_fp32_activations_rounded(precision):
    """The two training forwards run the same epilogue arithmetic and differ only in what they save.
    snb_field_forward_train16's raw output is the same bits as snb_field_forward_train's; each of its fp16 T32 cells is
    the fp32 activation the other saves, saturated and rounded to fp16; its ReLU mask bits are the signs of the saved
    layer outputs.  52 800 points leave the last tile partial; the padded points must be zero."""
    from sinnerf_b200 import _lib, synthetic
    lib = _lib.load()
    prec = _lib.precision_id(precision)
    img = packed_image(precision)
    rays = synthetic.frame_rays("lego", seed=0)[:N_RAYS].to(DEV).contiguous()
    g = torch.Generator(device=DEV).manual_seed(7)
    z = (torch.linspace(2, 6, S, device=DEV)[None, :] + torch.rand(N_RAYS, S, device=DEV, generator=g) * 0.1).contiguous()
    P = N_RAYS * S
    assert P % 128 != 0
    st = _lib.stream_ptr(torch.device(DEV))

    raw32 = torch.full((N_RAYS, S, 4), float("nan"), device=DEV)
    save = {k: torch.full(shape, float("nan"), device=DEV)
            for k, shape in (("enc", (P, 64)), ("dir", (P, 32)), ("h", (8, P, 256)), ("g", (P, 128)))}
    _lib.check(lib.snb_field_forward_train(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), N_RAYS, S, _lib.ptr(raw32),
                                           _lib.ptr(save["enc"]), _lib.ptr(save["dir"]), _lib.ptr(save["h"]),
                                           _lib.ptr(save["g"]), st), "snb_field_forward_train")
    raw16 = torch.full((N_RAYS, S, 4), float("nan"), device=DEV)
    act16 = torch.full((lib.snb_act16_bytes(P),), 0xAB, dtype=torch.uint8, device=DEV)   # no cell may keep this
    _lib.check(lib.snb_field_forward_train16(_lib.ptr(img), prec, _lib.ptr(rays), _lib.ptr(z), N_RAYS, S, _lib.ptr(raw16),
                                             _lib.ptr(act16), st), "snb_field_forward_train16")
    torch.cuda.synchronize()
    assert torch.isfinite(raw32).all()
    assert_rows_equal(raw16, raw32, f"{precision} raw")

    planes = act16_planes(act16, P)
    want = [("enc", save["enc"]), ("dir", save["dir"])] + [(f"h{l + 1}", save["h"][l]) for l in range(8)] + \
        [("g", save["g"])]
    for name, ref in want:
        got = planes[name]
        assert_rows_equal(got[:P], ref.clamp(-65504, 65504).half().view(torch.int16), f"{precision} {name}")
        assert not bool(got[P:].any()), f"{precision} {name}: padded points are not zero"
    bits = planes["mask"]
    for l in range(8):
        assert_rows_equal(bits[l, :P], save["h"][l] > 0, f"{precision} mask of h{l + 1}")
    assert not bool(bits[:, P:].any()), f"{precision} mask: padded points are not zero"
