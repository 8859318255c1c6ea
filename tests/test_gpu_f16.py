"""GPU tests of the single-product fp16 precision mode ('f16', SNB_PREC_F16: nn.Linear operands in fp16, fp32
accumulate, everything else fp32 -- the reference's arithmetic under Lightning's precision=16) and of the 'autocast'
precision policy that selects it inside fp16 CUDA autocast.

The mode is held to the CPU oracle restating exactly that arithmetic (tests/f16_oracle.py), to the fp32 oracle (it
must err less than half as much as bf16, the claim the mode exists for), layer by layer to float64, and bit for bit to
itself across tile offsets, training storages, the policy and GradScaler.  Measured numbers sit beside their bars
(NVIDIA H100 80GB HBM3 at a 400 W power limit)."""
import sys

import pytest
import torch

from oracle import render_oracle as orc
from tests import f16_oracle
from tests._common import rel_l2, room_params
from tests.test_gpu_field_schedule import ENTRIES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")
TT_KEYS = ("opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")


def weights(tag):
    return (room_params("coarse"), room_params("fine")) if tag == "room" else \
        (orc.default_init_params(0), orc.default_init_params(1))


def make_models(pc, pf):
    from sinnerf_b200.nerf import NeRF
    ms = []
    for p in (pc, pf):
        m = NeRF(use_new_activation=True)
        m.load_state_dict(p)
        ms.append(m.to(DEV))
    return ms


def embeddings():
    from sinnerf_b200.nerf import Embedding
    return [Embedding(3, 10), Embedding(3, 4)]


def room_rays(n):
    """n rays of the LLFF-shape patch (the scene room.ckpt was trained on), cut as the patch datasets cut them."""
    from sinnerf_b200 import synthetic
    return synthetic.patch_rays("llff", 63, 84, 4, seed=0)[:n].contiguous()


class storage:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        from sinnerf_b200 import config
        self.before = config.get_train_storage()
        config.set_train_storage(self.name)

    def __exit__(self, *exc):
        from sinnerf_b200 import config
        config.set_train_storage(self.before)


# --------------------------------------------------------------------------------------------------------------------
# 1. inference against the oracle's fp16 restatement
# --------------------------------------------------------------------------------------------------------------------
# rel-L2 per output, the oracle fed the kernels' own fine depths (the fine pass is chaotic in the coarse weights).
# Measured worst: 2.2e-6 default-init, 3.4e-4 room.ckpt (H100 80GB HBM3, 400 W)
INF_BAR = 3e-3


@pytest.mark.parametrize("tag", ["default", "room"])
@pytest.mark.parametrize("test_time", [False, True])
def test_inference_matches_fp16_oracle(tag, test_time):
    from sinnerf_b200.rendering import render_rays
    pc, pf = weights(tag)
    rays = room_rays(512)
    with torch.no_grad():
        out = render_rays(make_models(pc, pf), embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False,
                          test_time=test_time, precision="f16", _return_intermediates=True)
    z_f = out["_inter"]["z_fine"].cpu()
    with torch.no_grad():
        ref = f16_oracle.render_rays(pc, pf, rays, N_samples=64, N_importance=64, perturb=0, noise_std=0,
                                     test_time=test_time, z_fine_override=z_f)
    worst = 0.0
    for k in (TT_KEYS if test_time else KEYS):
        e = rel_l2(out[k].cpu(), ref[k])
        worst = max(worst, e)
        assert e <= INF_BAR, (tag, test_time, k, e)
    print(f"f16 inference vs fp16 oracle ({tag}, test_time={test_time}): worst rel-L2 {worst:.2e}", file=sys.stderr)


# --------------------------------------------------------------------------------------------------------------------
# 2. the claim: against the fp32 oracle, f16 errs at most half as much as bf16
# --------------------------------------------------------------------------------------------------------------------
def test_f16_error_is_at_most_half_of_bf16():
    from sinnerf_b200.rendering import render_rays
    pc, pf = weights("room")
    rays = room_rays(2048)
    models = make_models(pc, pf)
    with torch.no_grad():
        ref = orc.render_rays(pc, pf, rays, N_samples=64, N_importance=64, perturb=0, noise_std=0)
        err = {}
        for mode in ("bf16", "f16"):
            out = render_rays(models, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False, precision=mode)
            err[mode] = {k: rel_l2(out[k].cpu(), ref[k]) for k in ("rgb_fine", "depth_fine", "opacity_fine")}
    print(f"rel-L2 vs the fp32 oracle, room.ckpt, 2048 rays: {err}", file=sys.stderr)
    for k in ("rgb_fine", "depth_fine"):
        assert err["f16"][k] <= 0.5 * err["bf16"][k], (k, err)


# --------------------------------------------------------------------------------------------------------------------
# 3-4. the field-schedule checks of tests/test_gpu_field_schedule.py, run on the f16 mode
# --------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def schedule_checks(monkeypatch):
    """tests/test_gpu_field_schedule.py with 'f16' among the modes it builds images for."""
    from tests import test_gpu_field_schedule as fs
    modes = fs.tensor_modes()
    monkeypatch.setattr(fs, "tensor_modes", lambda: modes + ["f16"])
    return fs


@pytest.mark.parametrize("sigma_only,storage", ENTRIES)
def test_field_rows_independent_of_tile_offset(schedule_checks, sigma_only, storage):
    schedule_checks.test_field_rows_independent_of_tile_offset("f16", sigma_only, storage)


@pytest.mark.parametrize("sigma_only", [False, True])
def test_embedded_rows_independent_of_tile_offset(schedule_checks, sigma_only):
    schedule_checks.test_embedded_rows_independent_of_tile_offset("f16", sigma_only)


def test_train16_saves_the_fp32_activations_rounded(schedule_checks):
    """snb_field_forward_train16's raw output is the same bits as snb_field_forward_train's, and its act16 cells are
    the round-to-nearest fp16 of the fp32 saves."""
    schedule_checks.test_train16_saves_the_fp32_activations_rounded("f16")


# --------------------------------------------------------------------------------------------------------------------
# 5. training forward layer by layer against float64 (tests/test_gpu_layerwise.py with fp16 operands)
# --------------------------------------------------------------------------------------------------------------------
# Bars on the normalised error |h - h_ref| / (|W| |x| + |b|), ~10x above the worst case measured over both weight sets
# and both ray batches (H100 80GB HBM3, 400 W):
#            enc      h max    h rms    g        sigma    rgb
#   measured 4.8e-7   8.9e-7   2.0e-7   6.6e-7   2.6e-7   4.9e-8
F16_BOUNDS = (5.0e-6, 9.0e-6, 2.0e-6, 7.0e-6, 3.0e-6, 5.0e-7)
# The encodings are the fast sin / cos of the single-product modes; their bar must stay well below fp16's rounding of an
# encoded value in [-1, 1] (2^-11 relative), or the operand the MMA sees would depend on the approximation.
assert F16_BOUNDS[0] * 50 <= 2.0 ** -11


@pytest.mark.parametrize("tag", ["default", "room"])
def test_training_forward_layerwise(tag):
    """Every saved tensor of snb_field_forward_train in f16 against float64 from the kernel's own saved inputs, their
    MMA operands rounded to nearest fp16: 4096 lego rays x 128 samples and a ragged DTU batch."""
    from tests import test_gpu_layerwise as tl
    tl.check_forward_layers("f16", tag, "lego", 4096, 128, 21, bounds=F16_BOUNDS)
    tl.check_forward_layers("f16", tag, "dtu", 333, 97, 22, bounds=F16_BOUNDS)


# --------------------------------------------------------------------------------------------------------------------
# 6. parameter gradients against autograd through the fp16 restatement
# --------------------------------------------------------------------------------------------------------------------
# Per-tensor rel-L2 bars (coarse, fine).  The backward differentiates with the fp32 parameters, the oracle's
# straight-through gradients with the fp16-rounded ones (2^-11 relative per element), and the forwards differ by the
# order of their fp32 sums (3e-4 on room.ckpt outputs, test 1), which the first trunk layers' gradients amplify.
# Measured worst per tensor (H100 80GB HBM3, 400 W): room.ckpt 1.02e-2 (xyz_encoding_1/2, either storage; sigma-only
# passes 4.3e-3), default-init 6.7e-3 (sigma-only 8.5e-3).  The bf16 mode's bar is 2e-2 (tests/test_gpu_round2.py).
GRAD_BARS = (2e-2, 2e-2)


@pytest.mark.parametrize("store", ["fp16", "fp32"])
@pytest.mark.parametrize("test_time", [False, True])
@pytest.mark.parametrize("tag", ["default", "room"])
def test_gradients_match_fp16_oracle_autograd(store, test_time, tag):
    from sinnerf_b200.rendering import render_rays
    pc, pf = weights(tag)
    rays = room_rays(64)
    keys = TT_KEYS if test_time else KEYS
    with storage(store):
        models = make_models(pc, pf)
        out = render_rays(models, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False, test_time=test_time,
                          precision="f16", _return_intermediates=True)
    z_f = out["_inter"]["z_fine"].detach().cpu()
    oc = {k: v.clone().requires_grad_(True) for k, v in pc.items()}
    of = {k: v.clone().requires_grad_(True) for k, v in pf.items()}
    ref = f16_oracle.render_rays(oc, of, rays, N_samples=64, N_importance=64, perturb=0, noise_std=0,
                                 test_time=test_time, z_fine_override=z_f)
    g = torch.Generator().manual_seed(3)
    proj = {k: torch.randn(ref[k].shape, generator=g) for k in keys}
    sum((ref[k] * proj[k]).sum() for k in keys).backward()
    sum((out[k] * proj[k].to(DEV)).sum() for k in keys).backward()
    worst = 0.0
    for refp, model, bar in ((oc, models[0], GRAD_BARS[0]), (of, models[1], GRAD_BARS[1])):
        sd = dict(model.named_parameters())
        for k, v in refp.items():
            if v.grad is None:
                assert sd[k].grad is None, k
                continue
            if float(v.grad.norm()) == 0.0:
                continue
            e = rel_l2(sd[k].grad.cpu(), v.grad)
            worst = max(worst, e)
            assert e <= bar, (store, test_time, tag, k, e)
    print(f"f16 gradients vs fp16 oracle ({store}, test_time={test_time}, {tag}): worst rel-L2 {worst:.2e}",
          file=sys.stderr)


# --------------------------------------------------------------------------------------------------------------------
# 7. the 'autocast' policy, bit for bit
# --------------------------------------------------------------------------------------------------------------------
# The backward sums the per-point contributions to a parameter gradient with fp32 atomics from several CTAs, so at more
# than one 32-point tile per pass two identical runs differ in the last bits of the gradients (their order of addition
# varies).  Gradients are therefore compared bit for bit on one ray with 16 + 16 samples: each pass is a single tile
# and every gradient element receives exactly one atomic add onto zero.
ONE_TILE = (1, 16, 16)          # rays, N_samples, N_importance
WIDE = (1024, 64, 64)


def render_and_grads(pc, pf, precision, autocast_dtype, test_time, shape):
    from sinnerf_b200.rendering import render_rays
    n, S, Ni = shape
    rays = room_rays(n).to(DEV)
    models = make_models(pc, pf)
    keys = TT_KEYS if test_time else KEYS
    g = torch.Generator(device=DEV).manual_seed(9)
    rng = {"perturb_u": torch.rand(n, S, device=DEV, generator=g), "noise_coarse": torch.randn(n, S, device=DEV, generator=g),
           "pdf_u": torch.rand(n, Ni, device=DEV, generator=g), "noise_fine": torch.randn(n, S + Ni, device=DEV, generator=g)}
    with torch.autocast("cuda", dtype=autocast_dtype or torch.float16, enabled=autocast_dtype is not None):
        out = render_rays(models, embeddings(), rays, S, False, 1.0, 1.0, Ni, 32768, False, test_time=test_time,
                          precision=precision, _rng=rng)
        loss = sum((out[k] * torch.randn(out[k].shape, device=DEV, generator=g)).sum() for k in keys)
    loss.backward()
    return {k: out[k].detach() for k in keys}, [p.grad for m in models for p in m.parameters()]


def assert_same_bits(a, b, what):
    assert a.keys() == b.keys() if isinstance(a, dict) else len(a) == len(b)
    pairs = [(k, a[k], b[k]) for k in a] if isinstance(a, dict) else [(i, x, y) for i, (x, y) in enumerate(zip(a, b))]
    for k, x, y in pairs:
        if x is None or y is None:
            assert x is None and y is None, (what, k)
            continue
        assert x.dtype == y.dtype == torch.float32, (what, k, x.dtype, y.dtype)
        assert torch.equal(x.detach().view(torch.int32), y.detach().view(torch.int32)), (what, k)


@pytest.mark.parametrize("test_time", [False, True])
def test_autocast_policy_equals_the_mode_it_names(test_time):
    """Under precision='autocast' a training pass inside fp16 autocast is the f16 pass, inside bf16 autocast the bf16
    pass and outside autocast the f16x3 pass: outputs bit for bit on 1024 rays, outputs and parameter gradients bit for
    bit on one tile."""
    from sinnerf_b200 import config
    pc, pf = weights("room")
    for dtype, mode in ((torch.float16, "f16"), (torch.bfloat16, "bf16"), (None, "f16x3")):
        want = render_and_grads(pc, pf, mode, None, test_time, WIDE)
        got = render_and_grads(pc, pf, "autocast", dtype, test_time, WIDE)
        assert_same_bits(got[0], want[0], f"outputs, autocast {dtype}")
        want = render_and_grads(pc, pf, mode, None, test_time, ONE_TILE)
        got = render_and_grads(pc, pf, "autocast", dtype, test_time, ONE_TILE)
        assert_same_bits(got[0], want[0], f"outputs (one tile), autocast {dtype}")
        assert_same_bits(got[1], want[1], f"gradients (one tile), autocast {dtype}")
    # the process-wide setting takes the policy too, and inference follows it as well
    from sinnerf_b200.rendering import render_rays
    rays = room_rays(1024).to(DEV)
    models = make_models(pc, pf)
    before = config.get_precision()
    try:
        config.set_precision("autocast")
        with torch.no_grad():
            with torch.autocast("cuda", dtype=torch.float16):
                got = render_rays(models, embeddings(), rays, 64, False, 0, 0, 64, test_time=test_time)
            want = render_rays(models, embeddings(), rays, 64, False, 0, 0, 64, test_time=test_time, precision="f16")
    finally:
        config.set_precision(before)
    assert_same_bits({k: got[k] for k in TT_KEYS}, {k: want[k] for k in TT_KEYS}, "inference under set_precision('autocast')")


# --------------------------------------------------------------------------------------------------------------------
# 8. GradScaler with the fused optimisers, as Lightning drives them
# --------------------------------------------------------------------------------------------------------------------
def train_steps(pc, pf, opt_cls, scaler, n_steps, shape):
    from sinnerf_b200.rendering import render_rays
    n, S, Ni = shape
    rays = room_rays(n).to(DEV)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    models = make_models(pc, pf)
    opt = opt_cls(models, lr=1e-3, precision="autocast")
    for _ in range(n_steps):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            out = render_rays(models, embeddings(), rays, S, False, 0, 0, Ni, 32768, False, precision="autocast")
            loss = ((out["rgb_fine"] - target) ** 2).mean() + ((out["rgb_coarse"] - target) ** 2).mean()
        if scaler is None:
            loss.backward()
            opt.step()
        else:
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()
    return models


@pytest.mark.parametrize("opt_name", ["FusedAdam", "FusedRAdam"])
def test_grad_scaler_steps_equal_unscaled_steps(opt_name):
    """scaler.scale(loss).backward(); scaler.step(opt); scaler.update() with init_scale 2^16 gives the parameters of the
    unscaled steps bit for bit (on one tile, see ONE_TILE): a power-of-two scale passes exactly through the fp32
    compositing backward and the power-of-two fp16 gradient scales the backward chooses on the device, and unscale_
    multiplies by its exact inverse.  After the steps on 1024 rays the f16 image the next pass reads is already up to
    date: the step re-packs the image of the models' last pass, not the f16x3 image the policy names outside autocast."""
    from sinnerf_b200 import _lib, optim
    opt_cls = getattr(optim, opt_name)
    pc, pf = weights("room")
    plain = train_steps(pc, pf, opt_cls, None, 3, ONE_TILE)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    scaled = train_steps(pc, pf, opt_cls, scaler, 3, ONE_TILE)
    assert scaler.get_scale() == 2.0 ** 16          # no step was skipped for an inf / nan
    for a, b in zip(plain, scaled):
        assert_same_bits(dict(a.named_parameters()), dict(b.named_parameters()), f"{opt_name} parameters")
    scaled = train_steps(pc, pf, opt_cls, torch.amp.GradScaler("cuda", init_scale=2.0 ** 16), 3, WIDE)
    f16 = _lib.precision_id("f16")
    for m in scaled:
        assert m._last_prec == f16
        img = m._packed[(f16, str(torch.device(DEV)))].clone()     # as the step left it, before any refresh
        fresh = make_models(m.state_dict(), m.state_dict())[0]
        # past the 256-byte header (checksum and check scratch): constants, chunks, folded direction-layer weights
        assert torch.equal(img[256:], fresh.packed_weights(f16)[256:]), "the step left a stale f16 image"
