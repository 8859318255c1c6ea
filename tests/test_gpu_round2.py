"""Round-2 GPU tests: parity at BASELINE sizes, the weight-image freshness check, fused losses (SURVEY 8f-3),
fused Adam (8f-4), the importance-merge general path, per-device launch state."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

from oracle import render_oracle as orc
from tests._common import assert_close, load_npz, rel_l2, room_params

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def make_models(pc, pf, dev=DEV, new_act=True):
    from sinnerf_b200.nerf import NeRF
    models = []
    for p in (pc, pf):
        m = NeRF(use_new_activation=new_act)
        m.load_state_dict(p)
        models.append(m.to(dev))
    return models


def embeddings():
    from sinnerf_b200.nerf import Embedding
    return [Embedding(3, 10), Embedding(3, 4)]


# ------------------------------------------------------------------------------------------ parity at size
@pytest.mark.parametrize("shape,white_back", [("lego", True), ("dtu", True)])
def test_full_frame_subset_matches_oracle(shape, white_back):
    """BASELINE configs[1] (400x400 = 160 000 rays) and configs[3] (640x512 = 327 680 rays) rendered IN FULL by the
    persistent one-CTA-per-SM kernels; a seeded 2 048-ray subset of the result against the CPU oracle at the SURVEY 8c
    tolerances (tile tails / slot wrap-around only exist at this size).  Also pins how many fine-pass depths of a
    full frame land in a different bin than the oracle's (the cdf is a warp scan here, a serial cumsum there)."""
    from sinnerf_b200 import synthetic
    from sinnerf_b200.rendering import render_rays
    rays = synthetic.frame_rays(shape, seed=0)
    assert rays.shape[0] == (160000 if shape == "lego" else 327680)
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    models = make_models(pc, pf)
    with torch.no_grad():
        out = render_rays(models, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, white_back,
                          _return_intermediates=True)
    torch.cuda.synchronize()
    g = torch.Generator().manual_seed(123)
    idx = torch.sort(torch.randperm(rays.shape[0], generator=g)[:2048])[0]
    # always include the very first / last rays (first tile, tail tile)
    idx[:4] = torch.arange(4)
    idx[-4:] = torch.arange(rays.shape[0] - 4, rays.shape[0])
    sub = rays[idx]
    with torch.no_grad():
        ref = orc.render_rays(pc, pf, sub, N_samples=64, N_importance=64, noise_std=0.0, white_back=white_back)
        z_f = out["_inter"]["z_fine"][idx.to(DEV)].cpu()
        ref_inj = orc.render_rays(pc, pf, sub, N_samples=64, N_importance=64, noise_std=0.0, white_back=white_back,
                                  z_fine_override=z_f)
    for k in ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine"):
        assert_close(out[k][idx.to(DEV)].cpu(), ref[k], 1e-4, f"{shape}:{k}")
    assert_close(out["opacity_fine"][idx.to(DEV)].cpu(), ref_inj["opacity_fine"], 1e-4, f"{shape}:opacity_fine (injected z)")
    assert rel_l2(out["opacity_fine"][idx.to(DEV)].cpu(), ref["opacity_fine"]) <= 1e-3
    # fine depths: sorted everywhere; count the samples that differ from the oracle's own by more than rounding
    zf_all = out["_inter"]["z_fine"]
    assert bool((zf_all[:, 1:] >= zf_all[:, :-1]).all())
    with torch.no_grad():
        ref_z = orc.render_rays(pc, pf, sub, N_samples=64, N_importance=64, noise_std=0.0, white_back=white_back,
                                return_intermediates=True)["_inter"]["z_fine"]
    # (a) samples whose position differs beyond rounding: they sit in bins of near-zero pdf, where
    #     (u - cdf_below) / (cdf_above - cdf_below) divides by ~1e-5 and amplifies the last bits of the cdf
    #     (warp scan here, serial cumsum in torch) -- harmless for the render, bounded here;
    # (b) samples that moved by more than half a coarse bin, i.e. took a different bin at a cdf knot.
    dz = (z_f - ref_z).abs()
    moved = (dz > 1e-4 * ref_z.abs().clamp_min(1.0)).sum().item()
    half_bin = 0.5 * float((sub[0, 7] - sub[0, 6]) / 63)
    jumped = (dz > half_bin).sum().item()
    print(f"{shape}: of {z_f.numel()} fine depths {moved} differ from the oracle's by > 1e-4 rel ({moved / z_f.numel():.2e}), "
          f"{jumped} by more than half a coarse bin ({jumped / z_f.numel():.2e}); max |dz| {float(dz.max()):.3e}", file=sys.stderr)
    assert moved / z_f.numel() <= 5e-2
    assert jumped / z_f.numel() <= 1e-3


def test_c1_full_1024_rays_golden():
    """configs[0] in full: all 1 024 rays, 64 + 0 samples, against the reference-generated golden."""
    from sinnerf_b200.rendering import render_rays
    case = load_npz("render_c1_full_seed0_64p0.npz")
    models = make_models(orc.default_init_params(0), orc.default_init_params(1))
    rays = torch.from_numpy(case["rays"].copy()).to(DEV)
    assert rays.shape[0] == 1024
    for mode in ("fp32", "f16x3"):
        with torch.no_grad():
            out = render_rays(models[:1], embeddings(), rays, 64, False, 0, 0, 0, 32768, False, precision=mode)
        for k in ("rgb_coarse", "depth_coarse", "opacity_coarse"):
            assert_close(out[k].cpu(), case["out_" + k], 1e-4, f"{mode}:{k}")


# ------------------------------------------------------------------------------------------ weight image freshness
def test_packed_image_follows_data_updates_without_version_bump():
    """ADVICE r1 (high): the reference's RAdam / Ranger write weights through `p.data.copy_` (utils/optimizers.py:98),
    which leaves `_version` alone.  The image must follow anyway."""
    from sinnerf_b200.rendering import render_rays
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    models = make_models(pc, pf)
    rays = torch.from_numpy(load_npz("render_lego_seed0_64p64_wb.npz")["rays"].copy()).to(DEV)[:64]
    with torch.no_grad():
        a = render_rays(models, embeddings(), rays, 64, False, 0, 0, 64, 32768, True)
        p = models[1].xyz_encoding_3[0].weight
        v0 = p._version
        p.data.copy_(p.data * 1.5)                   # what RAdam.step does
        assert p._version == v0                      # invisible to the version counter
        b = render_rays(models, embeddings(), rays, 64, False, 0, 0, 64, 32768, True)
        assert not torch.equal(a["rgb_fine"], b["rgb_fine"])
        assert torch.equal(a["rgb_coarse"], b["rgb_coarse"])          # the coarse model did not change
        # and the result equals a freshly built model with the same weights
        pf2 = {k: v.clone() for k, v in pf.items()}
        pf2["xyz_encoding_3.0.weight"] = pf2["xyz_encoding_3.0.weight"] * 1.5
        fresh = make_models(pc, pf2)
        c = render_rays(fresh, embeddings(), rays, 64, False, 0, 0, 64, 32768, True)
        assert torch.equal(b["rgb_fine"], c["rgb_fine"])
        # an untouched model is not re-packed: same image bytes, header says clean
        img = models[0].packed_weights("f16x3")
        before = img.clone()
        models[0].packed_weights("f16x3")
        assert torch.equal(before, models[0].packed_weights("f16x3"))
        hdr = img[:32].cpu().numpy().view(np.int32)
        assert hdr[4] == 0, "dirty flag should be 0 after a no-op refresh"


def test_module_forward_refuses_to_drop_the_graph():
    models = make_models(orc.default_init_params(0), orc.default_init_params(1))
    x = torch.randn(8, 90, device=DEV)
    with pytest.raises(NotImplementedError):
        models[0](x)
    with torch.no_grad():
        assert models[0](x).shape == (8, 4)
    e = embeddings()[0]
    with pytest.raises(NotImplementedError):
        e(torch.randn(4, 3, device=DEV, requires_grad=True))
    assert e(torch.randn(4, 3, device=DEV)).shape == (4, 63)


# ------------------------------------------------------------------------------------------ importance merge
def test_importance_merge_general_path_matches_torch_sort():
    """near > far rays (descending coarse depths) and non-finite depths: the merge falls back to a rank sort with
    torch.sort's order and writes every slot (ADVICE r1: unwritten torch.empty slots fed the fine pass)."""
    from sinnerf_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(5)
    n, S, Ni = 67, 64, 64
    near = torch.full((n,), 6.0)
    far = torch.full((n,), 2.0)              # descending rows
    t = torch.linspace(0, 1, S)
    z = near[:, None] * (1 - t) + far[:, None] * t
    z[5:10] = torch.sort(torch.rand(5, S, generator=g) * 4 + 2, -1)[0]      # some ordinary rows in between
    z[11, 7] = float("nan")
    z[12, 63] = float("inf")
    w = torch.rand(n, S, generator=g)
    u = torch.linspace(0, 1, Ni)
    zf = torch.full((n, S + Ni), -777.0, device=DEV)
    znew = torch.empty(n, Ni, device=DEV)
    zc, wc, ud = z.to(DEV), w.to(DEV), u.to(DEV)
    _lib.check(lib.snb_importance_merge(_lib.ptr(zc), _lib.ptr(wc), _lib.ptr(ud), 0, n, S, Ni, 1e-5, _lib.ptr(zf),
                                        _lib.ptr(znew), _lib.stream_ptr(torch.device(DEV))), "snb_importance_merge")
    torch.cuda.synchronize()
    want = torch.sort(torch.cat([zc, znew], -1), -1)[0]
    got = zf
    assert not bool((got == -777.0).any()), "unwritten slots"
    same = (got == want) | (torch.isnan(got) & torch.isnan(want))
    assert bool(same.all())


# ------------------------------------------------------------------------------------------ fused losses (8f-3)
def _loss_case(n=96):
    case = load_npz("render_llff_room_64p64_train.npz")
    rays = torch.from_numpy(case["rays"].copy())[:n]
    g = torch.Generator().manual_seed(9)
    target_rgb = torch.rand(n, 3, generator=g)
    target_depth = torch.rand(n, generator=g) * 6 + 1.0       # some |depth - target| < 1, some > 1
    return rays, target_rgb, target_depth


def test_fused_losses_match_torch_losses_and_gradients():
    """loss_rgb / loss_depth from the compositing kernels == nn.MSELoss / nn.SmoothL1Loss on the outputs (reference
    losses.py:12-22, models/sinnerf.py:32-42), and the parameter gradients of their weighted sum == autograd
    through the unfused outputs."""
    from sinnerf_b200.rendering import render_rays, RayLosses
    rays, trgb, tdep = _loss_case()
    pc, pf = room_params("coarse"), room_params("fine")
    rng = {"noise_coarse": torch.zeros(rays.shape[0], 64), "noise_fine": torch.zeros(rays.shape[0], 128)}
    mse, sl1 = torch.nn.MSELoss(reduction="mean"), torch.nn.SmoothL1Loss(reduction="mean")

    ma = make_models(pc, pf)
    out = render_rays(ma, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False, _rng=rng)
    l2 = mse(out["rgb_coarse"], trgb.to(DEV)) + mse(out["rgb_fine"], trgb.to(DEV))
    ld = sl1(out["depth_fine"], tdep.to(DEV)) + sl1(out["depth_coarse"], tdep.to(DEV))
    (l2 + 0.25 * ld).backward()

    mb = make_models(pc, pf)
    fused = render_rays(mb, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False, _rng=rng,
                        losses=RayLosses(target_rgb=trgb, target_depth=tdep))
    assert abs(float(fused["loss_rgb"]) - float(l2)) <= 1e-5 * abs(float(l2))
    assert abs(float(fused["loss_depth"]) - float(ld)) <= 1e-5 * abs(float(ld))
    for k in ("rgb_fine", "depth_fine", "rgb_coarse"):
        assert torch.equal(fused[k], out[k]), k
    (fused["loss_rgb"] + 0.25 * fused["loss_depth"]).backward()
    for m_a, m_b in zip(ma, mb):
        for (k, pa), (_, pb) in zip(m_a.named_parameters(), m_b.named_parameters()):
            assert rel_l2(pb.grad.cpu(), pa.grad.cpu()) <= 1e-5, (k, rel_l2(pb.grad.cpu(), pa.grad.cpu()))
    # deterministic reduction
    again = render_rays(mb, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False, _rng=rng,
                        losses=RayLosses(target_rgb=trgb, target_depth=tdep))
    assert torch.equal(again["loss_coarse"], fused["loss_coarse"]) and torch.equal(again["loss_fine"], fused["loss_fine"])


def test_fused_losses_against_oracle_outputs():
    """The loss values against the CPU oracle's outputs run through torch's own loss modules."""
    from sinnerf_b200.rendering import render_rays, RayLosses
    rays, trgb, tdep = _loss_case(48)
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    models = make_models(pc, pf)
    fused = render_rays(models, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, True,
                        losses=RayLosses(target_rgb=trgb, target_depth=tdep), _return_intermediates=True)
    with torch.no_grad():
        ref = orc.render_rays(pc, pf, rays, N_samples=64, N_importance=64, noise_std=0.0, white_back=True,
                              z_fine_override=fused["_inter"]["z_fine"].detach().cpu())
    mse, sl1 = torch.nn.MSELoss(), torch.nn.SmoothL1Loss()
    want_rgb = mse(ref["rgb_coarse"], trgb) + mse(ref["rgb_fine"], trgb)
    want_dep = sl1(ref["depth_coarse"], tdep) + sl1(ref["depth_fine"], tdep)
    assert abs(float(fused["loss_rgb"]) - float(want_rgb)) <= 2e-4 * float(want_rgb)
    assert abs(float(fused["loss_depth"]) - float(want_dep)) <= 2e-4 * float(want_dep)


def test_multi_batch_losses_have_per_batch_normalisation():
    """render_rays_multi(batch_losses=...): batch 0 has rgb + depth targets, batch 1 none (its rgb goes to an external
    loss through ordinary autograd), batch 2 depth only -- the SinNeRF step's pattern (models/sinnerf.py:304-319)."""
    from sinnerf_b200.rendering import render_rays, render_rays_multi, RayLosses
    rays, trgb, tdep = _loss_case(96)
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    sizes = [40, 24, 32]
    parts = torch.split(rays, sizes)
    mse, sl1 = torch.nn.MSELoss(), torch.nn.SmoothL1Loss()
    ext_w = torch.randn(24, 3)

    ma = make_models(pc, pf)
    outs = [render_rays(ma, embeddings(), p.to(DEV), 64, False, 0, 0, 64, 32768, True) for p in parts]
    l2 = mse(outs[0]["rgb_coarse"], trgb[:40].to(DEV)) + mse(outs[0]["rgb_fine"], trgb[:40].to(DEV))
    ld = sl1(outs[0]["depth_fine"], tdep[:40].to(DEV)) + sl1(outs[0]["depth_coarse"], tdep[:40].to(DEV)) \
        + sl1(outs[2]["depth_fine"], tdep[64:].to(DEV)) + sl1(outs[2]["depth_coarse"], tdep[64:].to(DEV))
    ext = (outs[1]["rgb_fine"] * ext_w.to(DEV)).sum()
    (l2 + ld + ext).backward()

    mb = make_models(pc, pf)
    res = render_rays_multi(mb, embeddings(), [p.to(DEV) for p in parts], 64, False, 0, 0, 64, 32768, True,
                            batch_losses=[RayLosses(trgb[:40], tdep[:40]), None, RayLosses(None, tdep[64:])])
    assert abs(float(res[0]["loss_rgb"]) - float(l2)) <= 1e-5 * float(l2)
    assert abs(float(res[0]["loss_depth"]) - float(ld)) <= 1e-5 * float(ld)
    (res[0]["loss_rgb"] + res[0]["loss_depth"] + (res[1]["rgb_fine"] * ext_w.to(DEV)).sum()).backward()
    for m_a, m_b in zip(ma, mb):
        for (k, pa), (_, pb) in zip(m_a.named_parameters(), m_b.named_parameters()):
            assert rel_l2(pb.grad.cpu(), pa.grad.cpu()) <= 2e-4, (k, rel_l2(pb.grad.cpu(), pa.grad.cpu()))


# ------------------------------------------------------------------------------------------ fused Adam (8f-4)
@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
def test_fused_adam_matches_torch_adam(weight_decay):
    """10 steps of FusedAdam against torch.optim.Adam (single-tensor path, the arithmetic the kernel mirrors) on the same
    gradients: parameters and moments bit for bit (the kernel rounds every operation as torch's CUDA ops do); the packed
    image after the last step equals a fresh pack of the final weights."""
    from sinnerf_b200.optim import FusedAdam
    from sinnerf_b200.rendering import render_rays
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    ma, mb = make_models(pc, pf), make_models(pc, pf)
    ref_opt = torch.optim.Adam([p for m in ma for p in m.parameters()], lr=5e-4, eps=1e-8, weight_decay=weight_decay,
                               foreach=False)
    opt = FusedAdam(mb, lr=5e-4, eps=1e-8, weight_decay=weight_decay)
    g = torch.Generator().manual_seed(0)
    for step in range(10):
        if step == 5:
            for o in (ref_opt, opt):
                o.param_groups[0]["lr"] = 2.5e-4          # a scheduler moved the learning rate
        for m_a, m_b in zip(ma, mb):
            for pa, pb in zip(m_a.parameters(), m_b.parameters()):
                gr = (torch.randn(pa.shape, generator=g) * 1e-2).to(DEV)
                pa.grad = gr.clone()
                pb.grad = gr.clone()
        ref_opt.step()
        opt.step()
    worst, exact, total = 0.0, 0, 0
    for m_a, m_b in zip(ma, mb):
        for (k, pa), (_, pb) in zip(m_a.named_parameters(), m_b.named_parameters()):
            d = (pa.detach() - pb.detach()).abs().max().item()
            worst = max(worst, d / pa.detach().abs().max().item())
            exact += int((pa.detach() == pb.detach()).sum())
            total += pa.numel()
            st_a, st_b = ref_opt.state[pa], opt.state[pb]
            assert torch.equal(st_b["exp_avg"], st_a["exp_avg"]), (k, rel_l2(st_b["exp_avg"].cpu(), st_a["exp_avg"].cpu()))
            assert torch.equal(st_b["exp_avg_sq"], st_a["exp_avg_sq"]), k
    print(f"fused adam vs torch: {exact}/{total} parameters bit-equal, worst rel diff {worst:.2e}", file=sys.stderr)
    assert worst <= 3e-7
    assert exact == total
    # the image FusedAdam left behind is the image of the final weights, and it is stamped clean
    rays = torch.from_numpy(load_npz("render_lego_seed0_64p64_wb.npz")["rays"].copy()).to(DEV)[:64]
    img = mb[1].packed_image_buffer(1).clone()
    with torch.no_grad():
        a = render_rays(mb, embeddings(), rays, 64, False, 0, 0, 64, 32768, True)
        assert int(mb[1].packed_image_buffer(1)[:32].cpu().numpy().view(np.int32)[4]) == 0      # refresh found it clean
        fresh = make_models({k: v.detach().cpu() for k, v in mb[0].state_dict().items()},
                            {k: v.detach().cpu() for k, v in mb[1].state_dict().items()})
        b = render_rays(fresh, embeddings(), rays, 64, False, 0, 0, 64, 32768, True)
    assert torch.equal(a["rgb_fine"], b["rgb_fine"])
    body = slice(256, None)
    assert torch.equal(img[body], fresh[1].packed_weights("f16x3")[body])


def test_fused_adam_trains_and_skips_missing_grads():
    from sinnerf_b200.optim import FusedAdam
    from sinnerf_b200.rendering import render_rays, RayLosses
    rays, trgb, tdep = _loss_case(64)
    models = make_models(orc.default_init_params(0), orc.default_init_params(1))
    opt = FusedAdam(models, lr=1e-3)
    losses = []
    for _ in range(8):
        opt.zero_grad(set_to_none=True)
        out = render_rays(models, embeddings(), rays.to(DEV), 32, False, 0, 0, 32, 32768, True,
                          losses=RayLosses(target_rgb=trgb))
        out["loss_rgb"].backward()
        opt.step()
        losses.append(float(out["loss_rgb"]))
    assert losses[-1] < losses[0], losses
    # a tensor without gradient is left alone (torch.optim.Adam skips it too)
    w = models[0].sigma.weight
    before = w.detach().clone()
    w.grad = None
    opt.step()
    assert torch.equal(before, w.detach())
    sd = opt.state_dict()
    opt.load_state_dict(sd)
    opt.step()


# ------------------------------------------------------------------------------------------ per-device state
def test_second_device_in_one_process():
    """ADVICE r1 (medium): the dynamic-shared-memory opt-in and the SM count are per device."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs in one process")
    from sinnerf_b200.rendering import render_rays
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    rays = torch.from_numpy(load_npz("render_lego_seed0_64p64_wb.npz")["rays"].copy())[:64]
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        models = make_models(pc, pf, dev)
        o = render_rays(models, embeddings(), rays.to(dev), 64, False, 0, 0, 64, 32768, True)
        (o["rgb_fine"].sum() + o["rgb_coarse"].sum()).backward()
        torch.cuda.synchronize(dev)
        outs.append((o["rgb_fine"].detach().cpu(), models[1].xyz_encoding_2[0].weight.grad.cpu()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert rel_l2(outs[1][1], outs[0][1]) <= 1e-5


# ------------------------------------------------------------------------------------------ pixel scatter (multi-GPU epilogue)
@pytest.mark.parametrize("n_importance", [64, 0])
def test_pixel_scatter_rows_equal_outputs(n_importance):
    """render_rays(pixel_scatter=...): the last pass's compositing kernel also stores [r, g, b, depth] rows into the given
    frame buffers at (row offset + ray) -- here two local buffers stand in for peer GPUs' memory (the 2-GPU run of
    tools/p2p_check.py covers NVLink / multicast addresses).  Rows outside the slab stay untouched; the regular outputs
    are bit-identical to a call without the scatter."""
    from sinnerf_b200.rendering import render_rays
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    models = make_models(pc, pf)
    n, off = 333, 57          # odd count: ragged last warp pass of the four-samples-per-thread kernel
    case = load_npz("render_llff_room_64p64_train.npz")
    base = torch.from_numpy(case["rays"].copy())
    rays = base[torch.arange(n) % base.shape[0]].clone().to(DEV)
    bufs = [torch.full((n + 100, 4), -7.0, device=DEV) for _ in range(2)]
    with torch.no_grad():
        ref = render_rays(models, embeddings(), rays, 64, False, 0, 0, n_importance, 32768, True)
        out = render_rays(models, embeddings(), rays, 64, False, 0, 0, n_importance, 32768, True,
                          pixel_scatter=([b.data_ptr() for b in bufs], off))
    torch.cuda.synchronize()
    for k in ("rgb_coarse", "depth_coarse", "rgb_fine", "depth_fine", "opacity_fine"):
        assert torch.equal(out[k], ref[k]), k
    want = torch.cat([out["rgb_fine"], out["depth_fine"][:, None]], dim=1)
    for b in bufs:
        assert torch.equal(b[off:off + n], want)
        assert bool((b[:off] == -7.0).all()) and bool((b[off + n:] == -7.0).all())
    with pytest.raises(ValueError):
        render_rays(models, embeddings(), rays, 64, False, 0, 0, n_importance, 32768, True, pixel_scatter=([], 0))


# ------------------------------------------------------------------------------------------ 16-bit training storage
@pytest.mark.parametrize("weights,n_rays,train_noise", [("seed", 256, False), ("room", 256, True), ("seed", 1500, True)])
def test_fp16_training_storage_matches_fp32_storage_and_oracle(weights, n_rays, train_noise):
    """The training path's default keeps ONE fp16 copy of the activations (T32 tiles) and passes power-of-two-scaled fp16
    gradients between layers (csrc/act16.cuh).  Parameter gradients: vs the fp32-storage kernels of round 1 and vs
    autograd through the CPU oracle, <= 1e-3 rel-L2 per tensor (SURVEY 8c), with training noise and trained weights."""
    import sinnerf_b200
    from sinnerf_b200.rendering import render_rays
    case = load_npz("render_llff_room_64p64_train.npz")
    base = torch.from_numpy(case["rays"].copy())
    rays = base[torch.arange(n_rays) % base.shape[0]].clone()
    rays[:, :3] += torch.randn(n_rays, 3, generator=torch.Generator().manual_seed(1)) * 0.05
    if weights == "room":
        pc, pf = room_params("coarse"), room_params("fine")
    else:
        pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    perturb, noise_std = (1.0, 1.0) if train_noise else (0.0, 0.0)
    g = torch.Generator().manual_seed(2)
    rng = {"perturb_u": torch.rand(n_rays, 64, generator=g), "noise_coarse": torch.randn(n_rays, 64, generator=g),
           "pdf_u": torch.rand(n_rays, 64, generator=g), "noise_fine": torch.randn(n_rays, 128, generator=g)}
    proj = None
    grads = {}
    before = sinnerf_b200.get_train_storage()
    try:
        for storage in ("fp16", "fp32"):
            sinnerf_b200.set_train_storage(storage)
            models = make_models(pc, pf)
            out = render_rays(models, embeddings(), rays.to(DEV), 64, False, perturb, noise_std, 64, 32768, False,
                              _rng={k: v.to(DEV) for k, v in rng.items()}, _return_intermediates=True)
            if proj is None:
                gp = torch.Generator().manual_seed(5)
                proj = {k: torch.randn(v.shape, generator=gp).to(DEV) for k, v in out.items() if not k.startswith("_")}
                z_f = out["_inter"]["z_fine"].detach().cpu()
            loss = sum((out[k] * proj[k]).sum() for k in proj)
            loss.backward()
            grads[storage] = [{k: p.grad.detach().cpu() for k, p in m.named_parameters()} for m in models]
    finally:
        sinnerf_b200.set_train_storage(before)
    worst, worst_k = 0.0, ""
    for a, b in zip(grads["fp16"], grads["fp32"]):
        for k in a:
            if float(b[k].norm()) == 0.0:
                assert float(a[k].norm()) == 0.0, k
                continue
            if rel_l2(a[k], b[k]) > worst:
                worst, worst_k = rel_l2(a[k], b[k]), k
            assert rel_l2(a[k], b[k]) <= 1e-3, (k, rel_l2(a[k], b[k]))
    print(f"fp16 vs fp32 training storage ({weights}, {n_rays} rays, noise={train_noise}): worst rel-L2 {worst:.2e} ({worst_k})", file=sys.stderr)
    if True:      # also at 1 500 rays (288 000 points, several tiles per CTA): ~10 s of CPU autograd
        oc = {k: v.clone().requires_grad_(True) for k, v in pc.items()}
        of = {k: v.clone().requires_grad_(True) for k, v in pf.items()}
        ref = orc.render_rays(oc, of, rays, N_samples=64, N_importance=64, perturb=perturb, noise_std=noise_std, rng=rng,
                              z_fine_override=z_f)
        sum((ref[k] * proj[k].cpu()).sum() for k in proj).backward()
        worst_o = worst_o32 = 0.0
        table = []
        for which, got, got32, refp in zip(("coarse", "fine"), grads["fp16"], grads["fp32"], (oc, of)):
            for k, v in refp.items():
                if float(v.grad.norm()) == 0.0:
                    continue
                table.append((rel_l2(got[k], v.grad), rel_l2(got32[k], v.grad), f"{which}.{k}"))
        for e16, e32, k in sorted(table, reverse=True)[:6]:
            print(f"  vs oracle autograd: {k:40s} fp16 storage {e16:.2e}   fp32 storage {e32:.2e}", file=sys.stderr)
        for got, got32, refp in zip(grads["fp16"], grads["fp32"], (oc, of)):
            for k, v in refp.items():
                if float(v.grad.norm()) == 0.0:
                    continue
                e16, e32 = rel_l2(got[k], v.grad), rel_l2(got32[k], v.grad)
                worst_o, worst_o32 = max(worst_o, e16), max(worst_o32, e32)
                # Trained weights: the 1e-3 bar of SURVEY 8c against the oracle.  Default-init weights leave ReLU
                # pre-activations within rounding of zero that flip between ANY two implementations (all-fp32 ones too:
                # the smoke test's note) -- at 1 500 rays the first layer's gradient of the
                # fp32-STORAGE kernels already differs from the oracle's by ~1.4e-3 with or without training noise
                # (measured on HEAD 5fa9a95 and on this build alike), so there the 16-bit path is held to the
                # fp32-storage kernels (1e-3, above) and, against the oracle, to no more than 1.25x their deviation.
                tol_o = 1e-3 if weights == "room" else max(1e-3, 1.25 * e32)
                assert e16 <= tol_o, (k, e16, e32)
        print(f"fp32 training storage vs oracle autograd: worst rel-L2 {worst_o32:.2e}", file=sys.stderr)
        print(f"fp16 training storage vs oracle autograd: worst rel-L2 {worst_o:.2e}", file=sys.stderr)


# ------------------------------------------------------------------------------------------ bf16 mode vs its own oracle
@pytest.mark.parametrize("weights", ["seed", "room"])
def test_bf16_mode_forward_and_gradients_vs_bf16_oracle(weights):
    """BASELINE configs[2]'s arithmetic (MLP operands in bf16, fp32 accumulate, everything else fp32) against the oracle
    restating exactly that: nn.Linear operands rounded to bf16 (straight-through in the backward), bottleneck folded
    into the direction layer as the kernels do, heads / encodings / compositing fp32.  Forward <= 5e-3 on rgb / depth
    (different fp32 summation order + bf16 rounding ties), parameter gradients <= 2e-2 rel-L2 per tensor (the backward
    here uses the fp16 copy of the fp32 activations and un-rounded weights; the oracle's straight-through gradients use
    the bf16-rounded operands -- a 2^-9 relative difference per element) -- instead of round 1's 'finite and within 5x'."""
    from sinnerf_b200.rendering import render_rays
    case = load_npz("render_llff_room_64p64_train.npz")
    rays = torch.from_numpy(case["rays"].copy())[:64]
    if weights == "room":
        pc, pf = room_params("coarse"), room_params("fine")
    else:
        pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    models = make_models(pc, pf)
    out = render_rays(models, embeddings(), rays.to(DEV), 64, False, 0, 0, 64, 32768, False, precision="bf16",
                      _return_intermediates=True)
    z_f = out["_inter"]["z_fine"].detach().cpu()
    oc = {k: v.clone().requires_grad_(True) for k, v in pc.items()}
    of = {k: v.clone().requires_grad_(True) for k, v in pf.items()}
    ref = orc.render_rays(oc, of, rays, N_samples=64, N_importance=64, perturb=0, noise_std=0, z_fine_override=z_f,
                          linear_dtype=torch.bfloat16, fold_bottleneck=True)
    for k in ("rgb_coarse", "depth_coarse", "rgb_fine", "depth_fine"):
        assert rel_l2(out[k].detach().cpu(), ref[k].detach()) <= 5e-3, (k, rel_l2(out[k].detach().cpu(), ref[k].detach()))
    gp = torch.Generator().manual_seed(3)
    proj = {k: torch.randn(v.shape, generator=gp) for k, v in ref.items() if not k.startswith("_")}
    sum((ref[k] * proj[k]).sum() for k in proj).backward()
    sum((out[k] * proj[k].to(DEV)).sum() for k in proj).backward()
    worst = 0.0
    for refp, model in ((oc, models[0]), (of, models[1])):
        sd = dict(model.named_parameters())
        for k, v in refp.items():
            if float(v.grad.norm()) == 0.0:
                continue
            e = rel_l2(sd[k].grad.cpu(), v.grad)
            worst = max(worst, e)
            assert e <= 2e-2, (k, e)
    print(f"bf16 mode vs bf16 oracle ({weights}): worst gradient rel-L2 {worst:.2e}", file=sys.stderr)
