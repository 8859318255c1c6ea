"""GPU tests of FusedSGD / FusedRAdam / FusedRanger against the optimiser oracle (oracle/optim_oracle.py) stepped on the
same GPU with the same gradients, which come from a real render_rays backward."""
import copy
import sys

import numpy as np
import pytest
import torch

from oracle import optim_oracle
from oracle import render_oracle as orc
from tests._common import load_npz, rel_l2
from tests.test_optim_cpu import OPTIM_LR, make_optimizer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STEPS = 14          # RAdam turns adaptive at step 6; Ranger syncs at steps 6 and 12
SKIP = 3            # tensor without a gradient on steps 0 and 7 (first: its state starts one step late)


def make_models(pc, pf):
    from sinnerf_b200.nerf import NeRF
    models = []
    for p in (pc, pf):
        m = NeRF(use_new_activation=True)
        m.load_state_dict(p)
        models.append(m.to(DEV))
    return models


def embeddings():
    from sinnerf_b200.nerf import Embedding
    return [Embedding(3, 10), Embedding(3, 4)]


def fused_for(rule, models, wd):
    from sinnerf_b200.optim import FusedRAdam, FusedRanger, FusedSGD
    if rule == "sgd":
        return FusedSGD(models, lr=OPTIM_LR, momentum=0.9, weight_decay=wd)
    if rule == "radam":
        return FusedRAdam(models, lr=OPTIM_LR, eps=1e-8, weight_decay=wd)
    return FusedRanger(models, lr=OPTIM_LR, eps=1e-8, weight_decay=wd)


def params_of(models):
    return [p for m in models for p in m.parameters()]


_case = {}


def render_grads(models):
    """Gradients of an RGB loss through render_rays (64 rays, 32 + 32 samples) into the models' .grad."""
    from sinnerf_b200 import synthetic
    from sinnerf_b200.rendering import render_rays
    if not _case:
        g = torch.Generator().manual_seed(5)
        _case["rays"] = synthetic.random_rays("lego", 64, seed=5).to(DEV)
        _case["target"] = torch.rand(64, 3, generator=g).to(DEV)
    for m in models:
        m.zero_grad(set_to_none=True)
    out = render_rays(models, embeddings(), _case["rays"], 32, False, 0, 0, 32, 32768, True)
    t = _case["target"]
    (((out["rgb_coarse"] - t) ** 2).mean() + ((out["rgb_fine"] - t) ** 2).mean()).backward()


def copy_grads(src, dst, without=()):
    for i, (ps, pd) in enumerate(zip(params_of(src), params_of(dst))):
        if i in without:
            ps.grad = None
        pd.grad = None if ps.grad is None else ps.grad.clone()


def compare(ref, ref_models, opt, models, what):
    """Parameters and state tensors bit for bit (the FusedAdam bar, max |diff| <= 3e-7 max |ref| per tensor, is
    reported too), step counts and state keys exactly."""
    worst, exact, total = 0.0, 0, 0
    for i, (pa, pb) in enumerate(zip(params_of(ref_models), params_of(models))):
        d = (pa.detach() - pb.detach()).abs().max().item()
        worst = max(worst, d / pa.detach().abs().max().item())
        exact += int((pa.detach() == pb.detach()).sum())
        total += pa.numel()
        st_a, st_b = ref.state[pa], opt.state[pb]
        assert set(st_a) == set(st_b), (what, i, set(st_a), set(st_b))
        for k, v in st_a.items():
            if k == "step":
                assert st_b[k] == v, (what, i)
            else:
                assert torch.equal(st_b[k], v), (what, i, k, rel_l2(st_b[k].cpu(), v.cpu()))
    print(f"{what}: {exact}/{total} parameters bit-equal ({exact / total:.4f}), worst rel diff {worst:.2e}",
          file=sys.stderr)
    assert worst <= 3e-7, what
    assert exact == total, what           # SGD / RAdam / Ranger follow the oracle's ATen ops rounding for rounding


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("rule", ["sgd", "radam", "ranger"])
def test_fused_matches_oracle(rule, weight_decay):
    """14 steps of the fused rule and of the oracle on the same gradients; an lr change after step 7; one tensor
    without a gradient on steps 0 and 7 stays put and its count lags.  After the last step the packed image is the
    image of the final weights, stamped clean: a render right after step() packs nothing."""
    from sinnerf_b200.rendering import render_rays
    pc, pf = orc.default_init_params(0), orc.default_init_params(1)
    ma, mb = make_models(pc, pf), make_models(pc, pf)
    ref = make_optimizer(optim_oracle, params_of(ma), rule, weight_decay)
    opt = fused_for(rule, mb, weight_decay)
    skipped = params_of(mb)[SKIP]
    for step in range(STEPS):
        if step == 7:
            for o in (ref, opt):
                o.param_groups[0]["lr"] = 0.5 * OPTIM_LR
        render_grads(mb)
        copy_grads(mb, ma, without=(SKIP,) if step in (0, 7) else ())
        if step in (0, 7):
            skipped.grad = None
            before = skipped.detach().clone()
        ref.step()
        opt.step()
        if step in (0, 7):
            assert torch.equal(before, skipped.detach()), step
            if rule != "sgd":
                assert opt.state.get(skipped, {}).get("step", 0) == (0 if step == 0 else 6)
    compare(ref, ma, opt, mb, f"{rule} wd={weight_decay}")
    if rule != "sgd":
        assert opt.state[skipped]["step"] == STEPS - 2
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


@pytest.mark.parametrize("rule", ["sgd", "radam", "ranger"])
def test_state_dict_moves_between_oracle_and_fused(rule):
    """A state dict of the oracle after 7 steps (one tensor never stepped: no state, as in the reference) loads into
    the fused optimiser, and the two step on to 14 alike; the fused state dict loads back into the oracle, and one more
    step of each still agrees."""
    wd = 1e-2
    ma = make_models(orc.default_init_params(0), orc.default_init_params(1))
    ref = make_optimizer(optim_oracle, params_of(ma), rule, wd)
    never = 5
    for step in range(7):
        render_grads(ma)
        params_of(ma)[never].grad = None
        ref.step()
    assert params_of(ma)[never] not in ref.state
    mb = make_models(*[{k: v.detach().cpu() for k, v in m.state_dict().items()} for m in ma])
    opt = fused_for(rule, mb, 0.0)
    opt.load_state_dict(ref.state_dict())
    assert opt.param_groups[0]["weight_decay"] == wd
    assert params_of(mb)[never] not in opt.state
    for step in range(7, STEPS):
        render_grads(mb)
        copy_grads(mb, ma)
        ref.step()
        opt.step()
    compare(ref, ma, opt, mb, f"{rule} resumed from the oracle")
    # and back: the fused state dict into a fresh oracle on copies of the weights
    mc = make_models(*[{k: v.detach().cpu() for k, v in m.state_dict().items()} for m in mb])
    back = make_optimizer(optim_oracle, params_of(mc), rule, 0.0)
    back.load_state_dict(copy.deepcopy(opt.state_dict()))
    render_grads(mb)
    copy_grads(mb, mc)
    back.step()
    opt.step()
    compare(back, mc, opt, mb, f"{rule} resumed from the fused optimiser")
