"""GPU tests of the fused optimisers over the discriminator (`get_optimizer(hparams, [D], rate=0.2)`, C ABI
snb_optim_step_tensors): Adam against torch.optim.Adam's single-tensor path, SGD against torch's foreach SGD, RAdam /
Ranger against the oracle (oracle/optim_oracle.py), stepped on the same GPU with the same gradients, which come from
real discriminator backwards -- a generator-step call, then a hinge discriminator-step pair -- at imsize 64 and -1.
Also: state dicts moving between the fused and the replaced optimisers mid-run, GradScaler, repeatability, and the
INTEGRATION example's configure_optimizers."""
import copy
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests._common import rel_l2
from tests.test_disc_optim_cpu import HParams, oracle_get_optimizer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STEPS = 14          # RAdam turns adaptive at step 6; Ranger syncs at steps 6 and 12
SKIP = 1            # tensor without a gradient on steps 0 and 7 (first: its state starts one step late)
RULES = ["sgd", "adam", "radam", "ranger"]
SHAPES = {64: (64, 64), -1: (63, 84)}   # the blender and the LLFF / DTU patch


def make_d(imsize, seed=0):
    from sinnerf_b200.discriminator import Discriminator
    torch.manual_seed(seed)
    return Discriminator(False, "color,cutout", imsize=imsize).to(DEV)


def copy_d(d):
    c = copy.deepcopy(d)
    for p in c.parameters():
        p.grad = None
    return c


def reference_for(rule, d, wd):
    """The optimiser the reference's get_optimizer builds over d.parameters(), in the form the fused one is held to:
    torch's single-tensor Adam, torch's (default, foreach) SGD on CUDA, the oracle's RAdam / Ranger."""
    if rule == "sgd":
        return torch.optim.SGD(list(d.parameters()), lr=HParams.lr * 0.2, momentum=HParams.momentum, weight_decay=wd,
                               foreach=True)
    return oracle_get_optimizer(HParams(rule, wd), [d], rate=0.2)


def fused_for(rule, d, wd):
    from sinnerf_b200.optim import get_optimizer
    return get_optimizer(HParams(rule, wd), [d], rate=0.2)


def d_step_grads(d, step, scaler=None):
    """The adversarial sequence of one training step on d: a generator-step call (-mean, gradient to the input only),
    then the discriminator-step pair with one hinge backward into the weight_orig gradients (scaled by `scaler`)."""
    H, W = SHAPES[d.imsize]
    g = torch.Generator().manual_seed(1000 + step)
    fake, real = (torch.rand(2, 3, H, W, generator=g).to(DEV) for _ in range(2))
    np.random.seed(step)
    torch.cuda.manual_seed(step)
    xf = fake.clone().requires_grad_(True)
    torch.autograd.grad(-d(xf).mean(), xf)
    d.zero_grad(set_to_none=True)
    loss = F.relu(1 - d(real)).mean() + F.relu(1 + d(fake)).mean()
    (loss if scaler is None else scaler.scale(loss)).backward()


def copy_grads(src, dst, without=()):
    for i, (ps, pd) in enumerate(zip(src.parameters(), dst.parameters())):
        if i in without:
            ps.grad = None
        pd.grad = None if ps.grad is None else ps.grad.clone()


def compare(ref, da, opt, db, what):
    """Parameters and state tensors bit for bit (max |diff| / max |ref| per tensor is reported too); step counts and
    state keys exactly."""
    worst, exact, total = 0.0, 0, 0
    for i, (pa, pb) in enumerate(zip(da.parameters(), db.parameters())):
        worst = max(worst, (pa.detach() - pb.detach()).abs().max().item() / pa.detach().abs().max().item())
        exact += int((pa.detach() == pb.detach()).sum())
        total += pa.numel()
        st_a, st_b = ref.state.get(pa, {}), opt.state.get(pb, {})
        assert set(st_a) == set(st_b), (what, i, set(st_a), set(st_b))
        for k, v in st_a.items():
            if k == "step":
                assert float(st_b[k]) == float(v) and type(st_b[k]) is type(v), (what, i, st_b[k], v)
            else:
                assert torch.equal(st_b[k], v), (what, i, k, rel_l2(st_b[k].cpu(), v.cpu()))
    print(f"{what}: {exact}/{total} parameters bit-equal ({exact / total:.4f}), worst rel diff {worst:.2e}",
          file=sys.stderr)
    assert worst <= 3e-7, what
    assert exact == total, what           # the replaced optimiser's ATen ops, rounded alike: bit for bit


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("imsize", [64, -1])
@pytest.mark.parametrize("rule", RULES)
def test_fused_matches_reference(rule, imsize, weight_decay):
    """14 steps of the fused rule and of the rule it replaces on the same gradients; an lr change after step 7; one
    tensor without a gradient on steps 0 and 7 stays put and its count lags."""
    from sinnerf_b200.optim import FusedAdam, FusedRAdam, FusedRanger, FusedSGD
    db = make_d(imsize)
    da = copy_d(db)
    ref = reference_for(rule, da, weight_decay)
    opt = fused_for(rule, db, weight_decay)
    assert type(opt) is dict(sgd=FusedSGD, adam=FusedAdam, radam=FusedRAdam, ranger=FusedRanger)[rule]
    skipped = list(db.parameters())[SKIP]
    for step in range(STEPS):
        if step == 7:
            for o in (ref, opt):
                o.param_groups[0]["lr"] *= 0.5
        d_step_grads(db, step)
        copy_grads(db, da, without=(SKIP,) if step in (0, 7) else ())
        if step in (0, 7):
            skipped.grad = None
            before = skipped.detach().clone()
        ref.step()
        opt.step()
        if step in (0, 7):
            assert torch.equal(before, skipped.detach()), step
            if rule != "sgd":
                assert int(opt.state.get(skipped, {}).get("step", 0)) == (0 if step == 0 else 6)
    compare(ref, da, opt, db, f"{rule} imsize={imsize} wd={weight_decay}")
    if rule != "sgd":
        assert int(opt.state[skipped]["step"]) == STEPS - 2


def fixed_grads(imsize):
    """STEPS gradient sets from real discriminator backwards (one D, not stepped), so that separate runs see the same
    gradients; tensor 2 has none before step 7 (no state in a state dict saved at step 7), tensor SKIP none at 0 and 7."""
    d = make_d(imsize, seed=3)
    out = []
    for step in range(STEPS):
        d_step_grads(d, step)
        gs = [p.grad.clone() for p in d.parameters()]
        gs[SKIP] = None if step in (0, 7) else gs[SKIP]
        gs[2] = None if step < 7 else gs[2]
        out.append(gs)
    return out


def run(opt, d, grads, steps):
    for step in steps:
        for p, g in zip(d.parameters(), grads[step]):
            p.grad = None if g is None else g.clone()
        opt.step()


@pytest.mark.parametrize("rule", RULES)
def test_state_dict_round_trip(rule):
    """Resuming mid-run equals an uninterrupted run: fused for 7 steps, its state dict into a fresh fused optimiser
    (bit for bit), and through the replaced optimiser -- fused state dict into it for steps 7-9, its state dict back
    into a fused one for 10-13 -- to the comparison bars.  The state dict saved at step 7 has no entry for a tensor
    that had no gradient yet, like the reference's."""
    imsize, wd = -1, 1e-2
    grads = fixed_grads(imsize)
    d0 = make_d(imsize)
    du = copy_d(d0)
    uninterrupted = fused_for(rule, du, wd)
    run(uninterrupted, du, grads, range(STEPS))

    d1 = copy_d(d0)
    first = fused_for(rule, d1, wd)
    run(first, d1, grads, range(7))
    saved = copy.deepcopy(first.state_dict())
    assert sorted(saved["state"]) == [0, 1]
    # fused -> fused
    d2 = copy_d(d1)
    resumed = fused_for(rule, d2, 0.0)
    resumed.load_state_dict(copy.deepcopy(saved))
    assert resumed.param_groups[0]["weight_decay"] == wd
    run(resumed, d2, grads, range(7, STEPS))
    for pa, pb in zip(du.parameters(), d2.parameters()):
        assert torch.equal(pa, pb)
        for k, v in uninterrupted.state[pa].items():
            assert torch.equal(torch.as_tensor(resumed.state[pb][k]), torch.as_tensor(v)), k
    # fused -> replaced -> fused
    d3 = copy_d(d1)
    ref = reference_for(rule, d3, 0.0)
    ref.load_state_dict(copy.deepcopy(saved))
    if rule == "adam":
        ref.param_groups[0]["foreach"] = False      # the loaded group has no such key; keep the single-tensor path
    assert list(d3.parameters())[2] not in ref.state
    run(ref, d3, grads, range(7, 10))
    d4 = copy_d(d3)
    back = fused_for(rule, d4, 0.0)
    back.load_state_dict(copy.deepcopy(ref.state_dict()))
    run(back, d4, grads, range(10, STEPS))
    compare(uninterrupted, du, back, d4, f"{rule}: fused -> replaced -> fused")


@pytest.mark.parametrize("rule", RULES)
def test_grad_scaler_step_equals_unscaled_step(rule):
    """scaler.step(opt_d) under a power-of-two scale takes the step the unscaled gradients give, bit for bit."""
    da = make_d(64)
    db = copy_d(da)
    opt_a, opt_b = fused_for(rule, da, 1e-2), fused_for(rule, db, 1e-2)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
    for step in range(3):
        d_step_grads(db, step, scaler)
        for pa, pb in zip(da.parameters(), db.parameters()):
            pa.grad = pb.grad * 2.0 ** -12
        opt_a.step()
        scaler.step(opt_b)
        scaler.update()
        assert scaler.get_scale() == 2.0 ** 12
        for pa, pb in zip(da.parameters(), db.parameters()):
            assert torch.equal(pa, pb), (rule, step)


def test_repeatable():
    """Two identical runs of each rule give identical bits."""
    grads = fixed_grads(64)
    for rule in RULES:
        out = []
        for _ in range(2):
            d = make_d(64)
            opt = fused_for(rule, d, 1e-2)
            run(opt, d, grads, range(8))
            out.append([p.detach().clone() for p in d.parameters()] +
                       [v.clone() for st in opt.state.values() for v in st.values() if torch.is_tensor(v)])
        assert all(torch.equal(a, b) for a, b in zip(*out)), rule


def test_refuses_bad_parameters():
    from sinnerf_b200.optim import FusedAdam
    d = make_d(-1)
    opt = FusedAdam([d])
    for p in d.parameters():
        p.grad = torch.zeros_like(p)
    w = d.convs()[1].weight_orig
    w.grad = torch.zeros(w.shape[::-1], device=DEV).permute(3, 2, 1, 0)    # a non-contiguous gradient
    with pytest.raises(ValueError):
        opt.step()
    with pytest.raises(RuntimeError):
        FusedAdam([make_d(-1).cpu()]).step()


class _System:
    """The parts of models/sinnerf.py's SinNeRF that configure_optimizers reads."""

    def __init__(self, hparams):
        from sinnerf_b200.discriminator import Discriminator
        from sinnerf_b200.nerf import NeRF
        self.hparams = hparams
        self.models = [NeRF(use_new_activation=True).to(DEV), NeRF(use_new_activation=True).to(DEV)]
        torch.manual_seed(0)
        self.D = Discriminator(False, "color,cutout", imsize=64).to(DEV)

    def configure_optimizers(self):
        # INTEGRATION.md: models/sinnerf.py's configure_optimizers with `from sinnerf_b200.optim import get_optimizer`
        from sinnerf_b200.optim import get_optimizer
        from torch.optim.lr_scheduler import MultiStepLR
        self.optimizer = get_optimizer(self.hparams, self.models)

        scheduler = MultiStepLR(self.optimizer, milestones=[2], gamma=0.5)
        li = [self.optimizer]
        if self.hparams.dis_weight > 0:
            self.opt_d = get_optimizer(self.hparams, [self.D], rate=0.2)
            li.append(self.opt_d)
        return li, [scheduler]


@pytest.mark.parametrize("rule", RULES)
def test_integration_configure_optimizers(rule):
    """Both optimisers of configure_optimizers come from the one import and step fused: the NeRF one after a
    render_rays backward, opt_d after a discriminator step."""
    from sinnerf_b200 import synthetic
    from sinnerf_b200.nerf import Embedding
    from sinnerf_b200.rendering import render_rays
    hp = HParams(rule)
    hp.dis_weight = 0.01
    system = _System(hp)
    (opt, opt_d), _ = system.configure_optimizers()
    fused = dict(sgd="FusedSGD", adam="FusedAdam", radam="FusedRAdam", ranger="FusedRanger")[rule]
    assert type(opt).__name__ == fused and type(opt_d).__name__ == fused
    assert opt_d.param_groups[0]["lr"] == pytest.approx(0.2 * hp.lr)
    nerf_before = [p.detach().clone() for m in system.models for p in m.parameters()]
    d_before = [p.detach().clone() for p in system.D.parameters()]
    rays = synthetic.random_rays("lego", 64, seed=5).to(DEV)
    out = render_rays(system.models, [Embedding(3, 10), Embedding(3, 4)], rays, 32, False, 0, 0, 32, 32768, True)
    (out["rgb_fine"] ** 2).mean().backward()
    opt.step()
    d_step_grads(system.D, 0)
    opt_d.step()
    assert any(not torch.equal(a, p) for a, p in zip(nerf_before, (p for m in system.models for p in m.parameters())))
    assert all(not torch.equal(a, p) for a, p in zip(d_before, system.D.parameters()))
