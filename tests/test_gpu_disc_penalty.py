"""GPU tests of Discriminator.forward_with_penalty (csrc/disc.cu, snb_disc_penalty_*): the wgan_gp gradient penalty
compute_grad2(D(x), x) and its second-order gradients against the float64 oracle (tests/disc_oracle.py) under
torch.autograd.grad(create_graph=True), given the same random draws; equality with D(x) and its plain backward;
determinism, the absence of host synchronisation, the autocast policy and the input checks."""
import numpy as np
import pytest
import torch

from sinnerf_b200.discriminator import Discriminator, draw_augment, layer_schedule
from tests import disc_oracle as do
from tests._common import rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
POLICY = "color,cutout"
BRANCHES = [(64, 64, 64), (-1, 63, 84), (-1, 56, 70), (32, 32, 32), (128, 128, 128)]
# rel-L2 bars against float64 for (reg, its input gradient and each weight gradient), measured on an H100 80GB HBM3 at
# 700 W (README "Discriminator on the GPU").  Split mode: reg <= 5.2e-5, gradients <= 4.3e-5 where no LeakyReLU input
# took the other branch.  The single-product bars are twice the largest measured values (f16 7.3e-4 / 2.7e-2, bf16
# 3.4e-3 / 9.3e-2).
BARS = {"f16x3": (1e-4, 1e-4), "f16": (1.5e-3, 5.4e-2), "bf16": (7e-3, 1.9e-1)}
# LeakyReLU inputs within KINK of zero may take the other branch in the kernels' arithmetic (test_gpu_discriminator.py).
# reg = |g|^2 depends on the branch as well as its gradients do, so when either misses its bar the oracle's inputs are
# flipped greedily, and both must then come within twice their bars with at most MAX_FLIPS flips
KINK, MAX_FLIPS = 5e-5, 6


def _gate_seed(fire):
    for s in range(1000):
        np.random.seed(s)
        a, b = np.random.random(), np.random.random()
        if (a > 0.5 and b >= 0.5) == fire:
            return s
    raise AssertionError


def make(imsize, precision="f16x3", seed=0):
    np.random.seed(seed)
    torch.manual_seed(seed)
    return Discriminator(False, POLICY, imsize=imsize, precision=precision).to(DEV)


def snapshot(D):
    convs = D.convs()
    return ([m.weight_orig.detach().double().cpu().clone() for m in convs],
            [m.weight_u.double().cpu().clone() for m in convs], [m.weight_v.double().cpu().clone() for m in convs])


def as_layout(x, layout):
    B, _, H, W = x.shape
    if layout == "nchw":
        leaf = x.clone().requires_grad_(True)
        return leaf, leaf
    leaf = x.permute(0, 2, 3, 1).reshape(B * H * W, 3).contiguous().requires_grad_(True)
    return leaf, leaf.view(B, H, W, 3).permute(0, 3, 1, 2)


def grad_nchw(leaf, x_shape, layout):
    B, _, H, W = x_shape
    return leaf.grad if layout == "nchw" else leaf.grad.view(B, H, W, 3).permute(0, 3, 1, 2)


def call(D, x, np_seed, torch_seed, penalty=True):
    np.random.seed(np_seed)
    torch.cuda.manual_seed(torch_seed)
    return D.forward_with_penalty(x) if penalty else D(x)


def replay(x_shape, np_seed, torch_seed):
    np.random.seed(np_seed)
    torch.cuda.manual_seed(torch_seed)
    return draw_augment(POLICY, tuple(x_shape), DEV)


def oracle_penalty(ws, us, vs, x, imsize, training, aug, c, gout, flips=None, near_kink=None):
    """float64 compute_grad2 and the gradients of <gout, out> + <c, reg> (double backward through autograd)"""
    w2 = [w.clone().requires_grad_(True) for w in ws]
    xo = x.double().clone().requires_grad_(True)
    out, *_ = do.forward(w2, us, vs, xo, imsize, training, aug, near_kink, flips)
    (g,) = torch.autograd.grad(out.sum(), xo, create_graph=True)
    reg = g.pow(2).flatten(1).sum(1)
    ((out * gout.double()).sum() + (reg * c.double()).sum()).backward()
    return reg.detach(), xo.grad, [w.grad for w in w2]


def scaled_error(got_reg, got, want, bars):
    """the largest error of reg and of the gradients, each over its bar"""
    reg_o, dx_o, dw_o = want
    return max(rel_l2(got_reg, reg_o) / bars[0],
               max(rel_l2(a, b) for a, b in zip(got, [dx_o] + dw_o) if a is not None) / bars[1])


def explain_kinks(got_reg, got, args, cands, bars):
    """-> the scaled error left after greedy LeakyReLU flips of near-kink oracle inputs: reg = |g|^2 and its
    gradients change with the slope an input takes, so a flip can explain either"""
    def err(flips):
        return scaled_error(got_reg, got, oracle_penalty(*args, flips=flips), bars)
    flips, chosen = {}, 0
    best = err(flips)
    for layer, j, _, numel in sorted(cands, key=lambda c: c[2])[:64]:
        if best <= 1 or chosen == MAX_FLIPS:
            break
        trial = {k: v.clone() for k, v in flips.items()}
        trial.setdefault(layer, torch.zeros(numel, dtype=torch.bool))[j] = True
        e = err(trial)
        if e < best:
            best, flips, chosen = e, trial, chosen + 1
    return best


def check_case(imsize, H, W, B, layout, fire, precision, training=True, out_term=True, trained=None, input_grad=True):
    """reg and the gradients of <gout, out> + <c, reg> (out_term False: <c, reg> alone, as in wgan_gp_reg) to the input
    (input_grad) and to the weight_origs of the layers in trained (None: all; the others frozen) against the oracle"""
    D = make(imsize, precision, seed=1 + B)
    D.train(training)
    ws, us, vs = snapshot(D)
    convs = D.convs()
    trained = range(len(convs)) if trained is None else trained
    for i, m in enumerate(convs):
        m.weight_orig.requires_grad_(i in trained)
    g = torch.Generator().manual_seed(13 * B + H)
    x = torch.rand(B, 3, H, W, generator=g)
    c = torch.rand(B, generator=g) + 0.5
    leaf, view = as_layout(x.to(DEV), layout)
    if not input_grad:
        leaf.requires_grad_(False)
    s = _gate_seed(fire)
    out, reg = call(D, view, s, 7)
    gout = torch.randn(out.shape, generator=g) * 1e-2 if out_term else torch.zeros(out.shape)
    loss = (reg * c.to(DEV)).sum()
    if out_term:
        loss = loss + (out * gout.to(DEV)).sum()
    loss.backward()
    aug = replay(x.shape, s, 7)
    assert (aug is not None) == fire
    args = (ws, us, vs, x, imsize, training, aug, c, gout)
    cands = []
    want = oracle_penalty(*args, near_kink=(KINK, cands))
    got_reg = reg.detach().cpu().double()
    got = [grad_nchw(leaf, x.shape, layout).cpu().double() if input_grad else None]
    for i, m in enumerate(convs):
        assert (m.weight_orig.grad is not None) == (i in trained)
        got.append(m.weight_orig.grad.cpu().double() if i in trained else None)
    bars = BARS[precision]
    errs = {"reg": rel_l2(got_reg, want[0])}
    if input_grad:
        errs["dx"] = rel_l2(got[0], want[1])
    errs["dw"] = max(rel_l2(a, b) for a, b in zip(got[1:], want[2]) if a is not None)
    scaled = scaled_error(got_reg, got, want, bars)
    if scaled > 1:
        errs["scaled_flipped"] = explain_kinks(got_reg, got, args, cands, bars)
    print(f"penalty[{precision} imsize={imsize} {H}x{W} B={B} {layout} aug={fire} train={training} out={out_term} "
          f"trained={list(trained)} dx={input_grad}] " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()) +
          f" near_kink={len(cands)}")
    assert scaled <= 1 or errs["scaled_flipped"] <= 2, errs


@pytest.mark.parametrize("fire", [True, False])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("imsize,H,W", BRANCHES)
def test_penalty_split(imsize, H, W, B, fire):
    check_case(imsize, H, W, B, "rays" if fire else "nchw", fire, "f16x3")


@pytest.mark.parametrize("imsize,H,W", BRANCHES[:2])
def test_penalty_split_eval(imsize, H, W):
    check_case(imsize, H, W, 2, "nchw", True, "f16x3", training=False)


@pytest.mark.parametrize("fire", [True, False])
@pytest.mark.parametrize("imsize,H,W", BRANCHES[:3])
def test_penalty_reg_only(imsize, H, W, fire):
    """wgan_gp_reg's loss leaves out unused: the first-order part is absent and the penalty's gradients are written"""
    check_case(imsize, H, W, 2, "rays", fire, "f16x3", out_term=False)


@pytest.mark.parametrize("out_term", [True, False])
@pytest.mark.parametrize("trained", ["last", "first"])
@pytest.mark.parametrize("imsize,H,W", BRANCHES[:2])
def test_penalty_frozen_layers(imsize, H, W, trained, out_term):
    """the input does not require grad and only one weight_orig does, the last (where no input gradient of any layer is
    needed) or the first"""
    L = len(layer_schedule(imsize))
    check_case(imsize, H, W, 1, "nchw", True, "f16x3", out_term=out_term,
               trained=[L - 1] if trained == "last" else [0], input_grad=False)


@pytest.mark.parametrize("fire", [True, False])
@pytest.mark.parametrize("imsize,H,W", BRANCHES[:2])
@pytest.mark.parametrize("precision", ["f16", "bf16"])
def test_penalty_single_product(precision, imsize, H, W, fire):
    check_case(imsize, H, W, 2, "rays", fire, precision)


@pytest.mark.parametrize("fire", [True, False])
@pytest.mark.parametrize("imsize,H,W", BRANCHES[:2])
def test_matches_plain_call(imsize, H, W, fire):
    """out, u, v and the generators' state equal D(x)'s; with the penalty unused the gradients equal the plain
    backward's, bit for bit"""
    x = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(5)).to(DEV)
    s = _gate_seed(fire)
    res = []
    for penalty, reg_term in ((False, False), (True, False), (True, True)):
        D = make(imsize, seed=6)
        xl = x.clone().requires_grad_(True)
        r = call(D, xl, s, 3, penalty)
        out = r[0] if penalty else r
        after = [torch.tensor(np.random.random()), torch.rand(3, device=DEV)]
        gout = torch.linspace(-1, 1, out.numel(), device=DEV).view(out.shape)
        loss = (out * gout).sum()
        if reg_term:   # d_reg = 0: the second-order part adds exact zeros
            loss = loss + (r[1] * 0).sum()
        loss.backward()
        state = [t for m in D.convs() for t in (m.weight_u, m.weight_v, m.weight_orig.grad)]
        res.append([out.detach(), xl.grad] + state + after)
    for other in res[1:]:
        for a, b in zip(res[0], other):
            assert torch.equal(a, b)


def test_deterministic():
    outs = []
    for _ in range(2):
        D = make(-1, seed=3)
        x = torch.rand(2, 3, 63, 84, generator=torch.Generator().manual_seed(0)).to(DEV).requires_grad_(True)
        out, reg = call(D, x, _gate_seed(True), 4)
        (out.sum() + 10 * reg.mean()).backward()
        outs.append([out, reg, x.grad] + [t for m in D.convs() for t in (m.weight_orig.grad, m.weight_u, m.weight_v)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_no_host_sync():
    """the wgan_gp discriminator step: real call with its penalty, fake call, one backward"""
    D = make(64)
    real, fake = torch.rand(1, 3, 64, 64, device=DEV), torch.rand(1, 3, 64, 64, device=DEV)
    for sync_mode in (0, "error"):     # the first round loads the library
        np.random.seed(_gate_seed(True))
        torch.cuda.set_sync_debug_mode(sync_mode)
        try:
            pred_real, reg_real = D.forward_with_penalty(real)
            pred_fake = D(fake)
            # compute_loss(fake, 0) + compute_loss(real, 1) + 10 compute_grad2(real).mean()
            loss_d = -pred_fake.mean() + pred_real.mean() + 10 * reg_real.mean()
            loss_d.backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()


def test_autocast_policy_is_f16():
    x = torch.rand(1, 3, 64, 64, device=DEV)
    outs = []
    for precision, ac in (("f16", False), ("autocast", True)):
        D = make(64, precision, seed=4)
        with torch.autocast("cuda", dtype=torch.float16, enabled=ac):
            out, reg = call(D, x, _gate_seed(True), 2)
            reg.sum().backward()
        outs.append([out, reg] + [m.weight_orig.grad for m in D.convs()])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_input_checks():
    D = make(64)
    with pytest.raises(ValueError):
        D.forward_with_penalty(torch.rand(1, 4, 64, 64, device=DEV))
    with pytest.raises(TypeError):
        D.forward_with_penalty(torch.rand(1, 3, 64, 64, device=DEV, dtype=torch.float64))
    with pytest.raises(ValueError):
        D.forward_with_penalty(torch.rand(1, 3, 8, 8, device=DEV))
    with pytest.raises(RuntimeError):
        D.forward_with_penalty(torch.rand(1, 3, 64, 64))
