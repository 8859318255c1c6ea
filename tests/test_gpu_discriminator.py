"""GPU tests of sinnerf_b200.discriminator (csrc/disc.cu): the spectral-norm patch discriminator with DiffAugment
against the float64 oracle (tests/disc_oracle.py) given the same random draws -- the drop-in is re-seeded and its
draws are replayed through draw_augment -- on all four branches at the recipe shapes, in NCHW and in the
'(b p q) c -> b c p q' view of a ray-major tensor; output, input gradient, every weight_orig gradient, u, v and sigma.
Also train / eval mode, the hinge generator / discriminator step sequence, the random generators' state after a call,
determinism, the absence of host synchronisation, the no-grad pass, the autocast policy and the refused double
backward."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sinnerf_b200.discriminator import Discriminator, draw_augment
from tests import disc_oracle as do
from tests._common import rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D64 = torch.float64
POLICY = "color,cutout"

BRANCHES = [(64, 64, 64), (-1, 63, 84), (-1, 56, 70), (32, 32, 32), (128, 128, 128)]
# rel-L2 bars against float64: (output, input gradient and each weight gradient, u / v / sigma), measured on an H100
# 80GB HBM3 at 700 W (README "Discriminator on the GPU").  Split mode: output <= 8e-5 except the 32 branch at B = 2,
# whose two 1 x 1 outputs cancel to ~1e-2 of their 8192 terms (1.3e-4); gradients <= 2.6e-5.  The single-product bars
# are twice the largest measured values (f16 7.0e-3 / 4.8e-2, bf16 1.4e-2 / 1.3e-1).
BARS = {"f16x3": (2e-4, 1e-4, 1e-5), "f16": (1.4e-2, 1e-1, 1e-5), "bf16": (3e-2, 2.6e-1, 1e-5)}
# A LeakyReLU input within ~1e-5 of zero may land on the other side of the kink in the kernel's arithmetic (its
# forward is ~3e-5 of float64, fp32 PyTorch's ~1e-6), which scales the gradient through that element by 5 or 1/5: one
# such element among 8192 costs ~1e-2 of rel-L2.  When the gradients miss their bar, the oracle's inputs within KINK of
# zero are flipped one at a time, in order of distance, and a flip is kept if it brings the gradients closer; the
# gradients must then come within twice the bar with at most MAX_FLIPS flips (single flips found greedily can leave
# the residual of a combination they miss: 1.5e-4 at most in the cases here, 1.1e-5 to 1.8e-5 in the others).
KINK, MAX_FLIPS = 5e-5, 6


def _gate_seed(fire):
    """first numpy seed whose two gate draws apply (fire) or skip the augmentation"""
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
    ws = [m.weight_orig.detach().double().cpu().clone().requires_grad_(True) for m in convs]
    return ws, [m.weight_u.double().cpu().clone() for m in convs], [m.weight_v.double().cpu().clone() for m in convs]


def as_layout(x, layout):
    """-> (leaf, view): x (B,3,H,W) as a contiguous leaf, or as the '(b p q) c -> b c p q' view of a ray-major leaf"""
    B, _, H, W = x.shape
    if layout == "nchw":
        leaf = x.clone().requires_grad_(True)
        return leaf, leaf
    leaf = x.permute(0, 2, 3, 1).reshape(B * H * W, 3).contiguous().requires_grad_(True)
    return leaf, leaf.view(B, H, W, 3).permute(0, 3, 1, 2)


def grad_nchw(leaf, x_shape, layout):
    B, _, H, W = x_shape
    g = leaf.grad
    return g if layout == "nchw" else g.view(B, H, W, 3).permute(0, 3, 1, 2)


def gpu_call(D, x_view, np_seed, torch_seed):
    np.random.seed(np_seed)
    torch.cuda.manual_seed(torch_seed)
    return D(x_view)


def replay_draws(x_shape, np_seed, torch_seed):
    np.random.seed(np_seed)
    torch.cuda.manual_seed(torch_seed)
    return draw_augment(POLICY, tuple(x_shape), DEV)


def sigma_of(D):
    out = []
    for m in D.convs():
        w = m.weight_orig.detach().double().reshape(m.weight_orig.shape[0], -1)
        out.append(torch.dot(m.weight_u.double(), w @ m.weight_v.double()).cpu())
    return torch.stack(out)


def oracle_grads(ws, us, vs, x, imsize, training, aug, gout, flips=None, near_kink=None):
    w2 = [w.detach().clone().requires_grad_(True) for w in ws]
    xo = x.double().clone().requires_grad_(True)
    out, us2, vs2, sig = do.forward(w2, us, vs, xo, imsize, training, aug, near_kink, flips)
    (out * gout.double()).sum().backward()
    return out.detach(), xo.grad, [w.grad for w in w2], us2, vs2, sig


def explain_kinks(got_dx, got_dw, args, cands, bar):
    """-> (error, flips): greedy LeakyReLU flips of near-kink oracle inputs that bring the gradients within bar"""
    def err(flips):
        _, dx, dw, *_ = oracle_grads(*args, flips=flips)
        return max(rel_l2(a, b) for a, b in zip([got_dx] + got_dw, [dx] + dw) if b is not None)
    flips, chosen = {}, []
    best = err(flips)
    for layer, j, _, numel in sorted(cands, key=lambda c: c[2])[:64]:
        if best <= bar or len(chosen) == MAX_FLIPS:
            break
        trial = {k: v.clone() for k, v in flips.items()}
        trial.setdefault(layer, torch.zeros(numel, dtype=torch.bool))[j] = True
        e = err(trial)
        if e < best:
            best, flips = e, trial
            chosen.append((layer, j))
    return best, chosen


def check_case(imsize, H, W, B, layout, fire, precision, training=True):
    D = make(imsize, precision, seed=1 + B)
    D.train(training)
    ws, us, vs = snapshot(D)
    g = torch.Generator().manual_seed(11 * B + H)
    x = torch.rand(B, 3, H, W, generator=g)
    leaf, view = as_layout(x.to(DEV), layout)
    s = _gate_seed(fire)
    out = gpu_call(D, view, s, 7)
    gout = torch.randn(out.shape, generator=g)
    (out * gout.to(DEV)).sum().backward()
    aug = replay_draws(x.shape, s, 7)
    assert (aug is not None) == fire
    args = (ws, us, vs, x, imsize, training, aug, gout)
    cands = []
    want, dx_o, dw_o, us2, vs2, sig = oracle_grads(*args, near_kink=(KINK, cands))
    bar_out, bar_grad, bar_state = BARS[precision]
    got_dx = grad_nchw(leaf, x.shape, layout).cpu().double()
    got_dw = [m.weight_orig.grad.cpu().double() for m in D.convs()]
    errs = {"out": rel_l2(out.detach().cpu().double(), want), "dx": rel_l2(got_dx, dx_o)}
    errs["dw"] = max(rel_l2(a, b) for a, b in zip(got_dw, dw_o))
    errs["u"] = max(rel_l2(m.weight_u.cpu().double(), u) for m, u in zip(D.convs(), us2))
    errs["v"] = max(rel_l2(m.weight_v.cpu().double(), v) for m, v in zip(D.convs(), vs2))
    errs["sigma"] = rel_l2(sigma_of(D), torch.stack(sig))
    flips = []
    if max(errs["dx"], errs["dw"]) > bar_grad:
        errs["grad_flipped"], flips = explain_kinks(got_dx, got_dw, args, cands, bar_grad)
    print(f"disc[{precision} imsize={imsize} {H}x{W} B={B} {layout} aug={fire}] " +
          " ".join(f"{k}={v:.2e}" for k, v in errs.items()) + f" near_kink={len(cands)} flips={flips}")
    assert errs["out"] <= bar_out, errs
    assert max(errs["dx"], errs["dw"]) <= bar_grad or errs["grad_flipped"] <= 2 * bar_grad, errs
    assert errs["u"] <= bar_state and errs["v"] <= bar_state and errs["sigma"] <= bar_state, errs


@pytest.mark.parametrize("fire", [True, False])
@pytest.mark.parametrize("layout", ["nchw", "rays"])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("imsize,H,W", BRANCHES)
def test_parity_split(imsize, H, W, B, layout, fire):
    check_case(imsize, H, W, B, layout, fire, "f16x3")


@pytest.mark.parametrize("fire", [True, False])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("imsize,H,W", BRANCHES[:3])
@pytest.mark.parametrize("precision", ["f16", "bf16"])
def test_parity_single_product(precision, imsize, H, W, B, fire):
    check_case(imsize, H, W, B, "rays", fire, precision)


@pytest.mark.parametrize("imsize,H,W", BRANCHES[:2])
def test_eval_mode_keeps_u_v(imsize, H, W):
    check_case(imsize, H, W, 2, "nchw", True, "f16x3", training=False)
    D = make(imsize).eval()
    before = [(m.weight_u.clone(), m.weight_v.clone()) for m in D.convs()]
    D(torch.rand(1, 3, H, W, device=DEV))
    for m, (u, v) in zip(D.convs(), before):
        assert torch.equal(m.weight_u, u) and torch.equal(m.weight_v, v)


@pytest.mark.parametrize("imsize,H,W", BRANCHES[:3])
def test_hinge_generator_and_discriminator_steps(imsize, H, W):
    """G step (-mean backward to the input), then the D step pair with one hinge backward to the weights: the state
    advances across calls and each call's backward uses its own sigma, u and v"""
    D = make(imsize, seed=5)
    ws, us, vs = snapshot(D)
    g = torch.Generator().manual_seed(H)
    fake, real, fake2 = (torch.rand(1, 3, H, W, generator=g) for _ in range(3))
    seeds = [(_gate_seed(True), 1), (_gate_seed(False), 2), (_gate_seed(True), 3)]
    # the library
    xf = fake.to(DEV).requires_grad_(True)
    pf = gpu_call(D, xf, *seeds[0])
    (-pf.mean()).backward()
    for m in D.convs():
        m.weight_orig.grad = None
    pr = gpu_call(D, real.to(DEV), *seeds[1])
    pf2 = gpu_call(D, fake2.to(DEV), *seeds[2])
    ((F.relu(1 - pr).mean() + F.relu(1 + pf2).mean()) / 2).backward()
    # the oracle, with the replayed draws
    augs = [replay_draws(fake.shape, *s) for s in seeds]
    # the generator step: -mean of one call, backward to the input (kinks handled as in check_case)
    gout = torch.full(pf.shape, -1.0 / pf.numel(), dtype=D64)
    g_args = (ws, us, vs, fake, imsize, True, augs[0], gout)
    cands = []
    o_pf, dx_o, _, us, vs, _ = oracle_grads(*g_args, near_kink=(KINK, cands))
    err = rel_l2(xf.grad.cpu().double(), dx_o)
    if err > 1e-4:
        err, flips = explain_kinks(xf.grad.cpu().double(), [], g_args, cands, 1e-4)
        print(f"hinge imsize={imsize} {H}x{W}: G-step input gradient explained by LeakyReLU flips {flips}")
        err /= 2
    assert err <= 1e-4
    # the discriminator step: two calls, one hinge backward to the weights, each call with its own sigma, u and v
    w2 = [w.detach().clone().requires_grad_(True) for w in ws]
    o_pr, us, vs, _ = do.forward(w2, us, vs, real.double(), imsize, True, augs[1])
    o_pf2, us, vs, _ = do.forward(w2, us, vs, fake2.double(), imsize, True, augs[2])
    ((F.relu(1 - o_pr).mean() + F.relu(1 + o_pf2).mean()) / 2).backward()
    for a, b in ((pf, o_pf), (pr, o_pr), (pf2, o_pf2)):
        assert rel_l2(a.detach().cpu().double(), b.detach()) <= 1e-4
    for m, w, u, v in zip(D.convs(), w2, us, vs):
        assert rel_l2(m.weight_orig.grad.cpu().double(), w.grad) <= 1e-4
        assert rel_l2(m.weight_u.cpu().double(), u) <= 1e-5 and rel_l2(m.weight_v.cpu().double(), v) <= 1e-5


@pytest.mark.parametrize("fire", [True, False])
def test_rng_state_after_call(fire):
    D = make(64)
    x = torch.rand(2, 3, 64, 64, device=DEV)
    s = _gate_seed(fire)
    gpu_call(D, x, s, 9)
    after = (np.random.random(), torch.rand(3, device=DEV))
    replay_draws(x.shape, s, 9)
    assert np.random.random() == after[0]
    assert torch.equal(torch.rand(3, device=DEV), after[1])


def test_deterministic():
    outs = []
    for _ in range(2):
        D = make(-1, seed=3)
        x = torch.rand(2, 3, 63, 84, generator=torch.Generator().manual_seed(0)).to(DEV).requires_grad_(True)
        out = gpu_call(D, x, _gate_seed(True), 4)
        out2 = gpu_call(D, x.detach(), _gate_seed(True), 5)
        (out.square().sum() + out2.sum()).backward()
        outs.append([out, out2, x.grad] + [t for m in D.convs() for t in (m.weight_orig.grad, m.weight_u, m.weight_v)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_no_host_sync():
    D = make(64)
    x = torch.rand(1, 3, 64, 64, device=DEV).requires_grad_(True)
    gpu_call(D, x, _gate_seed(True), 1).sum().backward()       # warm-up (library load, device check)
    torch.cuda.synchronize()
    np.random.seed(_gate_seed(True))
    torch.cuda.set_sync_debug_mode("error")
    try:
        (-D(x).mean()).backward()
        pr, pf = D(torch.rand(1, 3, 64, 64, device=DEV)), D(x.detach())
        (F.relu(1 - pr).mean() + F.relu(1 + pf).mean()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_no_grad_pass_advances_state_and_matches():
    outs = []
    for grad in (True, False):
        D = make(-1, seed=2)
        x = torch.rand(1, 3, 56, 70, generator=torch.Generator().manual_seed(1)).to(DEV)
        with torch.set_grad_enabled(grad):
            out = gpu_call(D, x.requires_grad_(grad), _gate_seed(True), 3)
        assert out.requires_grad == grad
        outs.append([out.detach()] + [t.clone() for m in D.convs() for t in (m.weight_u, m.weight_v)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_autocast_policy_is_f16():
    x = torch.rand(1, 3, 64, 64, device=DEV)
    outs = []
    for precision, ac in (("f16", False), ("autocast", True)):
        D = make(64, precision, seed=4)
        with torch.autocast("cuda", dtype=torch.float16, enabled=ac):
            outs.append(gpu_call(D, x, _gate_seed(True), 2))
    assert outs[0].dtype == outs[1].dtype == torch.float32
    assert torch.equal(outs[0], outs[1])


def test_double_backward_raises():
    D = make(64)
    x = torch.rand(1, 3, 64, 64, device=DEV).requires_grad_(True)
    out = gpu_call(D, x, _gate_seed(False), 1)
    (gx,) = torch.autograd.grad(out.sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.pow(2).sum().backward()


def test_input_checks():
    D = make(64)
    with pytest.raises(ValueError):
        D(torch.rand(1, 4, 64, 64, device=DEV))
    with pytest.raises(TypeError):
        D(torch.rand(1, 3, 64, 64, device=DEV, dtype=torch.float64))
    with pytest.raises(ValueError):
        D(torch.rand(1, 3, 8, 8, device=DEV))
