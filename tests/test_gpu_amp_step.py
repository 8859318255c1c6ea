"""GPU tests of GradScaler-native stepping (`_step_supports_amp_scaling`, C ABI snb_*_amp): the fused optimisers
unscale the gradients and skip a step on found_inf inside their kernels, with the update counts on the device, and
must leave exactly what the plain path (`amp_scaling=False`: GradScaler's own unscale pass and its host check of
found_inf) leaves.  Every rule, over both NeRF models and over a Discriminator, on the same gradients: parameters,
`.grad` after `scaler.step`, every state buffer, `state()` / `state_dict()`, the scaler's scale and growth tracker and
the NeRF weight images past their headers are compared bit for bit (NaN payloads included).  Also: `scaler.unscale_`
before `scaler.step`, runs of queued steps longer than the scalar window, state dicts taken right after a skipped step
moving through the replaced optimisers and back, the 'autocast' policy, and that `scaler.step` no longer waits for
the GPU."""
import copy
import time

import pytest
import torch

from tests.test_disc_optim_cpu import HParams

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RULES = ["adam", "sgd", "radam", "ranger"]
WD = 1e-2
NO_GRAD = 1          # the tensor without a gradient on a schedule's "nograd" steps (its count lags)


def nerf_models(seed=0):
    from sinnerf_b200.nerf import NeRF
    torch.manual_seed(seed)
    return [NeRF(use_new_activation=True).to(DEV), NeRF(use_new_activation=True).to(DEV)]


def disc(seed=0):
    from sinnerf_b200.discriminator import Discriminator
    torch.manual_seed(seed)
    return [Discriminator(False, "color,cutout", imsize=64).to(DEV)]


def make_modules(kind):
    return nerf_models() if kind == "nerf" else disc()


def params_of(models):
    from sinnerf_b200.optim import _params
    return [p for m in models for p in _params(m)]


def make_opt(rule, models, amp_scaling):
    """get_optimizer's configuration of each rule (rate 0.2 for the discriminator), with amp_scaling chosen."""
    from sinnerf_b200 import optim
    from sinnerf_b200.discriminator import Discriminator
    lr = HParams.lr * (0.2 if isinstance(models[0], Discriminator) else 1.0)
    if rule == "sgd":
        return optim.FusedSGD(models, lr=lr, momentum=HParams.momentum, weight_decay=WD, amp_scaling=amp_scaling)
    cls = dict(adam=optim.FusedAdam, radam=optim.FusedRAdam, ranger=optim.FusedRanger)[rule]
    return cls(models, lr=lr, eps=1e-8, weight_decay=WD, amp_scaling=amp_scaling)


def grad_sets(models, n_steps, seed=0):
    """n_steps lists of unscaled gradients, one per tensor, of a training step's magnitude."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    ps = params_of(models)
    return [[torch.randn(p.shape, generator=g, device=DEV) * 1e-2 for p in ps] for _ in range(n_steps)]


def set_grads(models, scaler, grads, event):
    """The scaled gradients a backward of scaler.scale(loss) gives (no host sync), with the step's event planted:
    'inf' / 'nan' in one element of tensor 0, 'nograd' drops tensor NO_GRAD's gradient."""
    for i, (p, g) in enumerate(zip(params_of(models), grads)):
        p.grad = None if (event == "nograd" and i == NO_GRAD) else scaler.scale(g)
    if event in ("inf", "nan"):
        params_of(models)[0].grad.view(-1)[7] = float(event)


class Run:
    """One optimiser over its own copy of the modules, with its own GradScaler."""

    def __init__(self, rule, kind, amp_scaling, init_scale, models=None):
        self.models = models if models is not None else make_modules(kind)
        self.opt = make_opt(rule, self.models, amp_scaling)
        assert self.opt._step_supports_amp_scaling is amp_scaling
        self.scaler = torch.amp.GradScaler("cuda", init_scale=init_scale, growth_interval=3)

    def step(self, grads, event="ok", unscale_first=False):
        set_grads(self.models, self.scaler, grads, event)
        if unscale_first:
            self.scaler.unscale_(self.opt)
        self.scaler.step(self.opt)
        self.scaler.update()


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_same(a, b, what):
    """Bit-for-bit equality of nested state: tensors (dtype, device and bits, NaNs included), dicts, lists, scalars."""
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.dtype == b.dtype and a.device == b.device and a.shape == b.shape, what
        assert torch.equal(bits(a), bits(b)), what
    elif isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (what, list(a), list(b))
        for k in a:
            assert_same(a[k], b[k], f"{what}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{what}[{i}]")
    else:
        assert type(a) is type(b) and a == b, (what, a, b)


def compare(old, new, what, extra_group_keys=False):
    """Everything the two runs leave: parameters, gradients, state (through `state` and `state_dict()`), the scaler,
    and the NeRF weight images past their 256-byte headers plus the checksum stamped in the header.  extra_group_keys:
    `new` went through torch's Adam / SGD, whose param groups add their own defaults."""
    pa, pb = params_of(old.models), params_of(new.models)
    for i, (x, y) in enumerate(zip(pa, pb)):
        assert_same(x.detach(), y.detach(), f"{what}: parameter {i}")
        assert (x.grad is None) == (y.grad is None), (what, i)
        if x.grad is not None:
            assert_same(x.grad, y.grad, f"{what}: .grad {i}")
    for i, (x, y) in enumerate(zip(pa, pb)):
        assert_same(old.opt.state.get(x, {}), new.opt.state.get(y, {}), f"{what}: state of {i}")
    sd_old, sd_new = old.opt.state_dict(), new.opt.state_dict()
    assert_same(sd_old["state"], sd_new["state"], f"{what}: state_dict state")
    for ga, gb in zip(sd_old["param_groups"], sd_new["param_groups"]):
        assert_same(ga, {k: gb[k] for k in ga} if extra_group_keys else gb, f"{what}: state_dict param group")
    assert_same(old.scaler._scale, new.scaler._scale, f"{what}: scale")
    assert_same(old.scaler._growth_tracker, new.scaler._growth_tracker, f"{what}: growth tracker")
    for ma, mb in zip(old.models, new.models):
        packed_a, packed_b = getattr(ma, "_packed", {}), getattr(mb, "_packed", {})
        assert packed_a.keys() == packed_b.keys(), what
        for key in packed_a:
            assert torch.equal(packed_a[key][24:32], packed_b[key][24:32]), (what, key, "checksum")
            assert torch.equal(packed_a[key][256:], packed_b[key][256:]), (what, key, "image")


# A run with two skipped steps (an inf, then a NaN) and a tensor without a gradient on two steps.  Ranger (k = 6)
# syncs on a tensor's 6th taken step: step 7 here, right after the skip at step 6.
SCHEDULE = ["ok", "nograd", "ok", "inf", "ok", "ok", "nan", "ok", "ok", "nograd", "ok", "ok"]


@pytest.mark.parametrize("init_scale", [2.0 ** 12, 3000.0])
@pytest.mark.parametrize("kind", ["nerf", "disc"])
@pytest.mark.parametrize("rule", RULES)
def test_amp_steps_match_plain_path(rule, kind, init_scale):
    """Step by step, the GradScaler-native path leaves what the plain path leaves; skipped steps move nothing but
    `.grad` (unscaled) and the scale (backed off), and the growth interval of 3 makes the scale grow mid-run."""
    old = Run(rule, kind, False, init_scale)
    new = Run(rule, kind, True, init_scale)
    grads = grad_sets(old.models, len(SCHEDULE))
    scales = set()
    for step, event in enumerate(SCHEDULE):
        before = [p.detach().clone() for p in params_of(new.models)]
        scale = new.scaler.get_scale()
        scales.add(scale)
        old.step(grads[step], event)
        new.step(grads[step], event)
        if event in ("inf", "nan"):
            assert all(torch.equal(x, p.detach()) for x, p in zip(before, params_of(new.models))), step
            assert new.scaler.get_scale() == scale * 0.5, step
        compare(old, new, f"{rule} {kind} scale {init_scale} step {step} ({event})")
    assert len(scales) == 3, scales          # grown after steps 0-2, backed off at 3 and at 6


@pytest.mark.parametrize("kind", ["nerf", "disc"])
@pytest.mark.parametrize("rule", RULES)
def test_queued_steps_past_the_window(rule, kind):
    """20 steps queued behind 100 ms of GPU sleep, so the host never sees a count until it must: 5 taken, 10 skipped
    (more than the window's 8, which forces one blocking read), 5 taken (Ranger's 6th update of each tensor is the
    first taken step after the skips).  The plain path runs the same schedule; they end equal."""
    from sinnerf_b200 import _lib
    assert _lib.OPTIM_WINDOW < 10
    schedule = ["ok"] * 5 + ["inf"] * 10 + ["ok"] * 5
    old = Run(rule, kind, False, 2.0 ** 12)
    new = Run(rule, kind, True, 2.0 ** 12)
    grads = grad_sets(old.models, len(schedule), seed=1)
    for step, event in enumerate(schedule):
        old.step(grads[step], event)
    new.step(grads[0], "ok")                  # first step: the count buffers and read-back ring are allocated
    torch.cuda.synchronize()
    torch.cuda._sleep(sleep_cycles(0.1))
    for step, event in enumerate(schedule[1:], 1):
        new.step(grads[step], event)
    compare(old, new, f"{rule} {kind} queued")


@pytest.mark.parametrize("kind", ["nerf", "disc"])
@pytest.mark.parametrize("rule", RULES)
def test_unscale_then_step(rule, kind):
    """scaler.unscale_(opt) then scaler.step(opt): GradScaler hands the step grad_scale=None, and the gradients are
    not unscaled a second time."""
    old = Run(rule, kind, False, 3000.0)
    new = Run(rule, kind, True, 3000.0)
    schedule = ["ok", "ok", "inf", "ok"]
    grads = grad_sets(old.models, len(schedule), seed=2)
    for step, event in enumerate(schedule):
        old.step(grads[step], event, unscale_first=True)
        new.step(grads[step], event, unscale_first=True)
        compare(old, new, f"{rule} {kind} unscale_ step {step}")


def replaced_optimizer(rule, kind, models):
    """The optimiser the fused one replaces, over the same tensors in the same order: torch's Adam (single-tensor) and
    SGD, the oracle's RAdam / Ranger."""
    from oracle import optim_oracle
    ps = params_of(models)
    lr = HParams.lr * (0.2 if kind == "disc" else 1.0)
    if rule == "adam":
        return torch.optim.Adam(ps, lr=lr, eps=1e-8, weight_decay=WD, foreach=False)
    if rule == "sgd":
        return torch.optim.SGD(ps, lr=lr, momentum=HParams.momentum, weight_decay=WD)
    return dict(radam=optim_oracle.RAdam, ranger=optim_oracle.Ranger)[rule](ps, lr=lr, eps=1e-8, weight_decay=WD)


@pytest.mark.parametrize("kind", ["nerf", "disc"])
@pytest.mark.parametrize("rule", RULES)
def test_state_dict_after_a_skipped_step(rule, kind):
    """state_dict() read right after a skipped step (the counts still on the device) equals the plain path's, loads
    into the replaced optimiser, comes back from it unchanged into a fresh fused optimiser, and that one steps on
    exactly like the original."""
    schedule = ["ok", "nograd", "ok", "inf"]
    old = Run(rule, kind, False, 2.0 ** 12)
    new = Run(rule, kind, True, 2.0 ** 12)
    grads = grad_sets(old.models, len(schedule) + 2, seed=3)
    for step, event in enumerate(schedule):
        old.step(grads[step], event)
        new.step(grads[step], event)
    assert new.opt._stale
    saved = copy.deepcopy(new.opt.state_dict())
    assert_same(copy.deepcopy(old.opt.state_dict()), saved, "state_dict after the skip")

    twin = copy.deepcopy(new.models)
    ref = replaced_optimizer(rule, kind, twin)
    ref.load_state_dict(copy.deepcopy(saved))
    back = make_opt(rule, twin, True)
    back.load_state_dict(copy.deepcopy(ref.state_dict()))
    returned = back.state_dict()
    assert_same(returned["state"], saved["state"], "fused -> replaced -> fused: state")
    for ga, gb in zip(saved["param_groups"], returned["param_groups"]):   # the replaced one adds its own defaults
        assert_same(ga, {k: gb[k] for k in ga}, "fused -> replaced -> fused: param group")
    resumed = Run(rule, kind, True, 2.0 ** 12, models=twin)
    resumed.opt = back
    resumed.scaler.load_state_dict(new.scaler.state_dict())
    for step in range(len(schedule), len(schedule) + 2):
        new.step(grads[step])
        resumed.step(grads[step])
        compare(new, resumed, f"{rule} {kind} resumed step {step}", extra_group_keys=True)


def room_rays(n):
    from sinnerf_b200 import synthetic
    return synthetic.patch_rays("llff", 63, 84, 4, seed=0)[:n].contiguous()


@pytest.mark.parametrize("rule", RULES)
def test_autocast_policy(rule):
    """precision='autocast' under fp16 autocast, as Lightning's precision=16 runs it: each step re-packs the f16 image
    of the model's last pass.  The gradients of one backward go to both runs (larger passes differ in their last bits
    from run to run); each run still makes its own pass first, so its image is the one its forward refreshed."""
    from sinnerf_b200 import _lib, optim
    from sinnerf_b200.nerf import Embedding
    from sinnerf_b200.rendering import render_rays
    runs = []
    for amp_scaling in (False, True):
        models = nerf_models(seed=4)
        cls = dict(adam=optim.FusedAdam, sgd=optim.FusedSGD, radam=optim.FusedRAdam, ranger=optim.FusedRanger)[rule]
        kw = dict(momentum=HParams.momentum) if rule == "sgd" else {}
        r = Run(rule, "nerf", amp_scaling, 2.0 ** 16, models=models)
        r.opt = cls(models, lr=1e-3, precision="autocast", amp_scaling=amp_scaling, **kw)
        runs.append(r)
    rays = room_rays(256).to(DEV)
    target = torch.rand(256, 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    embeddings = [Embedding(3, 10), Embedding(3, 4)]
    for step in range(5):
        for r in runs:
            for p in params_of(r.models):
                p.grad = None
            with torch.autocast("cuda", dtype=torch.float16):
                out = render_rays(r.models, embeddings, rays, 32, False, 0, 0, 32, 32768, False, precision="autocast")
                loss = ((out["rgb_fine"] - target) ** 2).mean() + ((out["rgb_coarse"] - target) ** 2).mean()
            r.scaler.scale(loss).backward()
        for p, q in zip(params_of(runs[0].models), params_of(runs[1].models)):
            q.grad = p.grad.clone()
        if step == 2:
            for r in runs:
                params_of(r.models)[4].grad.view(-1)[0] = float("inf")
        for r in runs:
            r.scaler.step(r.opt)
            r.scaler.update()
        compare(runs[0], runs[1], f"{rule} autocast step {step}")
    f16 = _lib.precision_id("f16")
    for m in runs[1].models:
        assert m._last_prec == f16 and (f16, str(torch.device(DEV))) in m._packed


def sleep_cycles(seconds):
    """torch.cuda._sleep's argument for about `seconds` of GPU time, calibrated once."""
    if not hasattr(sleep_cycles, "rate"):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        torch.cuda._sleep(10 ** 7)
        end.record()
        end.synchronize()
        sleep_cycles.rate = 10 ** 7 / (start.elapsed_time(end) * 1e-3)
    return int(seconds * sleep_cycles.rate)


def host_time_of_step(run, grads):
    """Host seconds `scaler.step(opt)` takes with ~200 ms of GPU work queued ahead of it."""
    set_grads(run.models, run.scaler, grads, "ok")
    torch.cuda.synchronize()
    torch.cuda._sleep(sleep_cycles(0.2))
    t0 = time.perf_counter()
    run.scaler.step(run.opt)
    t1 = time.perf_counter()
    run.scaler.update()
    torch.cuda.synchronize()
    return t1 - t0


@pytest.mark.parametrize("kind", ["nerf", "disc"])
def test_scaler_step_does_not_wait_for_the_gpu(kind):
    """The plain path's scaler.step reads found_inf on the host, so it waits out the queued work; the
    GradScaler-native step returns at once.  Generous bounds: this checks the sync, not the speed."""
    times = {}
    for amp_scaling in (False, True):
        run = Run("adam", kind, amp_scaling, 2.0 ** 12)
        grads = grad_sets(run.models, 3, seed=5)
        run.step(grads[0])                          # first step: lazy allocations
        run.step(grads[1])
        times[amp_scaling] = host_time_of_step(run, grads[2])
    assert times[False] > 0.1, times
    assert times[True] < 0.05, times
