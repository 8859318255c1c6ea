"""CPU tests of the fused optimisers over the discriminator (`get_optimizer(hparams, [D], rate=0.2)`): the rules they
are held to on the GPU -- oracle/optim_oracle.py for SGD / RAdam / Ranger, torch.optim.Adam's single-tensor path for
Adam -- against the reference's own get_optimizer on the discriminator's parameter shapes, bit for bit
(tests/golden/disc_optim_steps.npz, written by tests/golden/make_disc_optim_golden.py); get_optimizer's choices for a
Discriminator and its refusals of other modules; and the argument checks of snb_optim_step_tensors.  No compute is
launched on a GPU here."""
import ctypes as C

import numpy as np
import pytest
import torch

from sinnerf_b200 import _lib, build
from tests._common import load_npz
from tests.test_optim_cpu import optim_case_grad, optim_digests

# The fixture cases: 14 steps on the weight_orig tensors of a Discriminator (imsize 64: 5 convolutions, -1: 3), lr
# halved after step 7, and tensor 1 without a gradient on steps 0 and 7 (so its state starts one step late and its
# count lags).  14 steps cover RAdam's switch to the adaptive step (step 6) and Ranger's two syncs (steps 6 and 12).
DISC_OPTIM_STEPS = 14
DISC_NO_GRAD = {1: (0, 7)}
DISC_CASES = [(rule, imsize, wd) for rule in ("sgd", "adam", "radam", "ranger") for imsize in (64, -1)
              for wd in (0.0, 1e-2)]


class HParams:
    """The options get_optimizer reads (opt.py defaults, --weight_decay as given)."""
    lr, momentum = 5e-4, 0.9

    def __init__(self, optimizer, weight_decay=0.0):
        self.optimizer, self.weight_decay = optimizer, weight_decay


def disc_case_module(imsize):
    """A CPU Discriminator whose weight_orig tensors hold seeded values (numpy's generator: the same bits everywhere)."""
    from sinnerf_b200.discriminator import Discriminator
    d = Discriminator(False, "color,cutout", imsize=imsize)
    with torch.no_grad():
        for i, p in enumerate(d.parameters()):
            p.copy_(torch.from_numpy(np.random.default_rng([77, i]).uniform(-0.1, 0.1, tuple(p.shape))
                                     .astype(np.float32)))
    return d


def oracle_get_optimizer(hparams, models, rate=1):
    """utils/__init__.py:10-31 over the rules the tests hold the fused optimisers to."""
    from oracle import optim_oracle
    params = [p for m in models for p in m.parameters()]
    lr, wd = hparams.lr * rate, hparams.weight_decay
    if hparams.optimizer == "sgd":
        return optim_oracle.SGD(params, lr=lr, momentum=hparams.momentum, weight_decay=wd)
    if hparams.optimizer == "adam":
        return torch.optim.Adam(params, lr=lr, eps=1e-8, weight_decay=wd, foreach=False)
    if hparams.optimizer == "radam":
        return optim_oracle.RAdam(params, lr=lr, eps=1e-8, weight_decay=wd)
    return optim_oracle.Ranger(params, lr=lr, eps=1e-8, weight_decay=wd)


def run_disc_case(get_optimizer, rule, imsize, wd):
    d = disc_case_module(imsize)
    opt = get_optimizer(HParams(rule, wd), [d], rate=0.2)
    params = list(d.parameters())
    for step in range(DISC_OPTIM_STEPS):
        if step == 7:
            opt.param_groups[0]["lr"] *= 0.5
        for i, p in enumerate(params):
            p.grad = None if step in DISC_NO_GRAD.get(i, ()) else optim_case_grad(step, i, p.shape)
        opt.step()
    return params, opt


def case_tag(rule, imsize, wd):
    return f"{rule}_im{imsize}_wd{wd:g}"


@pytest.mark.parametrize("rule,imsize,wd", DISC_CASES)
def test_oracle_matches_reference_get_optimizer_on_discriminator(rule, imsize, wd):
    want = load_npz("disc_optim_steps.npz")
    tag = case_tag(rule, imsize, wd)
    got = optim_digests(tag, *run_disc_case(oracle_get_optimizer, rule, imsize, wd))
    keys = sorted(k for k in want if k.startswith(tag + "/"))
    assert keys and keys == sorted(got), tag
    bad = [k for k in keys if (str(int(want[k])) if k.endswith("/step") else want[k].tobytes().hex()) != got[k]]
    assert not bad, f"{len(bad)} of {len(keys)} tensors differ from the reference, first {bad[:5]}"
    if rule != "sgd":   # the tensor without a gradient on two steps: its count lags by two
        assert int(want[f"{tag}/1/step"]) == DISC_OPTIM_STEPS - 2


@pytest.mark.parametrize("imsize,n_tensors", [(128, 6), (64, 5), (32, 4), (-1, 3)])
def test_get_optimizer_fuses_the_discriminator(imsize, n_tensors):
    from sinnerf_b200.discriminator import Discriminator
    from sinnerf_b200.optim import FusedAdam, FusedRAdam, FusedRanger, FusedSGD, get_optimizer
    d = Discriminator(False, "color,cutout", imsize=imsize)
    want = {"sgd": (FusedSGD, dict(lr=1e-4, momentum=0.9, weight_decay=1e-3, dampening=0.0, nesterov=False)),
            "adam": (FusedAdam, dict(lr=1e-4, eps=1e-8, weight_decay=1e-3, betas=(0.9, 0.999))),
            "radam": (FusedRAdam, dict(lr=1e-4, eps=1e-8, weight_decay=1e-3, betas=(0.9, 0.999))),
            "ranger": (FusedRanger, dict(lr=1e-4, eps=1e-8, weight_decay=1e-3, betas=(0.95, 0.999), alpha=0.5, k=6,
                                         N_sma_threshhold=5))}
    for name, (cls, hp) in want.items():
        opt = get_optimizer(HParams(name, 1e-3), [d], rate=0.2)
        assert type(opt) is cls, name
        group = opt.param_groups[0]
        assert [id(p) for p in group["params"]] == [id(c.weight_orig) for c in d.convs()]
        assert len(group["params"]) == n_tensors
        for k, v in hp.items():
            assert group[k] == pytest.approx(v), (name, k)
        assert not opt.state                      # state appears on a parameter's first step, as in torch
        # the state dict has the layout torch's / the reference's optimiser over D.parameters() has
        ref = oracle_get_optimizer(HParams(name, 1e-3), [d], rate=0.2)
        assert opt.state_dict()["param_groups"][0]["params"] == ref.state_dict()["param_groups"][0]["params"]


def test_get_optimizer_refuses_other_modules():
    from sinnerf_b200.discriminator import Discriminator
    from sinnerf_b200.nerf import NeRF
    from sinnerf_b200.optim import FusedAdam, FusedRAdam, FusedRanger, FusedSGD, get_optimizer
    d = Discriminator(False, None, imsize=-1)
    others = [[torch.nn.Linear(3, 3)], [torch.nn.Conv2d(3, 8, 4)], list(d.parameters()), [d, NeRF()], [], [d.main]]
    for name in ("sgd", "adam", "radam", "ranger"):
        for models in others:
            with pytest.raises(TypeError):
                get_optimizer(HParams(name), models, rate=0.2)
    for cls in (FusedAdam, FusedRAdam, FusedRanger):
        with pytest.raises(TypeError):
            cls([torch.nn.Linear(3, 3)])
    with pytest.raises(TypeError):
        FusedSGD([torch.nn.Linear(3, 3)], lr=1e-3)


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_optim_step_tensors_argument_validation_without_gpu(lib):
    """Every refusal returns SNB_ERR_INVALID with a message before anything is launched (the pointers are fake)."""
    fake = C.c_void_p(256)
    n = 3
    params = (C.c_void_p * n)(*([256] * n))
    grads = (C.c_void_p * n)(*([256] * n))
    numel = (C.c_int64 * n)(12288, 2097152, 8192)
    steps = (C.c_int * n)(1, 1, 1)

    def call(rule=_lib.OPTIM_ADAM, n=n, params=params, grads=grads, numel=numel, steps=steps, bufs=(fake, fake, fake),
             **hp):
        a = _lib.SnbOptimArgs(rule=rule, **dict(dict(lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, alpha=0.5, k=6), **hp))
        rc = lib.snb_optim_step_tensors(n, params, grads, numel, steps, *bufs, C.byref(a), None)
        return rc, lib.snb_last_error()

    for table in ("params", "grads", "numel", "steps"):
        assert call(**{table: None}) == (-1, b"snb_optim_step_tensors: null table or args"), table
    assert lib.snb_optim_step_tensors(n, params, grads, numel, steps, fake, fake, fake, None, None) == -1
    for bad_n in (0, -1, _lib.OPTIM_MAX_TENSORS + 1):
        rc, msg = call(n=bad_n)
        assert rc == -1 and b"1 <= n <= 32" in msg, bad_n
    rc, msg = call(rule=7)
    assert rc == -1 and b"unknown rule 7" in msg
    for bad in (0, -5):
        rc, msg = call(numel=(C.c_int64 * n)(12288, bad, 8192))
        assert rc == -1 and b"numel of tensor 1" in msg, bad
    rc, msg = call(params=(C.c_void_p * n)(256, 256, None))
    assert rc == -1 and b"parameter tensor 2 is null" in msg
    # the state buffers each rule needs
    for rule, bufs in ((_lib.OPTIM_ADAM, (None, fake, None)), (_lib.OPTIM_ADAM, (fake, None, None)),
                       (_lib.OPTIM_RADAM, (fake, None, None)), (_lib.OPTIM_RANGER, (fake, fake, None)),
                       (_lib.OPTIM_SGD, (None, None, None))):
        rc, msg = call(rule=rule, bufs=bufs, momentum=0.9)
        assert rc == -1 and b"null state buffer" in msg, (rule, bufs)
    rc, msg = call(steps=(C.c_int * n)(1, 0, 1))
    assert rc == -1 and b"step of tensor 1 counts from 1" in msg
    rc, msg = call(beta2=1.0)
    assert rc == -1 and b"hyper-parameters" in msg
    rc, msg = call(rule=_lib.OPTIM_RANGER, k=0)
    assert rc == -1 and b"hyper-parameters" in msg
    # accepted shapes of the checks, stopped only by the hyper-parameter check so nothing launches: a tensor without a
    # gradient needs no step count, and SGD without momentum needs no buffer
    rc, msg = call(grads=(C.c_void_p * n)(256, None, 256), steps=(C.c_int * n)(1, 0, 1), lr=-1.0)
    assert rc == -1 and b"hyper-parameters" in msg
    rc, msg = call(rule=_lib.OPTIM_SGD, bufs=(None, None, None), steps=(C.c_int * n)(0, 0, 0), lr=-1.0)
    assert rc == -1 and b"hyper-parameters" in msg
    # the 24-tensor NeRF entry point does not take the Adam rule (snb_adam_step serves it)
    a = _lib.SnbOptimArgs(rule=_lib.OPTIM_ADAM, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, k=1)
    nerf = (C.c_void_p * 24)(*([256] * 24))
    assert lib.snb_optim_step(nerf, nerf, fake, fake, fake, C.byref(a), 0, 1, None, None) == -1
    assert b"unknown rule 3" in lib.snb_last_error()
