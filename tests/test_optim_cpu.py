"""CPU tests of the fused SGD / RAdam / Ranger: the oracle (oracle/optim_oracle.py) against the reference's own
optimisers bit for bit (tests/golden/optim_steps.npz, written by tests/golden/make_optim_golden.py), the new C-ABI entry
point's argument checks, and get_optimizer's choices.  No compute is launched on a GPU here."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

from sinnerf_b200 import _lib, build
from tests._common import load_npz

# The fixture cases: 14 steps on the 48 tensors of two default-init NeRFs (seeds 0 and 1, state-dict order), lr
# halved after step 7 (a scheduler), and two tensors without a gradient on some steps (tensor 3 on its first step,
# so its state starts late; tensor 30 in the middle).  14 steps cover RAdam's switch to the adaptive step (N_sma
# reaches 5 at step 6) and two Ranger lookahead syncs (k = 6).
OPTIM_STEPS = 14
OPTIM_LR = 5e-4
OPTIM_CASES = [(rule, wd) for rule in ("sgd", "radam", "ranger") for wd in (0.0, 1e-2)]
NO_GRAD = {3: (0, 7), 30: (4, 5)}   # tensor index -> steps on which it has no gradient


def optim_case_params():
    from oracle.render_oracle import default_init_params
    return [v.clone() for seed in (0, 1) for v in default_init_params(seed).values()]


def optim_case_grad(step, i, shape):
    # numpy's generator: the same bits on every platform
    g = np.random.default_rng([step, i]).standard_normal(tuple(shape), dtype=np.float32) * np.float32(1e-2)
    return torch.from_numpy(g)


def make_optimizer(mod, params, rule, wd):
    """The optimiser get_optimizer builds for `rule` (utils/__init__.py:15-27), from module `mod` (the oracle or
    the reference's classes)."""
    if rule == "sgd":
        return mod.SGD(params, lr=OPTIM_LR, momentum=0.9, weight_decay=wd)
    if rule == "radam":
        return mod.RAdam(params, lr=OPTIM_LR, eps=1e-8, weight_decay=wd)
    return mod.Ranger(params, lr=OPTIM_LR, eps=1e-8, weight_decay=wd)


def run_optim_case(mod, rule, wd):
    params = [torch.nn.Parameter(p) for p in optim_case_params()]
    opt = make_optimizer(mod, params, rule, wd)
    for step in range(OPTIM_STEPS):
        if step == 7:
            opt.param_groups[0]["lr"] *= 0.5
        for i, p in enumerate(params):
            p.grad = None if step in NO_GRAD.get(i, ()) else optim_case_grad(step, i, p.shape)
        opt.step()
    return params, opt


def optim_digests(tag, params, opt):
    """{key: sha256 of the tensor's bytes, or the step count} for every parameter and state tensor."""
    out = {}
    for i, p in enumerate(params):
        out[f"{tag}/{i}/param"] = hashlib.sha256(p.detach().numpy().tobytes()).hexdigest()
        for k, v in opt.state[p].items():
            out[f"{tag}/{i}/{k}"] = str(int(v)) if k == "step" else hashlib.sha256(v.numpy().tobytes()).hexdigest()
    return out


@pytest.mark.parametrize("rule,wd", OPTIM_CASES)
def test_oracle_matches_reference_optimizers(rule, wd):
    from oracle import optim_oracle
    want = load_npz("optim_steps.npz")
    tag = f"{rule}_wd{wd:g}"
    got = optim_digests(tag, *run_optim_case(optim_oracle, rule, wd))
    keys = sorted(k for k in want if k.startswith(tag + "/"))
    assert keys == sorted(got), tag
    bad = [k for k in keys if (str(int(want[k])) if k.endswith("/step") else want[k].tobytes().hex()) != got[k]]
    assert not bad, f"{len(bad)} of {len(keys)} tensors differ from the reference, first {bad[:5]}"


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_optim_step_argument_validation_without_gpu(lib):
    nul = (C.c_void_p * 24)()
    a = _lib.SnbOptimArgs(rule=_lib.OPTIM_RADAM, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, k=1)
    assert lib.snb_optim_step(None, None, None, None, None, C.byref(a), 0, 1, None, None) == -1
    assert b"null pointer" in lib.snb_last_error()
    fake = C.c_void_p(256)
    assert lib.snb_optim_step(nul, nul, fake, None, None, C.byref(a), 0, 1, None, None) == -1
    assert b"state buffer" in lib.snb_last_error()
    params = (C.c_void_p * 24)(*([256] * 24))
    grads = (C.c_void_p * 24)(*([256] * 24))
    assert lib.snb_optim_step(params, grads, fake, fake, None, C.byref(a), 0, 1, None, None) == -1
    assert b"counts from 1" in lib.snb_last_error()
    a.rule = 7
    assert lib.snb_optim_step(params, grads, fake, fake, fake, C.byref(a), 0, 1, None, None) == -1
    assert b"unknown rule" in lib.snb_last_error()
    a = _lib.SnbOptimArgs(rule=_lib.OPTIM_RANGER, lr=1e-3, beta1=0.95, beta2=0.999, eps=1e-8, alpha=0.5, k=0)
    a.step[:] = [1] * 24
    assert lib.snb_optim_step(params, grads, fake, fake, fake, C.byref(a), 0, 1, None, None) == -1
    assert b"hyper-parameters" in lib.snb_last_error()


class _HParams:
    lr, momentum, weight_decay = 5e-4, 0.9, 1e-3

    def __init__(self, optimizer):
        self.optimizer = optimizer


def test_get_optimizer_choices():
    from sinnerf_b200.nerf import NeRF
    from sinnerf_b200.optim import FusedAdam, FusedRAdam, FusedRanger, FusedSGD, get_optimizer
    models = [NeRF(use_new_activation=True), NeRF(use_new_activation=True)]
    want = {"sgd": (FusedSGD, dict(lr=1e-3, momentum=0.9, weight_decay=1e-3, dampening=0.0, nesterov=False)),
            "adam": (FusedAdam, dict(lr=1e-3, eps=1e-8, weight_decay=1e-3, betas=(0.9, 0.999))),
            "radam": (FusedRAdam, dict(lr=1e-3, eps=1e-8, weight_decay=1e-3, betas=(0.9, 0.999))),
            "ranger": (FusedRanger, dict(lr=1e-3, eps=1e-8, weight_decay=1e-3, betas=(0.95, 0.999), alpha=0.5, k=6,
                                         N_sma_threshhold=5))}
    for name, (cls, hp) in want.items():
        opt = get_optimizer(_HParams(name), models, rate=2)
        assert type(opt) is cls, name
        group = opt.param_groups[0]
        assert len(group["params"]) == 48
        for k, v in hp.items():
            assert group[k] == v, (name, k)
    with pytest.raises(ValueError):
        get_optimizer(_HParams("lbfgs"), models)


def test_fused_group_keys_match_the_reference():
    """A state dict carries the param-group keys the reference's step reads, so it loads back into the reference."""
    from oracle import optim_oracle
    from sinnerf_b200.nerf import NeRF
    from sinnerf_b200.optim import FusedRAdam, FusedRanger, FusedSGD
    models = [NeRF(use_new_activation=True)]
    ps = list(models[0].parameters())
    for fused, ref in ((FusedSGD(models, lr=1e-3, momentum=0.9), optim_oracle.SGD(ps, lr=1e-3, momentum=0.9)),
                       (FusedRAdam(models), optim_oracle.RAdam(ps)), (FusedRanger(models), optim_oracle.Ranger(ps))):
        assert set(ref.param_groups[0]) <= set(fused.param_groups[0]), type(fused).__name__
    assert "buffer" in FusedRAdam(models).param_groups[0]     # utils/optimizers.py:70 reads group['buffer']
