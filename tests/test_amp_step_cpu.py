"""CPU tests of the GradScaler-native optimiser entry points (snb_adam_step_amp, snb_optim_step_amp,
snb_optim_step_tensors_amp): their ctypes signatures and SnbAmpStep's layout match the header, and every refusal
returns SNB_ERR_INVALID with a message before anything is launched (the pointers are fake).  Also the Python side that
needs no GPU: which optimisers GradScaler drives natively, and the per-instance way back."""
import ctypes as C
import os
import re

import pytest

from sinnerf_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = C.c_void_p(256)


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def header():
    return open(os.path.join(ROOT, "include", "sinnerf_b200.h")).read()


def test_header_constants_and_struct_layout():
    src = header()
    assert int(re.search(r"#define SNB_OPTIM_WINDOW (\d+)", src).group(1)) == _lib.OPTIM_WINDOW
    body = re.search(r"typedef struct SnbAmpStep \{(.*?)\} SnbAmpStep;", src, re.S).group(1)
    fields = re.findall(r"(\w+)(?:\[\w+\])?;", body)
    assert fields == [f for f, _ in _lib.SnbAmpStep._fields_]
    assert C.sizeof(_lib.SnbAmpStep) == 4 * 8 + 4 * _lib.OPTIM_MAX_TENSORS
    assert _lib.SnbAmpStep.base.offset == 32


def test_signatures():
    """Argument counts against the header's prototypes; grads are writable (float* const*) in the _amp forms."""
    src = re.sub(r"/\*.*?\*/", "", header(), flags=re.S)
    for name in ("snb_adam_step_amp", "snb_optim_step_amp", "snb_optim_step_tensors_amp"):
        proto = re.search(name + r"\((.*?)\);", src, re.S).group(1)
        assert len(proto.split(",")) == len(_lib.SIGNATURES[name][1]), name
        assert re.search(r"float\* const\* grads", proto), name
        assert "const SnbAmpStep* amp" in proto, name


def amp_ctl(n, base=1, out_offset=32, **kw):
    """An SnbAmpStep over host memory (never dereferenced: every call here is refused first); count_out starts
    out_offset ints after count_in."""
    counts = (C.c_int * 64)()
    a = _lib.SnbAmpStep(scale=None, found_inf=None, count_in=C.cast(counts, C.c_void_p),
                        count_out=C.c_void_p(C.addressof(counts) + 4 * out_offset))
    for i in range(_lib.OPTIM_MAX_TENSORS):
        a.base[i] = base
    for k, v in kw.items():
        setattr(a, k, v)
    return a, counts


def test_adam_step_amp_argument_validation_without_gpu(lib):
    params = (C.c_void_p * 24)(*([256] * 24))
    args = _lib.SnbAdamArgs(1e-3, 0.9, 0.999, 1e-8, 0.0, 0)     # step is not read by the _amp form

    def call(amp, params=params, beta1=0.9):
        args.beta1 = beta1
        rc = lib.snb_adam_step_amp(params, params, FAKE, FAKE, C.byref(args), amp, 0, 1, None, None)
        return rc, lib.snb_last_error()

    assert call(None) == (-1, b"snb_adam_step_amp: null amp or count array")
    a, counts = amp_ctl(1, count_in=None)
    assert call(C.byref(a)) == (-1, b"snb_adam_step_amp: null amp or count array")
    a, counts = amp_ctl(1, out_offset=0)
    assert call(C.byref(a)) == (-1, b"snb_adam_step_amp: count_in and count_out overlap")
    a, counts = amp_ctl(1, base=0)
    rc, msg = call(C.byref(a))
    assert rc == -1 and b"step counts from 1 (got 0)" in msg
    a, counts = amp_ctl(1)
    rc, msg = call(C.byref(a), params=(C.c_void_p * 24)(*([256] * 23 + [None])))
    assert rc == -1 and b"parameter tensor 23 is null" in msg
    rc, msg = call(C.byref(a), beta1=1.0)
    assert rc == -1 and msg == b"snb_adam_step_amp: invalid hyper-parameters"


def test_optim_step_amp_argument_validation_without_gpu(lib):
    params = (C.c_void_p * 24)(*([256] * 24))
    a, counts = amp_ctl(24)

    def call(amp, rule=_lib.OPTIM_RADAM, grads=params, bufs=(FAKE, FAKE, FAKE), **hp):
        args = _lib.SnbOptimArgs(rule=rule, **dict(dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, alpha=0.5, k=6),
                                                    **hp))
        rc = lib.snb_optim_step_amp(params, grads, *bufs, C.byref(args), amp, 0, 1, None, None)
        return rc, lib.snb_last_error()

    assert call(None)[1] == b"snb_optim_step_amp: null amp or count array"
    overlap, _ = amp_ctl(24, out_offset=23)
    assert call(C.byref(overlap))[1] == b"snb_optim_step_amp: count_in and count_out overlap"
    rc, msg = call(C.byref(a), rule=_lib.OPTIM_ADAM)
    assert rc == -1 and b"unknown rule 3" in msg
    rc, msg = call(C.byref(a), rule=_lib.OPTIM_RANGER, bufs=(FAKE, FAKE, None))
    assert rc == -1 and b"null state buffer" in msg
    a.base[5] = 0
    rc, msg = call(C.byref(a))
    assert rc == -1 and b"step of tensor 5 counts from 1" in msg
    # a tensor without a gradient needs no base, nor does SGD without momentum; stopped at the hyper-parameter check
    rc, msg = call(C.byref(a), grads=(C.c_void_p * 24)(*([256] * 5 + [None] + [256] * 18)), lr=-1.0)
    assert rc == -1 and b"hyper-parameters" in msg
    rc, msg = call(C.byref(a), rule=_lib.OPTIM_SGD, momentum=0.0, lr=-1.0)
    assert rc == -1 and b"hyper-parameters" in msg


def test_optim_step_tensors_amp_argument_validation_without_gpu(lib):
    n = 3
    params = (C.c_void_p * n)(*([256] * n))
    numel = (C.c_int64 * n)(12288, 2097152, 8192)
    a, counts = amp_ctl(n)

    def call(amp, n=n, rule=_lib.OPTIM_ADAM, numel=numel, bufs=(FAKE, FAKE, FAKE), **hp):
        args = _lib.SnbOptimArgs(rule=rule, **dict(dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, alpha=0.5, k=6),
                                                    **hp))
        rc = lib.snb_optim_step_tensors_amp(n, params, params, numel, *bufs, C.byref(args), amp, None)
        return rc, lib.snb_last_error()

    assert call(None)[1] == b"snb_optim_step_tensors_amp: null amp or count array"
    assert call(C.byref(a), numel=None)[1] == b"snb_optim_step_tensors_amp: null table or args"
    for bad_n in (0, _lib.OPTIM_MAX_TENSORS + 1):
        rc, msg = call(C.byref(a), n=bad_n)
        assert rc == -1 and b"1 <= n <= 32" in msg, bad_n
    rc, msg = call(C.byref(a), bufs=(None, FAKE, None))
    assert rc == -1 and b"null state buffer" in msg
    a.base[2] = -1
    rc, msg = call(C.byref(a))
    assert rc == -1 and b"step of tensor 2 counts from 1 (got -1)" in msg
    a.base[2] = 1
    rc, msg = call(C.byref(a), beta2=1.0)
    assert rc == -1 and b"hyper-parameters" in msg


def test_gradscaler_native_flag_and_way_back():
    """All four classes declare GradScaler-native stepping; amp_scaling=False turns it off for one instance."""
    from sinnerf_b200.discriminator import Discriminator
    from sinnerf_b200.nerf import NeRF
    from sinnerf_b200.optim import FusedAdam, FusedRAdam, FusedRanger, FusedSGD, get_optimizer
    from tests.test_disc_optim_cpu import HParams
    for cls, kw in ((FusedAdam, {}), (FusedSGD, dict(lr=1e-3, momentum=0.9)), (FusedRAdam, {}), (FusedRanger, {})):
        for models in ([NeRF(use_new_activation=True)], [Discriminator(False, "color,cutout", imsize=64)]):
            assert cls(models, **kw)._step_supports_amp_scaling is True
            off = cls(models, amp_scaling=False, **kw)
            assert off._step_supports_amp_scaling is False
            assert cls._step_supports_amp_scaling is True
    for rule in ("sgd", "adam", "radam", "ranger"):
        assert get_optimizer(HParams(rule), [NeRF()])._step_supports_amp_scaling is True
