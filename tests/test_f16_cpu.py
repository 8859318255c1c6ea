"""CPU tests of the single-product fp16 precision mode ('f16', SNB_PREC_F16) and the 'autocast' precision policy:
the C ABI's constant and image size, the Python tables, the policy's resolution, and the oracle's fp16 restatement.
No compute is launched here."""
import os
import re

import pytest
import torch

from oracle import render_oracle as orc
from sinnerf_b200 import _lib, build, config
from tests import f16_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def header_modes():
    src = open(os.path.join(ROOT, "include", "sinnerf_b200.h")).read()
    return {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r"#define SNB_PREC_(\w+) (\d+)", src)}


def test_header_constants_and_tables_agree():
    assert header_modes() == {**_lib.PRECISIONS, **_lib.REDUCED_PRECISIONS}
    assert _lib.REDUCED_PRECISIONS == {"f16": 4}


def test_parity_table_is_unchanged():
    assert _lib.PRECISIONS == {"fp32": 0, "f16x3": 1, "bf16x3": 2, "bf16": 3}


def test_f16_image_is_the_bf16_image_size(lib):
    assert lib.snb_packed_weights_bytes(4) == lib.snb_packed_weights_bytes(3) > 0
    assert lib.snb_packed_weights_bytes(5) == 0


def test_c_abi_accepts_f16_and_rejects_the_next_id(lib):
    # an empty pass validates the mode and launches nothing
    assert lib.snb_field_forward(None, 4, None, None, 0, 64, 0, None, None) == 0
    assert lib.snb_mlp_forward(None, 4, None, 90, 0, 0, None, None) == 0
    assert lib.snb_field_forward(None, 5, None, None, 0, 64, 0, None, None) == -1
    assert b"unknown precision mode 5" in lib.snb_last_error()


def test_names():
    assert _lib.precision_id("f16") == 4
    assert _lib.precision_id("bf16") == 3
    for bad in ("fp16", "F16", "autocast", "f16x2"):
        with pytest.raises(ValueError, match="unknown precision"):
            _lib.precision_id(bad)
    with pytest.raises(ValueError, match="unknown precision"):
        config.set_precision("fp16")


def test_autocast_policy_resolution():
    assert config.resolve_precision("autocast", torch.float16) == _lib.precision_id("f16")
    assert config.resolve_precision("autocast", torch.bfloat16) == _lib.precision_id("bf16")
    assert config.resolve_precision("autocast", None) == _lib.precision_id("f16x3")
    # an explicit mode is not touched by the autocast state
    for mode in ("fp32", "f16x3", "bf16x3", "bf16", "f16"):
        for state in (torch.float16, torch.bfloat16, None):
            assert config.resolve_precision(mode, state) == _lib.precision_id(mode)
    assert config.resolve_precision(3, torch.float16) == 3


def test_set_precision_accepts_the_policy_and_the_default_is_unchanged():
    before = config.get_precision()
    try:
        config.set_precision("autocast")
        assert config.get_precision() == "autocast"
        assert config.resolve_precision(None, torch.float16) == 4
        assert config.resolve_precision(None, None) == 1
        config.set_precision("f16")
        assert config.resolve_precision(None, torch.bfloat16) == 4
    finally:
        config.set_precision(before)
    if "SINNERF_B200_PRECISION" not in os.environ:
        assert before == "f16x3"
        assert config.resolve_precision(None, torch.float16) == 1


def test_step_precision_follows_the_last_pass_under_the_policy():
    assert config.step_precision("autocast", 4) == 4
    assert config.step_precision("autocast", 3) == 3
    assert config.step_precision("autocast", None) == config.resolve_precision("autocast")
    assert config.step_precision("f16x3", 4) == 1       # an explicit mode re-packs its own image


def test_fp16_restatement_saturates():
    p = {"l.weight": torch.tensor([[1.0, -2.0]]), "l.bias": torch.tensor([0.5])}
    x = torch.tensor([[1e5, 3.0], [-7e4, 1.0]])
    got = f16_oracle.affine(p, "l", x)
    want = torch.tensor([[65504.0 - 6.0 + 0.5], [-65504.0 - 2.0 + 0.5]])
    assert torch.isfinite(got).all() and torch.equal(got, want)
    # plain fp16 rounding overflows; the oracle's own helper is back in place after the call
    assert torch.isinf(orc._affine(p, "l", x, torch.float16)).all()
    assert orc._round_st is f16_oracle._round_st
    # straight-through backward, like the rounding
    xr = x.clone().requires_grad_(True)
    f16_oracle.affine(p, "l", xr).sum().backward()
    assert torch.equal(xr.grad, p["l.weight"].expand(2, 2))


def test_bf16_restatement_is_unchanged():
    g = torch.Generator().manual_seed(0)
    p = orc.default_init_params(0)
    enc = orc.embed(torch.randn(64, 3, generator=g) * 3e4, orc.N_XYZ_FREQS)     # x itself far beyond fp16's range
    dirs = orc.embed(torch.randn(64, 3, generator=g), orc.N_DIR_FREQS)
    want = orc.field_mlp(p, enc, dirs, linear_dtype=torch.bfloat16, fold_bottleneck=True)
    with f16_oracle.fp16_saturation():
        got = orc.field_mlp(p, enc, dirs, linear_dtype=torch.bfloat16, fold_bottleneck=True)
    assert torch.equal(got, want)
    # the fp16 restatement of the same rows stays finite where unsaturated fp16 does not
    assert torch.isfinite(f16_oracle.field_mlp(p, enc, dirs)).all()
    assert not torch.isfinite(orc.field_mlp(p, enc, dirs, linear_dtype=torch.float16, fold_bottleneck=True)).all()
