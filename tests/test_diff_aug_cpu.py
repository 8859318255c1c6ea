"""CPU tests of the standalone DiffAugment (sinnerf_b200.discriminator.DiffAugment): the float64 oracle
(tests/diff_aug_oracle.py) against the reference's own models/diff_aug.py (tests/golden/diff_aug.npz), the
draw sequence against the reference's use of numpy's and torch's generators, the gate's identity return, the
KeyError of an unknown op and the C ABI's argument checks, none of which needs a device."""
import ctypes

import numpy as np
import pytest
import torch

from sinnerf_b200 import _lib
from sinnerf_b200 import discriminator as disc
from sinnerf_b200.discriminator import DiffAugment, diff_augment_draws
from tests import diff_aug_oracle as dao
from tests._common import load_npz

D64 = torch.float64
C_i64 = ctypes.c_int64


@pytest.fixture(scope="module")
def gold():
    return load_npz("diff_aug.npz")


def cases(gold):
    for i in range(int(gold["n_cases"])):
        pi, H, W, B, fire, np_seed, torch_seed, input_seed = (int(v) for v in gold[f"c{i}_meta"])
        yield i, str(gold["policies"][pi]), H, W, B, bool(fire), np_seed, torch_seed, input_seed


def golden_draws(gold, i, policy, B):
    """the recorded torch draws of case i grouped per op as diff_augment_draws returns them"""
    flat = [torch.from_numpy(gold[f"c{i}_draw{j}"]) for j in range(int(gold[f"c{i}_n_draws"]))]
    out = []
    for op in policy.split(","):
        n = 3 if op == "color" else 2
        out.append((op, tuple(flat[:n])))
        flat = flat[n:]
    assert not flat
    return out


def test_golden_covers_the_issue_grid(gold):
    seen = {(p, H, W, B, f) for _, p, H, W, B, f, *_ in cases(gold)}
    assert len(seen) == 7 * 4 * 2 * 2


def test_oracle_matches_reference(gold):
    for i, policy, H, W, B, fire, _, _, input_seed in cases(gold):
        if not fire:
            continue
        x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(input_seed)).double()
        y = dao.diff_augment(x, golden_draws(gold, i, policy, B))
        got = y.reshape(-1)[torch.from_numpy(gold[f"c{i}_idx"])]
        want = torch.from_numpy(gold[f"c{i}_out64"])
        sums = torch.from_numpy(gold[f"c{i}_sum64"])
        if "color" in policy:
            assert float((got - want).norm() / want.norm()) <= 1e-12, (policy, H, W, B)
            assert float((y.sum((2, 3)) - sums).norm() / sums.norm()) <= 1e-12, (policy, H, W, B)
        else:
            assert torch.equal(got, want), (policy, H, W, B)
            assert torch.allclose(y.sum((2, 3)), sums, rtol=1e-13, atol=0), (policy, H, W, B)
        # the reference's own fp32 run, for scale: fp32 rounding only
        assert torch.allclose(got, torch.from_numpy(gold[f"c{i}_out32"]).double(), rtol=1e-5, atol=1e-6)


def test_oracle_channels_last_and_general_c():
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 5, 9, 11, generator=g, dtype=D64)
    draws = [("cutout", (torch.tensor([3, 8]), torch.tensor([0, 10]))),
             ("translation", (torch.tensor([-1, 1]), torch.tensor([2, 0]))),
             ("color", (torch.rand(2, generator=g), torch.rand(2, generator=g), torch.rand(2, generator=g)))]
    nchw = dao.diff_augment(x, draws)
    nhwc = dao.diff_augment(x.permute(0, 2, 3, 1), draws, channels_first=False)
    assert nhwc.is_contiguous() and nhwc.shape == (2, 9, 11, 5)
    assert torch.equal(nhwc.permute(0, 3, 1, 2), nchw)
    # saturation's mean runs over the 5 channels, contrast's over channels, rows and columns of each image
    c0 = dao.diff_augment(x, draws[2:])
    rb, rs, rc = (t.view(2, 1, 1, 1) for t in draws[2][1])
    s = x + rb - 0.5
    s = (s - s.mean(1, keepdim=True)) * 2 * rs + s.mean(1, keepdim=True)
    want = (s - s.mean((1, 2, 3), keepdim=True)) * (rc + 0.5) + s.mean((1, 2, 3), keepdim=True)
    assert torch.allclose(c0, want, rtol=1e-14, atol=1e-14)


def test_draw_sequence_matches_reference(gold):
    for i, policy, H, W, B, fire, np_seed, torch_seed, _ in cases(gold):
        np.random.seed(np_seed)
        torch.manual_seed(torch_seed)
        draws = diff_augment_draws(policy, (B, 3, H, W), "cpu")
        assert (draws is not None) == fire
        if fire:
            for (op, got), (op2, want) in zip(draws, golden_draws(gold, i, policy, B)):
                assert op == op2
                for a, b in zip(got, want):
                    assert a.dtype == b.dtype and torch.equal(a, b), (policy, op)
        assert np.random.random() == float(gold[f"c{i}_after_np"])
        assert torch.equal(torch.rand(4), torch.from_numpy(gold[f"c{i}_after_torch"]))


def test_draw_augment_is_the_shared_helper():
    """the discriminator's draws: its own gate, then DiffAugment's gate, color and cutout draws"""
    for seed in range(40):
        np.random.seed(seed)
        torch.manual_seed(seed)
        got = disc.draw_augment("color,cutout", (2, 3, 16, 20), "cpu")
        nxt = (np.random.random(), torch.rand(2))
        np.random.seed(seed)
        torch.manual_seed(seed)
        want = None
        if np.random.random() > 0.5:
            d = diff_augment_draws("color,cutout", (2, 3, 16, 20), "cpu")
            want = None if d is None else d[0][1] + d[1][1]
        assert (got is None) == (want is None)
        if got is not None:
            assert all(torch.equal(a, b) for a, b in zip(got, want))
        assert nxt[0] == np.random.random() and torch.equal(nxt[1], torch.rand(2))


@pytest.fixture
def no_device_check(monkeypatch):
    """DiffAugment's Python layer on a CPU tensor: the device check stubbed, so that the paths that return before any
    kernel (the gate, an empty policy, an unknown op) run here"""
    monkeypatch.setattr(_lib, "require_device", lambda t, what: None)


def _seed(fire):
    for s in range(100):
        np.random.seed(s)
        if (np.random.random() >= 0.5) == fire:
            return s
    raise AssertionError


@pytest.mark.parametrize("policy", ["color,cutout", "translation", "", None])
def test_gate_returns_the_input_itself(no_device_check, policy):
    x = torch.rand(1, 3, 8, 8)
    np.random.seed(_seed(False))
    torch.manual_seed(0)
    assert DiffAugment(x, policy) is x
    after = torch.rand(2)
    torch.manual_seed(0)
    assert torch.equal(after, torch.rand(2))   # no torch draw made


@pytest.mark.parametrize("policy", ["", None])
def test_empty_policy_returns_the_input_itself(no_device_check, policy):
    x = torch.rand(1, 3, 8, 8)
    np.random.seed(_seed(True))
    assert DiffAugment(x, policy) is x


def test_unknown_op_raises_key_error_after_the_draws_before_it(no_device_check):
    x = torch.rand(2, 3, 8, 8)
    np.random.seed(_seed(True))
    torch.manual_seed(3)
    with pytest.raises(KeyError):
        DiffAugment(x, "color,zoom")
    after = torch.rand(1)
    torch.manual_seed(3)
    for _ in range(3):
        torch.rand(2, 1, 1, 1)
    assert torch.equal(after, torch.rand(1))


def test_input_checks_before_any_draw():
    state = np.random.get_state()[1].copy()
    with pytest.raises(RuntimeError):
        DiffAugment(torch.rand(1, 3, 8, 8))                       # CPU tensor: no CPU path
    with pytest.raises(ValueError):
        DiffAugment(torch.rand(3, 8, 8))
    with pytest.raises(TypeError):
        DiffAugment(np.zeros((1, 3, 8, 8), np.float32))
    assert np.array_equal(np.random.get_state()[1], state)


def test_cabi_argument_checks():
    lib = _lib.load()
    st = (C_i64 * 4)(1, 1, 1, 1)
    ops = (ctypes.c_int * 2)(0, 2)
    none = _lib.SnbDiffAugDraws()
    fwd, bwd = lib.snb_diff_augment_forward, lib.snb_diff_augment_backward
    assert fwd(ops, 9, ctypes.byref(none), 16, st, 1, 3, 8, 8, 16, st, 16, None) == -1
    assert b"n_ops" in lib.snb_last_error()
    assert fwd(ops, 2, ctypes.byref(none), 16, st, 1, 3, 8, 8, 16, st, 16, None) == -1
    assert b"color" in lib.snb_last_error()
    bad = (ctypes.c_int * 1)(7)
    assert bwd(bad, 1, ctypes.byref(none), 16, st, 1, 3, 8, 8, 16, st, 16, None) == -1
    assert b"unknown op" in lib.snb_last_error()
    d = _lib.SnbDiffAugDraws(16, 16, 16, None, None, 16, 16)
    assert fwd(ops, 2, ctypes.byref(d), 16, st, 0, 3, 8, 8, 16, st, 16, None) == -1
    assert fwd(ops, 2, ctypes.byref(d), None, st, 1, 3, 8, 8, 16, st, 16, None) == -1
    assert fwd(ops, 2, ctypes.byref(d), 16, st, 1, 3, 8, 8, 16, st, None, None) == -1
    assert b"workspace" in lib.snb_last_error()
    tr = (ctypes.c_int * 1)(1)
    assert bwd(tr, 1, ctypes.byref(d), 16, st, 1, 3, 8, 8, 16, st, 16, None) == -1
    assert b"translation" in lib.snb_last_error()
