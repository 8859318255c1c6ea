"""CPU tests of tests/optim_emulation.py: the exact FMA against rational arithmetic, the host scalars against the
optimiser oracle, the emulation against float64 on every input set tests/test_gpu_optim_stages.py uses, and every
checker on the CPU stand-in -- passing when it is faithful, failing on the defect aimed at it.  The last test restates
the bars the older optimiser tests hold the kernels to (3e-7 max |diff| / max |p| per tensor, rel-L2 1e-6 on state,
>= 90 % of parameters bit-equal) and shows that the subtle defects pass them."""
import math
import sys
from fractions import Fraction

import numpy as np
import pytest

from oracle import optim_oracle
from tests import optim_emulation as emu

f32 = np.float32


# ------------------------------------------------------------------------------------------------ exact FMA
def round_f32(x: Fraction, sign_if_zero=1.0):
    """A rational rounded to the nearest float32, ties to even, with overflow to +-inf."""
    if x == 0:
        return f32(math.copysign(0.0, sign_if_zero))
    s = -1 if x < 0 else 1
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)
    n, r = divmod(a, q)
    if r * 2 > q or (r * 2 == q and n % 2 == 1):
        n += 1
    v = n * q
    if v >= Fraction(2) ** 128:
        return f32(s * np.inf)
    return f32(s * float(v))


def fma_exact(a, b, c):
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    # an exact zero keeps IEEE's sign: -0 only when both addends are -0
    sign = -1.0 if (math.copysign(1, float(a) * float(b)) < 0 and math.copysign(1, float(c)) < 0) else 1.0
    return round_f32(x, sign)


def edge_triples():
    one = 1 + 2.0 ** -12
    mid = 1 + 2.0 ** -11 + 2.0 ** -24            # one * one: exactly between two float32
    return [
        (one, one, 0.0),                          # tie, exact: to even
        (one, one, 2.0 ** -60), (one, one, -2.0 ** -60),    # tie broken by a term float64 loses
        (one, -one, -2.0 ** -70), (-one, one, 2.0 ** -70),
        (1 + 2.0 ** -23, 1 + 2.0 ** -23, -1.0),   # cancellation: 2^-22 + 2^-46
        (one, one, -(1 + 2.0 ** -11)),            # cancellation to 2^-24 exactly
        (2.0 ** -70, 2.0 ** -70, 0.0), (2.0 ** -75, 3.0 * 2.0 ** -75, 1e-45), (1e-45, 0.5, 0.0),   # subnormals
        (1e-45, 0.5, 1e-45), (-1e-45, 0.5, 0.0), (2.0 ** -63, 2.0 ** -63, -2.0 ** -126),
        (3.4e38, 2.0, -3.4e38), (3.4e38, 1.0, 3.4e38), (2.0 ** 64, 2.0 ** 64, 0.0), (-2.0 ** 64, 2.0 ** 64, 1.0),
        (float(np.finfo(f32).max), 1.0, 2.0 ** 103), (float(np.finfo(f32).max), 1.0, 2.0 ** 103 - 2.0 ** 79),
        (0.0, 5.0, -0.0), (-0.0, 5.0, -0.0), (mid, 1.0, 0.0),
    ]


def test_fma32_matches_rational_arithmetic():
    rng = np.random.default_rng(0)
    n = 20000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, n))).astype(f32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, n))).astype(f32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * 2.0 ** -20)).astype(f32)   # heavy cancellation
    c[::3] = (rng.standard_normal(n) * np.exp2(rng.integers(-90, 90, n))).astype(f32)[::3]
    # ties: products of 13-bit significands land on float32 midpoints
    k = np.arange(0, n, 7)
    a[k] = ((rng.integers(1 << 12, 1 << 13, k.size) | 1) * 2.0 ** -12).astype(f32)
    b[k] = ((rng.integers(1 << 12, 1 << 13, k.size) | 1) * 2.0 ** -12).astype(f32)
    c[k] = np.where(rng.random(k.size) < 0.5, 0, rng.choice([-1, 1], k.size) * 2.0 ** -70).astype(f32)
    triples = list(zip(a, b, c)) + [tuple(f32(x) for x in t) for t in edge_triples()]
    A, B, Cc = (np.array(x, f32) for x in zip(*triples))
    got = emu.fma32(A, B, Cc)
    for i, (x, y, z) in enumerate(triples):
        want = fma_exact(x, y, z)
        assert got[i].view(np.uint32) == want.view(np.uint32), (i, x, y, z, got[i], want)


# ------------------------------------------------------------------------------------------------ host scalars
@pytest.mark.parametrize("beta2", [0.9, 0.99, 0.999])
@pytest.mark.parametrize("rule", ["radam", "ranger"])
def test_scalars_equal_the_oracle(rule, beta2):
    """(adaptive, step_size) exactly as oracle/optim_oracle.rectification forms them, and step_lr its float32 cast."""
    a = emu.Args(rule, lr=1e-3, beta1=0.95 if rule == "ranger" else 0.9, beta2=beta2)
    test = (lambda n: n >= 5) if rule == "radam" else (lambda n: n > a.n_sma_threshold)
    for step in list(range(1, 21)) + [10 ** 4, 10 ** 6]:
        want = optim_oracle.rectification(step, a.beta1, beta2, test)
        assert emu.rectification(a, step) == want, (step, emu.rectification(a, step), want)
        step_lr, flags = emu.rule_scalars(a, step)
        assert step_lr == f32(-want[1] * a.lr) and bool(flags & emu.K_ADAPTIVE) == want[0], step
    assert any(emu.rectification(a, s)[0] for s in range(1, 21)) or beta2 == 0.999


def test_ranger_threshold_edge_is_exact():
    """scenario_counts sets Ranger's threshold to N_sma at its crossing count: > and >= differ there."""
    for beta2 in (0.9, 0.99, 0.999):
        a = emu.Args("ranger", beta2=beta2)
        c = emu.first_adaptive(a)
        a = a.with_(n_sma_threshold=emu.n_sma(a, c))
        assert not emu.rectification(a, c)[0] and emu.rectification(a, c, swap=True)[0]


# ------------------------------------------------------------------------------------------------ checkers
def scenarios():
    """Every scenario test_gpu_optim_stages.py runs, as (name, function, args)."""
    out = []
    for rule in emu.RULES:
        for wd in (0.0, 1e-2):
            out.append((f"table-{rule}-{wd}", emu.scenario_table, (rule, wd)))
        out.append((f"table32-{rule}", emu.scenario_table32, (rule,)))
        for beta2 in (0.9, 0.99, 0.999):
            out.append((f"counts-{rule}-{beta2}", emu.scenario_counts, (rule, beta2)))
        for scale in (1.0, 2.0 ** 16, 3000.0):
            out.append((f"amp-{rule}-{scale}", emu.scenario_amp, (rule, scale)))
        out.append((f"nonfinite-{rule}", emu.scenario_nonfinite, (rule,)))
        out.append((f"nerf-{rule}", emu.scenario_nerf, (rule,)))
    for alpha in (0.0, 0.5, 1.0):
        for k in (1, 5, 6):
            out.append((f"ranger-{alpha}-{k}", emu.scenario_ranger, (alpha, k)))
    for momentum in (0.0, 0.9):
        for wd in (0.0, 1e-2):
            out.append((f"sgd-{momentum}-{wd}", emu.scenario_sgd, (momentum, wd)))
    return out


@pytest.mark.parametrize("name,fn,args", scenarios(), ids=[s[0] for s in scenarios()])
def test_faithful_stand_in_passes(name, fn, args):
    """The emulation stays within its float64 bounds on every input set of the GPU test, and the faithful stand-in
    passes every checker."""
    fn(emu.StandIn(), *args)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print(f"\nemulation stages, largest |got - float64| / (u * terms + 2^-149): {emu.measured_report()}",
          file=sys.stderr)


# The checker aimed at each defect, with the scenario that exposes it.
AIMED = {
    "state_offset": (emu.scenario_table, ("radam", 1e-2)),
    "last_skipped": (emu.scenario_table32, ("adam",)),
    "sweep2_dropped": (emu.scenario_table, ("sgd", 0.0)),
    "count_minus_1": (emu.scenario_counts, ("adam", 0.999)),
    "stale_slot": (emu.scenario_amp, ("radam", 2.0 ** 16)),
    "threshold_swap": (emu.scenario_counts, ("ranger", 0.99)),
    "ranger_global_step": (emu.scenario_ranger, (0.5, 5)),
    "slow_every_step": (emu.scenario_ranger, (0.5, 6)),
    "gradless_state": (emu.scenario_table32, ("radam",)),
    "found_inf_counts": (emu.scenario_amp, ("sgd", 3000.0)),
    "no_writeback": (emu.scenario_amp, ("adam", 3000.0)),
    "always_writeback": (emu.scenario_amp, ("adam", 1.0)),
    "v_alpha_g_g": (emu.scenario_counts, ("adam", 0.999)),
}
assert set(AIMED) == set(emu.DEFECTS)


@pytest.mark.parametrize("defect", emu.DEFECTS)
def test_checker_catches_defect(defect):
    fn, args = AIMED[defect]
    with pytest.raises(AssertionError) as info:
        fn(emu.StandIn(defect=defect), *args)
    print(f"{defect}: {str(info.value).splitlines()[0]}", file=sys.stderr)


# ------------------------------------------------------------------------------------------------ the older bars
def realistic_step(rule, numel, seed):
    """Inputs of a training step's magnitude (parameters ~0.1, gradients ~1e-2), no edge values."""
    rng = np.random.default_rng(seed)
    a = emu.Args(rule, lr=1e-3, weight_decay=1e-2, momentum=0.9 if rule == "sgd" else 0.0, k=6)
    params = [(rng.standard_normal(n) * 0.1).astype(f32) for n in numel]
    grads = [(rng.standard_normal(n) * 1e-2).astype(f32) for n in numel]
    z = np.zeros(int(sum(numel)), f32)
    return a, emu.Step(params, grads, z.copy(), z.copy(), z.copy())


def old_bars(ref: emu.Step, got: emu.Step):
    """The bars of test_gpu_optim.py / test_gpu_disc_optim.py: True when `got` passes them against `ref`."""
    exact = total = 0
    for pa, pb in zip(ref.params, got.params):
        if np.abs(pa.astype(np.float64) - pb).max() > 3e-7 * np.abs(pa).max():
            return False
        exact += int((pa == pb).sum())
        total += pa.size
    for x, y in ((ref.exp_avg, got.exp_avg), (ref.exp_avg_sq, got.exp_avg_sq)):
        d = np.linalg.norm(x.astype(np.float64) - y)
        if d > 1e-6 * max(np.linalg.norm(x.astype(np.float64)), 1e-30):
            return False
    return exact >= 0.9 * total


# a defect that a run of realistic steps leaves inside the older bars (and that the checkers above catch)
SUBTLE = {"v_alpha_g_g": "adam"}


@pytest.mark.parametrize("defect", sorted(SUBTLE))
def test_old_bars_miss_subtle_defects(defect):
    """14 realistic steps of the faithful stand-in and of the defective one, compared with the older bars."""
    rule = SUBTLE[defect]
    numel = [256 * 63, 256, 1, 3, 256 * 283]
    a, ref = realistic_step(rule, numel, 0)
    got = ref.copy()
    rng = np.random.default_rng(1)
    for step in range(1, 15):
        counts = np.full(len(numel), step)
        emu.StandIn().step_tensors(a, ref, counts)
        emu.StandIn(defect=defect).step_tensors(a, got, counts)
        for g1, g2 in zip(ref.grads, got.grads):
            g1[:] = (rng.standard_normal(g1.size) * 1e-2).astype(f32)
            g2[:] = g1
    differs = any(not np.array_equal(x, y) for x, y in zip(ref.params + [ref.exp_avg, ref.exp_avg_sq],
                                                           got.params + [got.exp_avg, got.exp_avg_sq]))
    passes = old_bars(ref, got)
    print(f"{defect}: results differ {differs}, older bars pass {passes}", file=sys.stderr)
    assert differs and passes
