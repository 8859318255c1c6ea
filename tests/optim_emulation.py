"""References for the fused optimiser steps (sinnerf_b200/csrc/optim.cu) and a CPU stand-in for them.

Three things, none of which imports the library or reads anything outside the tree:

* float32 emulation, operation for operation, of the kernels' element arithmetic (`adam32`: adam_update;
  `rule32`: rule_update for SGD / RAdam / Ranger; `unscale32`: the GradScaler unscale of the _amp forms) with the
  host scalars formed as optim.cu forms them, in Python doubles cast to float32 (`adam_scalars`, `rule_scalars`,
  `consts`).  The kernels use only explicitly rounded multiplies, adds, divides and square roots, and fmaf, so numpy
  float32 plus an exact fused multiply-add (`fma32`) reproduces them bit for bit.  `emulate_*` run one whole entry
  point of include/sinnerf_b200.h.
* float64 truth of each stage from the kernel's own float32 inputs to that stage (`truth64`), with the sum of the
  absolute values of the stage's terms, which normalises the error, and the bound that follows from counting the
  stage's roundings (`BOUND_K`).
* `StandIn`: the four entry points on numpy arrays, as tests/test_gpu_optim_stages.py's `Lib` drives the C ABI, with
  the kernels' grid-stride mapping written out so that `StandIn(defect=...)` can plant one defect (names in DEFECTS).
  The checker (`check_launch`) and the scenarios built on it (`scenario_*`) take an implementation, so
  tests/test_optim_emulation_cpu.py shows each one passing on the faithful stand-in and failing on the defect it is
  there for.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import numpy as np

f32 = np.float32
U = 2.0 ** -24                   # unit roundoff of float32
TINY = 2.0 ** -149               # smallest float32 subnormal: absolute rounding error below the normal range
FLT_MAX = float(np.finfo(f32).max)
OVF_MID = 2.0 ** 128 - 2.0 ** 103  # midpoint between FLT_MAX and 2^128: the overflow threshold of round-to-nearest
SENTINEL = np.array([0x7FA5A5A5], np.uint32).view(f32)[0]   # a signalling-NaN payload no arithmetic produces
WINDOW = 8                        # SNB_OPTIM_WINDOW
MAX_TENSORS = 32                  # SNB_OPTIM_MAX_TENSORS
BLOCK = 256
K_FIRST, K_ADAPTIVE, K_SYNC = 1, 2, 4
RULES = ("adam", "sgd", "radam", "ranger")
RULE_ID = dict(sgd=0, radam=1, ranger=2, adam=3)     # SNB_OPTIM_*

# element counts of the 24 NeRF tensors in state-dict order (common.cuh param_numel)
NERF_NUMEL = [256 * 63, 256] + [256 * 256, 256] * 3 + [256 * 319, 256] + [256 * 256, 256] * 4 + \
    [128 * 283, 128, 256, 1, 384, 3]
assert len(NERF_NUMEL) == 24 and sum(NERF_NUMEL) == 595844

DEFECTS = (
    "state_offset",        # tensor t >= 1 reads and writes its state one entry early
    "last_skipped",        # the last element of every tensor is not updated
    "sweep2_dropped",      # the grid-stride loop's second sweep is skipped
    "count_minus_1",       # step-dependent scalars of count t - 1
    "stale_slot",          # _amp: the window entry of the previous count (j - 1)
    "threshold_swap",      # RAdam N_sma >= 5 -> > 5; Ranger N_sma > threshold -> >=
    "ranger_global_step",  # Ranger syncs on the largest count of the launch, not the tensor's own
    "slow_every_step",     # Ranger writes slow_buffer on non-sync steps too
    "gradless_state",      # a tensor without a gradient has its state regions zeroed
    "found_inf_counts",    # _amp: the counts advance on a skipped step
    "no_writeback",        # _amp: the unscaled gradient is not stored back
    "always_writeback",    # _amp: the gradient is stored back at scale 1 too (g * 1 quiets a signalling NaN)
    "v_alpha_g_g",         # v = fma((1 - beta2) * g, g, v) instead of ATen's fma(1 - beta2, g * g, v)
)


@dataclass(frozen=True)
class Args:
    """SnbOptimArgs / SnbAdamArgs as Python doubles, the rule named."""
    rule: str
    lr: float = 1e-3
    weight_decay: float = 0.0
    momentum: float = 0.0
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    n_sma_threshold: float = 5.0
    alpha: float = 0.5
    k: int = 6

    def with_(self, **kw):
        return replace(self, **kw)


# ------------------------------------------------------------------------------------------------ exact fp32 FMA
def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays, rounded once.  a * b is exact in float64 (two 24-bit significands); s = ab + c
    is rounded to float64 and TwoSum gives its error e exactly.  Rounding s to float32 is then the correctly rounded
    result unless s is exactly a float32 midpoint (a float32 rounding boundary strictly between s and ab + c would be
    a float64 closer to ab + c than s), and there the sign of e says which neighbour the exact sum is nearer."""
    a, b, c = (np.asarray(x, f32).astype(np.float64) for x in (a, b, c))
    with np.errstate(all="ignore"):
        ab = a * b
        s = ab + c
        bp = s - ab
        ap = s - bp
        e = (ab - ap) + (c - bp)
        r = s.astype(f32)
        r64 = r.astype(np.float64)
        fin = np.isfinite(s) & np.isfinite(e)
        n = np.nextafter(r, np.where(s > r64, f32(np.inf), f32(-np.inf)).astype(f32))
        n64 = n.astype(np.float64)
        tie = fin & np.isfinite(r64) & (r64 != s) & (2 * s == r64 + n64)
        r = np.where(tie & (e != 0) & ((e > 0) == (n64 > r64)), n, r)
        # s exactly at the overflow midpoint: round-half-even gives inf; the exact sum may lie below it
        below = fin & (np.abs(s) == OVF_MID) & (e != 0) & ((e > 0) != (s > 0))
        r = np.where(below, np.copysign(f32(FLT_MAX), s).astype(f32), r)
    return np.asarray(r, f32)


# ------------------------------------------------------------------------------------------------ host scalars
def adam_scalars(a: Args, step: int):
    """optim.cu adam_bias_scalars: (float)(-(lr / (1 - beta1^t))), (float)(1.0 / pow(1 - beta2^t, 0.5))."""
    bc1 = 1.0 - math.pow(a.beta1, float(step))
    bc2 = 1.0 - math.pow(a.beta2, float(step))
    return f32(-(a.lr / bc1)), f32(1.0 / math.pow(bc2, 0.5))


def rectification(a: Args, step: int, swap=False):
    """(adaptive, step_size) of RAdam / Ranger at the tensor's count `step`, optim.cu rule_tensor_scalars' double
    arithmetic in the reference's expression order.  swap: the comparison with the other strictness."""
    beta2_t = math.pow(a.beta2, float(step))
    n_sma_max = 2 / (1 - a.beta2) - 1
    n_sma = n_sma_max - 2 * step * beta2_t / (1 - beta2_t)
    if a.rule == "radam":
        adaptive = n_sma > 5 if swap else n_sma >= 5
    else:
        adaptive = n_sma >= a.n_sma_threshold if swap else n_sma > a.n_sma_threshold
    bc1 = 1 - math.pow(a.beta1, float(step))
    if adaptive:
        return True, math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_sma_max - 4) * (n_sma - 2) / n_sma * n_sma_max /
                               (n_sma_max - 2)) / bc1
    return False, 1.0 / bc1


def n_sma(a: Args, step: int) -> float:
    beta2_t = math.pow(a.beta2, float(step))
    n_sma_max = 2 / (1 - a.beta2) - 1
    return n_sma_max - 2 * step * beta2_t / (1 - beta2_t)


def rule_scalars(a: Args, step: int, sync_step=None, swap=False):
    """optim.cu rule_tensor_scalars: (float)(-step_size * lr) and kFirst | kAdaptive | kSync at the tensor's count.
    sync_step: the count the Ranger sync is decided on (the tensor's own unless a defect says otherwise)."""
    if a.rule == "sgd":
        return f32(0.0), (K_FIRST if step == 1 else 0)
    adaptive, step_size = rectification(a, step, swap)
    sync = a.rule == "ranger" and (step if sync_step is None else sync_step) % a.k == 0
    return f32(-step_size * a.lr), ((K_ADAPTIVE if adaptive else 0) | (K_FIRST if step == 1 else 0) |
                                    (K_SYNC if sync else 0))


@dataclass(frozen=True)
class Consts:
    lr_neg: np.float32
    decay: np.float32
    momentum: np.float32
    beta1: np.float32
    beta1_w: np.float32
    beta2: np.float32
    beta2_w: np.float32
    eps: np.float32
    alpha: np.float32


def consts(a: Args) -> Consts:
    """optim.cu rule_consts (Adam's launch passes the same casts)."""
    z = f32(0.0)
    if a.rule == "sgd":
        return Consts(f32(-a.lr), f32(a.weight_decay), f32(a.momentum), z, z, z, z, z, z)
    decay = f32(a.weight_decay) if a.rule == "adam" else f32(-a.weight_decay * a.lr)
    return Consts(z, decay, z, f32(a.beta1), f32(1.0 - a.beta1), f32(a.beta2), f32(1.0 - a.beta2), f32(a.eps),
                  f32(a.alpha))


# ------------------------------------------------------------------------------------------------ element arithmetic
def adam32(p, g, m, v, c: Consts, lr_neg_step, inv_bc2_sqrt, defect=None):
    """optim.cu adam_update on float32 arrays: (p', m', v')."""
    with np.errstate(all="ignore"):
        if c.decay != 0:
            g = fma32(c.decay, p, g)
        m = fma32(c.beta1_w, g - m, m)
        v = v * c.beta2
        v = fma32(c.beta2_w * g, g, v) if defect == "v_alpha_g_g" else fma32(c.beta2_w, g * g, v)
        den = np.sqrt(v) * inv_bc2_sqrt + c.eps
        return fma32(lr_neg_step, m / den, p), m, v


def rule32(rule, p, g, m, v, slow, c: Consts, flags, step_lr, defect=None):
    """optim.cu rule_update<RULE> on float32 arrays: (p', m', v', slow') -- for SGD m is the momentum buffer; state a
    rule does not keep comes back as given."""
    with np.errstate(all="ignore"):
        if rule == "sgd":
            if c.decay != 0:
                g = fma32(c.decay, p, g)
            if c.momentum != 0:
                if not flags & K_FIRST:
                    g = m * c.momentum + g
                m = g
            return fma32(c.lr_neg, g, p), m, v, slow
        v = v * c.beta2
        v = fma32(c.beta2_w * g, g, v) if defect == "v_alpha_g_g" else fma32(c.beta2_w, g * g, v)
        m = m * c.beta1
        m = fma32(c.beta1_w, g, m)
        s = (p.copy() if flags & K_FIRST else slow) if rule == "ranger" else None
        w = p
        if c.decay != 0:
            w = fma32(c.decay, w, w)
        if flags & K_ADAPTIVE:
            w = fma32(step_lr, m / (np.sqrt(v) + c.eps), w)
        else:
            w = fma32(step_lr, m, w)
        if rule == "ranger":
            if flags & K_SYNC:
                s = fma32(c.alpha, w - s, s)
                w = s
            if flags & (K_FIRST | K_SYNC) or defect == "slow_every_step":
                slow = w if defect == "slow_every_step" and not flags & (K_FIRST | K_SYNC) else s
        return w, m, v, slow


def inv_scale32(scale):
    """optim.cu amp_inv_scale: (float)(1.0 / (double)*scale); 1 when there is no scale."""
    return f32(1.0) if scale is None else f32(1.0 / float(f32(scale)))


def unscale32(g, inv):
    """optim.cu amp_unscale: g * inv, rounded on its own, unless inv == 1 (then g is neither changed nor written)."""
    return g if inv == 1 else (g * inv).astype(f32)


# ------------------------------------------------------------------------------------------------ whole entry points
@dataclass
class Step:
    """The inputs one entry point reads and writes, as numpy arrays (flat float32 state buffers; None where the caller
    passes NULL).  Entry points step it in place."""
    params: list
    grads: list
    exp_avg: np.ndarray | None
    exp_avg_sq: np.ndarray | None
    slow: np.ndarray | None

    def copy(self):
        cp = lambda x: None if x is None else x.copy()      # noqa: E731
        return Step([cp(p) for p in self.params], [cp(g) for g in self.grads], cp(self.exp_avg), cp(self.exp_avg_sq),
                    cp(self.slow))


def offsets(numel):
    return np.concatenate([[0], np.cumsum(numel)[:-1]]).astype(np.int64)


def _grid(form, sm_count):
    return (2 if form.startswith("nerf") else 4) * sm_count


def _walk(form, a: Args, st: Step, counts, defect=None, sm_count=132, amp=None):
    """One launch of `form` (tensors | tensors_amp | nerf | nerf_amp) over st, in place.  counts: per tensor, the count
    the scalars are formed at (None where the tensor has no gradient or keeps no count).  amp: (inv, skip) or None.
    The grid-stride mapping is written out so that the mapping defects can be planted."""
    c = consts(a)
    numel = [p.size for p in st.params]
    off = offsets(numel)
    grid = _grid(form, sm_count)
    inv, skip = amp if amp is not None else (f32(1.0), False)
    live_counts = [x for x in counts if x is not None]
    top = max(live_counts) if live_counts else None
    for t, (p, g) in enumerate(zip(st.params, st.grads)):
        n = p.size
        live = np.ones(n, bool)
        if defect == "last_skipped":
            live[-1] = False
        if defect == "sweep2_dropped":
            live[grid * BLOCK:2 * grid * BLOCK] = False
        if g is None:
            if defect == "gradless_state":
                for buf in (st.exp_avg, st.exp_avg_sq):
                    if buf is not None:
                        buf[off[t]:off[t] + n] = 0
            continue
        gu = unscale32(g, inv) if amp is not None else g
        if amp is not None and defect == "always_writeback":
            gu = (g * inv).astype(f32)
        if amp is not None and defect != "no_writeback" and gu is not g:
            g[live] = gu[live]
        if skip:
            continue
        o = off[t] - (1 if defect == "state_offset" and t >= 1 else 0)
        sl = slice(o, o + n)
        count = counts[t]
        if count is not None and defect in ("count_minus_1", "stale_slot") and count > 1:
            count -= 1
        m = st.exp_avg[sl] if st.exp_avg is not None else None
        v = st.exp_avg_sq[sl] if st.exp_avg_sq is not None else None
        s = st.slow[sl] if st.slow is not None else None
        if a.rule == "adam":
            lr_neg_step, inv_bc2 = adam_scalars(a, count)
            w, m2, v2 = adam32(p, gu, m, v, c, lr_neg_step, inv_bc2, defect)
            s2 = s
        else:
            if count is None:                            # SGD without momentum keeps no count
                step_lr, flags = f32(0.0), 0
            else:
                step_lr, flags = rule_scalars(a, count, top if defect == "ranger_global_step" else None,
                                              defect == "threshold_swap")
            w, m2, v2, s2 = rule32(a.rule, p, gu, m, v, s, c, flags, step_lr, defect)
        p[live] = w[live]
        for buf, new in ((m, m2), (v, v2), (s, s2)):
            if buf is not None and new is not buf:
                buf[live] = new[live]


def _amp_counts(form, a: Args, st: Step, count_in, base, skip, defect):
    """(counts the scalars are formed at, count_out) of an _amp launch; asserts the window the header requires."""
    count_in = np.asarray(count_in, np.int64)
    base = np.asarray(base, np.int64)
    if form == "nerf_amp" and a.rule == "adam":
        adv = np.array([True])
    else:
        adv = np.array([g is not None and (a.rule != "sgd" or a.momentum != 0) for g in st.grads])
    counts = []
    for t in range(len(st.grads)):
        i = 0 if adv.size == 1 else t
        if st.grads[t] is None or not adv[i]:
            counts.append(None)
            continue
        j = int(count_in[i] + 1 - base[i])
        assert 0 <= j < WINDOW, f"tensor {t}: count {count_in[i]} + 1 outside the window at base {base[i]}"
        counts.append(int(base[i]) + j)
    step = adv & (not skip or defect == "found_inf_counts")
    return counts, (count_in + step).astype(np.int32)


def emulate_tensors(a: Args, st: Step, step, defect=None, sm_count=132):
    """snb_optim_step_tensors (any rule; step: per tensor)."""
    counts = [None if g is None or (a.rule == "sgd" and a.momentum == 0) else int(step[t])
              for t, g in enumerate(st.grads)]
    _walk("tensors", a, st, counts, defect, sm_count)


def emulate_nerf(a: Args, st: Step, step, defect=None, sm_count=132):
    """snb_adam_step (step: the one count) and snb_optim_step (step: per tensor)."""
    if a.rule == "adam":
        counts = [None if g is None else int(step) for g in st.grads]
    else:
        counts = [None if g is None or (a.rule == "sgd" and a.momentum == 0) else int(step[t])
                  for t, g in enumerate(st.grads)]
    _walk("nerf", a, st, counts, defect, sm_count)


def emulate_amp(form, a: Args, st: Step, scale, found_inf, count_in, base, defect=None, sm_count=132):
    """snb_optim_step_tensors_amp (form 'tensors_amp') or snb_adam_step_amp / snb_optim_step_amp ('nerf_amp'):
    returns count_out."""
    skip = found_inf is not None and found_inf != 0
    counts, count_out = _amp_counts(form, a, st, count_in, base, skip, defect)
    _walk(form, a, st, counts, defect, sm_count, amp=(inv_scale32(scale), skip))
    return count_out


class StandIn:
    """The four entry points on numpy arrays, faithful or with one planted defect (DEFECTS).  Same methods as the GPU
    test's `Lib`."""

    def __init__(self, defect=None, sm_count=132):
        assert defect is None or defect in DEFECTS, defect
        self.defect, self.sm_count = defect, sm_count

    def step_tensors(self, a, st, step):
        emulate_tensors(a, st, step, self.defect, self.sm_count)

    def step_nerf(self, a, st, step, precision=None):
        emulate_nerf(a, st, step, self.defect, self.sm_count)

    def step_tensors_amp(self, a, st, scale, found_inf, count_in, base):
        return emulate_amp("tensors_amp", a, st, scale, found_inf, count_in, base, self.defect, self.sm_count)

    def step_nerf_amp(self, a, st, scale, found_inf, count_in, base, precision=None):
        return emulate_amp("nerf_amp", a, st, scale, found_inf, count_in, base, self.defect, self.sm_count)


# ------------------------------------------------------------------------------------------------ float64 truth
# Bounds, in units of u = 2^-24, on |got - f64| / (sum of |terms|) of each stage: one u per rounding the stage makes
# (each rounding errs by at most u times its result, and the sum of the stage's absolute terms bounds every
# intermediate result times whatever later multiplies it, first order), the host-scalar casts counted with them.
#   grad (AMP unscale)   g * inv:                  inv cast, multiply                                             = 2
#   adam exp_avg         m + b1w (g + wd p - m):   wd cast, fma, b1w cast, subtract, fma                          = 5
#   adam exp_avg_sq      b2 v + b2w (g + wd p)^2:  b2 cast, multiply, b2w cast, g * g, fma; gr twice (the
#                                                  decayed gradient's fma and wd cast enter squared)              = 9
#   adam param           p - s m / den:            den = sqrt(v) inv + eps: sqrt, multiply, add, eps cast, and
#                                                  inv = (float)(1 / sqrt(bc2)): one; divide; lr / bc1 cast; fma  = 8
#   sgd exp_avg          mom b + g + wd p:         wd cast, fma, momentum cast, multiply, add                     = 5
#   sgd param            p - lr (g + wd p) | p - lr b:   wd cast, fma, lr cast, fma                               = 4
#   radam exp_avg        b1 m + b1w g:             b1 cast, multiply, b1w cast, fma                               = 4
#   radam exp_avg_sq     b2 v + b2w g^2:           b2 cast, multiply, b2w cast, g * g, fma                        = 5
#   radam param          p - wd lr p + s q:        -wd * lr (double) and its cast, fma; q = m / (sqrt(v) + eps):
#                                                  sqrt, eps cast, add, divide; step_size * lr cast; fma          = 10
#   ranger param (sync)  slow + a (w - slow):      the param stage's 10, a cast, subtract, fma                    = 13
# Below the normal range each rounding errs by up to half a subnormal in absolute terms; every multiplier that
# follows a rounding here is at most 1 in magnitude, so k * 2^-149 absolute is added to each bound.
BOUND_K = {
    "grad": 2, ("adam", "exp_avg"): 5, ("adam", "exp_avg_sq"): 9, ("adam", "param"): 8,
    ("sgd", "exp_avg"): 5, ("sgd", "param"): 4,
    ("radam", "exp_avg"): 4, ("radam", "exp_avg_sq"): 5, ("radam", "param"): 10,
    ("ranger", "exp_avg"): 4, ("ranger", "exp_avg_sq"): 5, ("ranger", "param"): 13,
}
MEASURED = {}        # largest |got - f64| / (u * terms + 2^-149) seen per (rule, stage), printed by the tests


def _square32(x):
    """x * x in float64, +inf where float32's rounding of the product overflows."""
    sq = x * x
    return np.where(sq >= OVF_MID, np.inf, sq)


def truth64(a: Args, count, p, g, m, v, slow, got_m, got_v, got_slow_in=None):
    """{stage: (f64 value, sum of |terms|)} of one tensor's step at `count` (None: SGD without momentum), from the
    kernel's float32 inputs: m' and v' from (m, v, g, p); p' from (p, g) and the kernel's own m', v' (and slow)."""
    d = lambda x: None if x is None else np.asarray(x, f32).astype(np.float64)     # noqa: E731
    p, g, m, v, slow, gm, gv = map(d, (p, g, m, v, slow, got_m, got_v))
    out = {}
    with np.errstate(all="ignore"):
        if a.rule == "adam":
            ge = g + a.weight_decay * p if a.weight_decay != 0 else g
            ga = np.abs(g) + abs(a.weight_decay) * np.abs(p)
            b1w, b2w = 1 - a.beta1, 1 - a.beta2
            out["exp_avg"] = (m + b1w * (ge - m), np.abs(m) + b1w * (ga + np.abs(m)))
            out["exp_avg_sq"] = (a.beta2 * v + b2w * _square32(ge), a.beta2 * np.abs(v) + b2w * ga * ga)
            bc1 = 1 - a.beta1 ** count
            bc2 = 1 - a.beta2 ** count
            upd = (a.lr / bc1) * gm / (np.sqrt(gv) / math.sqrt(bc2) + a.eps)
            out["param"] = (p - upd, np.abs(p) + np.abs(upd))
            return out
        if a.rule == "sgd":
            ge = g + a.weight_decay * p if a.weight_decay != 0 else g
            ga = np.abs(g) + a.weight_decay * np.abs(p)
            if a.momentum != 0:
                if count == 1:
                    out["exp_avg"] = (ge, ga)
                else:
                    out["exp_avg"] = (a.momentum * m + ge, a.momentum * np.abs(m) + ga)
                out["param"] = (p - a.lr * gm, np.abs(p) + a.lr * np.abs(gm))
            else:
                out["param"] = (p - a.lr * ge, np.abs(p) + a.lr * ga)
            return out
        b1w, b2w = 1 - a.beta1, 1 - a.beta2
        out["exp_avg"] = (a.beta1 * m + b1w * g, a.beta1 * np.abs(m) + b1w * np.abs(g))
        out["exp_avg_sq"] = (a.beta2 * v + b2w * _square32(g), a.beta2 * np.abs(v) + b2w * g * g)
        adaptive, step_size = rectification(a, count)
        upd = step_size * a.lr * (gm / (np.sqrt(gv) + a.eps) if adaptive else gm)
        dec = a.weight_decay * a.lr * p
        w = p - dec - upd
        terms = np.abs(p) + np.abs(dec) + np.abs(upd)
        if a.rule == "ranger" and count % a.k == 0:
            s0 = p if count == 1 else slow
            w = s0 + a.alpha * (w - s0)
            terms = np.abs(s0) + a.alpha * (terms + np.abs(s0))
        out["param"] = (w, terms)
        return out


def measure(rule, stage, got, truth, terms, where):
    """Asserts got against float64 truth: the same non-finite class (NaN, +inf, -inf) at every element, and
    |got - truth| <= k (u terms + 2^-149) at the finite ones.  Records the largest |got - truth| / (u terms + 2^-149).
    exp_avg_sq's truth is +inf where the stage's own product g * g is past float32's range: ATen's addcmul, which the
    kernel follows, rounds that product to float32 before the fused add."""
    k = BOUND_K["grad"] if stage == "grad" else BOUND_K[(rule, stage)]
    got = np.asarray(got, np.float64)
    with np.errstate(all="ignore"):        # float32 holds nothing at or past the overflow threshold
        truth = np.where(np.abs(truth) >= OVF_MID, truth * np.inf, truth)
    for cls, f in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
        bad = np.flatnonzero(f(got) != f(truth))
        if bad.size:
            e = int(bad[0])
            raise AssertionError(f"{where}: {stage} element {e}: {cls} class differs from float64 "
                                 f"(got {got[e]!r}, float64 {truth[e]!r}; {bad.size} elements)")
    fin = np.isfinite(got)
    if not fin.any():
        return
    with np.errstate(all="ignore"):
        err = np.abs(got[fin] - truth[fin])
        unit = U * terms[fin] + TINY
        lim = k * unit
        bad = np.flatnonzero(~(err <= lim))
        if bad.size:
            e = int(np.flatnonzero(fin)[bad[0]])
            raise AssertionError(f"{where}: {stage} element {e}: |got - float64| = {err[bad[0]]:.3e} exceeds "
                                 f"{k} (u * terms + 2^-149) = {lim[bad[0]]:.3e} (got {got[e]!r}, float64 "
                                 f"{truth[e]!r})")
        rel = err / unit
    key = (rule, stage)
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(rel.max()))


def measured_report():
    return "; ".join(f"{r} {s}: {v:.2f} u (bound {BOUND_K['grad'] if s == 'grad' else BOUND_K[(r, s)]} u)"
                     for (r, s), v in sorted(MEASURED.items()))


# ------------------------------------------------------------------------------------------------ checkers
KERNELS = {
    ("nerf", "rule"): "step_kernel<{}> (NeRF)", ("nerf_amp", "rule"): "step_kernel<{}> (NeRF, _amp)",
    ("tensors", "rule"): "step_kernel<{}> (table)", ("tensors_amp", "rule"): "step_kernel<{}> (table, _amp)",
}


def kernel_name(form, rule):
    k = KERNELS.get((form, "adam")) if rule == "adam" else None
    return k or KERNELS[(form, "rule")].format(rule.upper() if rule == "sgd" else rule.capitalize())


def _bits(x):
    return np.asarray(x, f32).view(np.uint32)


def _compare_bits(got, exp, computed, where, what):
    """Bit equality; a NaN may differ in payload only where the element was computed (the GPU's canonical NaN against
    numpy's propagated one)."""
    gb, eb = _bits(got), _bits(exp)
    diff = gb != eb
    if computed is not None:
        diff &= ~(computed & np.isnan(got) & np.isnan(exp))
    bad = np.flatnonzero(diff)
    if bad.size:
        e = int(bad[0])
        raise AssertionError(f"{where}: {what} element {e}: got {got.flat[e]!r} (0x{gb.flat[e]:08x}), emulation "
                             f"{exp.flat[e]!r} (0x{eb.flat[e]:08x}); {bad.size} elements differ")


def check_launch(form, a: Args, impl, st: Step, step=None, amp=None, step_no=0, precision=None):
    """One launch of `form` on impl against the emulation (bit for bit: params, every state buffer passed, grads for
    _amp, count_out) and each stepped tensor's stages against float64.  Steps `st` in place to impl's result.
    amp: dict(scale, found_inf, count_in, base).  Returns count_out (amp) or None."""
    before = st.copy()
    exp = st.copy()
    if form in ("tensors", "nerf"):
        (emulate_tensors if form == "tensors" else emulate_nerf)(a, exp, step, sm_count=impl.sm_count)
        getattr(impl, "step_" + form)(a, st, step, **({"precision": precision} if form == "nerf" else {}))
        count_out = exp_counts = None
    else:
        exp_counts = emulate_amp(form, a, exp, amp["scale"], amp["found_inf"], amp["count_in"], amp["base"],
                                 sm_count=impl.sm_count)
        kw = {"precision": precision} if form == "nerf_amp" else {}
        count_out = getattr(impl, "step_" + form)(a, st, amp["scale"], amp["found_inf"], amp["count_in"], amp["base"],
                                                  **kw)
    kname = kernel_name(form, a.rule)
    where0 = f"{kname} {a.rule} step {step_no}"
    if exp_counts is not None:
        got_c = np.asarray(count_out, np.int64)
        bad = np.flatnonzero(got_c != exp_counts)
        if bad.size:
            raise AssertionError(f"{where0}: count_out[{bad[0]}] = {got_c[bad[0]]}, expected {exp_counts[bad[0]]}")
    numel = [p.size for p in st.params]
    off = offsets(numel)
    stepped = np.zeros(sum(numel), bool)
    for t, g in enumerate(st.grads):
        if g is not None:
            stepped[off[t]:off[t] + numel[t]] = True
    written = amp is not None and inv_scale32(amp["scale"]) != 1      # gradients are stored back only then
    for t in range(len(st.params)):
        where = f"{where0} tensor {t}"
        comp = np.full(numel[t], before.grads[t] is not None)
        _compare_bits(st.params[t], exp.params[t], comp, where, "param")
        if form.endswith("amp") and before.grads[t] is not None:
            _compare_bits(st.grads[t], exp.grads[t], comp & written, where, "grad")
    used = used_buffers(a)
    for name in ("exp_avg", "exp_avg_sq", "slow"):
        g_buf, e_buf = getattr(st, name), getattr(exp, name)
        if e_buf is None:
            continue
        # a computed NaN's payload may differ, but only in the stepped regions of the buffers the rule keeps
        nan_ok = stepped & np.isnan(g_buf) & np.isnan(e_buf) if name in used else False
        bad = np.flatnonzero((_bits(g_buf) != _bits(e_buf)) & ~nan_ok)
        if bad.size:
            i = int(bad[0])
            t = int(np.searchsorted(off, i, side="right") - 1)
            raise AssertionError(f"{where0} tensor {t}: {name} element {i - off[t]}: got {g_buf[i]!r} "
                                 f"(0x{_bits(g_buf)[i]:08x}), emulation {e_buf[i]!r} (0x{_bits(e_buf)[i]:08x}); "
                                 f"{bad.size} elements differ")
    # float64, stage by stage
    skip = amp is not None and amp["found_inf"] is not None and amp["found_inf"] != 0
    counts = None
    if amp is not None:
        counts, _ = _amp_counts(form, a, before, amp["count_in"], amp["base"], skip, None)
    for t, g in enumerate(before.grads):
        if g is None:
            continue
        where = f"{where0} tensor {t}"
        inv = inv_scale32(amp["scale"]) if amp is not None else f32(1.0)
        g_in = st.grads[t] if amp is not None else g
        if amp is not None and inv != 1:
            measure(a.rule, "grad", st.grads[t], g.astype(np.float64) / float(f32(amp["scale"])),
                    np.abs(g.astype(np.float64)) / float(f32(amp["scale"])), where)
        if skip:
            continue
        if amp is not None:
            count = counts[t]
        elif a.rule == "adam" and form == "nerf":
            count = int(step)
        elif a.rule == "sgd" and a.momentum == 0:
            count = None
        else:
            count = int(step[t])
        sl = slice(off[t], off[t] + numel[t])
        sel = lambda b: None if b is None else b[sl]      # noqa: E731
        tr = truth64(a, count, before.params[t], g_in, sel(before.exp_avg), sel(before.exp_avg_sq), sel(before.slow),
                     sel(st.exp_avg), sel(st.exp_avg_sq))
        for stage, (val, terms) in tr.items():
            got = st.params[t] if stage == "param" else getattr(st, stage)[sl]
            measure(a.rule, stage, got, val, terms, where)
    return count_out


# ------------------------------------------------------------------------------------------------ inputs
def edge_values(n, rng, kind, nonfinite=False):
    """float32 values for one tensor, the edge classes interleaved by index (so the first, last and every sweep's
    elements see all of them) and the rest random:
      kind 'param':  magnitudes 2^-30 .. 2^30, both signs, +-0
      kind 'grad':   as param, plus 0, subnormals, |g| >= 2^64 (its square overflows float32) and, with nonfinite,
                     NaN and +-inf
      kind 'm':      as param;  kind 'v': non-negative, 0 included."""
    x = (np.exp2(rng.uniform(-30, 30, n)) * rng.choice([-1.0, 1.0], n)).astype(f32)
    if kind == "v":
        x = np.abs(x)
    specials = {"param": [0.0, -0.0, 1.0, -2.0 ** -30, 2.0 ** 30],
                "m": [0.0, -0.0, 2.0 ** -30, -2.0 ** 30],
                "v": [0.0, 2.0 ** -60, 2.0 ** 60, 1.0],
                "grad": [0.0, -0.0, 1e-45, -3e-42, 1.1754942e-38, 2.0 ** 64, -2.0 ** 70, 2.0 ** 100, 2.0 ** -30,
                         -2.0 ** 30]}[kind]
    if nonfinite and kind == "grad":
        specials = specials + [np.nan, np.inf, -np.inf]
    period = 3 * len(specials) + 1
    idx = np.arange(n)
    which = idx % period
    hit = which < len(specials)
    x[hit] = np.asarray(specials, f32)[which[hit]]
    x[-1:] = np.asarray(specials[(n - 1) % len(specials)], f32)
    return x


def zero_pairs(st: Step, rng):
    """Zero gradient on zero state in a scattered tenth of the stepped elements (den = eps, update 0)."""
    numel = [p.size for p in st.params]
    off = offsets(numel)
    for t, g in enumerate(st.grads):
        if g is None:
            continue
        z = rng.random(numel[t]) < 0.1
        g[z] = 0
        for buf in (st.exp_avg, st.exp_avg_sq):
            if buf is not None:
                buf[off[t]:off[t] + numel[t]][z] = 0


def used_buffers(a: Args):
    """The state buffers the rule reads and writes."""
    return {"adam": ("exp_avg", "exp_avg_sq"), "radam": ("exp_avg", "exp_avg_sq"),
            "ranger": ("exp_avg", "exp_avg_sq", "slow"), "sgd": ("exp_avg",) if a.momentum != 0 else ()}[a.rule]


def make_step(a: Args, numel, gradless=(), seed=0, nonfinite=False, used=None):
    """Inputs for one launch: edge-valued params, grads and state; tensors in `gradless` have no gradient and their
    params and state regions hold SENTINEL; state buffers the rule does not use are passed full of SENTINEL.
    used: the buffers the rule reads (default: by rule)."""
    rng = np.random.default_rng(seed)
    params = [edge_values(n, rng, "param") for n in numel]
    grads = [None if t in gradless else edge_values(n, rng, "grad", nonfinite) for t, n in enumerate(numel)]
    total = int(sum(numel))
    if used is None:
        used = used_buffers(a)
    bufs = {}
    for name, kind in (("exp_avg", "m"), ("exp_avg_sq", "v"), ("slow", "param")):
        bufs[name] = (np.concatenate([edge_values(n, rng, kind) for n in numel]) if name in used
                      else np.full(total, SENTINEL, f32))
    st = Step(params, grads, bufs["exp_avg"], bufs["exp_avg_sq"], bufs["slow"])
    zero_pairs(st, rng)
    off = offsets(numel)
    for t in gradless:
        st.params[t][:] = SENTINEL
        for name in used:
            getattr(st, name)[off[t]:off[t] + numel[t]] = SENTINEL
    return st


def first_adaptive(a: Args) -> int:
    """The first count at which RAdam / Ranger takes the adaptive step."""
    for t in range(1, 100000):
        if rectification(a, t)[0]:
            return t
    raise ValueError(a)


# ------------------------------------------------------------------------------------------------ scenarios
# Each runs a few launches of one entry point through check_launch on `impl`; the GPU test runs them on the library,
# the CPU test on the stand-in.  They raise AssertionError naming kernel, rule, step, tensor, element and stage.
def table_shapes(sm_count):
    """numel 1, 255, 256, 257, one tensors-kernel sweep +- 1, and one tensor of more than 2^21 elements (many
    sweeps), with gradless tensors between them."""
    sweep = 4 * sm_count * BLOCK
    return [1, 255, 7, 256, 257, sweep - 1, 5, sweep + 1, (1 << 21) + 3, 3]


GRADLESS = (2, 6, 9)


def scenario_table(impl, rule, weight_decay, n_steps=3):
    """snb_optim_step_tensors over table_shapes: gradless tensors interleaved (sentinel params and state), counts that
    differ per tensor, an lr change after the first step.  SGD runs with momentum 0.9."""
    a = Args(rule, lr=1e-3, weight_decay=weight_decay, momentum=0.9 if rule == "sgd" else 0.0,
             beta1=0.95 if rule == "ranger" else 0.9, k=5)
    numel = table_shapes(impl.sm_count)
    st = make_step(a, numel, GRADLESS, seed=1)
    step = np.array([1, 2, 1, 5, 6, 4, 1, 9, 1, 1]) if rule != "sgd" else np.array([1, 2, 1, 3, 1, 4, 1, 2, 1, 1])
    for s in range(n_steps):
        check_launch("tensors", a, impl, st, step=step, step_no=s)
        step = step + 1
        a = a.with_(lr=a.lr * 0.5)
        _fresh_grads(st, s + 10)


def scenario_table32(impl, rule):
    """A 32-entry table (the last entry sets bit 31 of the _amp form's advance mask), plain and _amp."""
    a = Args(rule, weight_decay=1e-2, momentum=0.9 if rule == "sgd" else 0.0)
    numel = [(37 * t) % 300 + 1 for t in range(MAX_TENSORS)]
    st = make_step(a, numel, (0, 13), seed=2)
    check_launch("tensors", a, impl, st, step=np.arange(1, MAX_TENSORS + 1), step_no=0)
    _fresh_grads(st, 3)
    count_in = np.arange(MAX_TENSORS, dtype=np.int32)
    check_launch("tensors_amp", a, impl, st, step_no=1,
                 amp=dict(scale=3000.0, found_inf=0.0, count_in=count_in, base=count_in + 1 - (np.arange(32) % 8)))


def _fresh_grads(st: Step, seed):
    rng = np.random.default_rng(seed)
    for t, g in enumerate(st.grads):
        if g is not None:
            g[:] = edge_values(g.size, rng, "grad")


def count_set(a: Args):
    """Counts 1 and 2, both sides of the adaptive crossing, 1e4 and 1e6."""
    c = first_adaptive(a) if a.rule in ("radam", "ranger") else 3
    return sorted({1, 2, c - 1, c, c + 1, 10 ** 4, 10 ** 6})


def scenario_counts(impl, rule, beta2):
    """One launch of snb_optim_step_tensors with one tensor per count of count_set, so that some turn adaptive (or
    sync) and others do not.  Ranger's threshold is set to N_sma at its crossing count exactly, so N_sma > threshold
    and >= differ there."""
    a = Args(rule, lr=1e-3, weight_decay=1e-2, momentum=0.9 if rule == "sgd" else 0.0, beta2=beta2, k=6)
    if rule == "ranger":
        c = first_adaptive(a)
        a = a.with_(n_sma_threshold=n_sma(a, c))
    counts = count_set(a)
    if rule == "ranger":
        counts = sorted(set(counts) | {6, 12})
    numel = [300 + 7 * i for i in range(len(counts))]
    st = make_step(a, numel, (), seed=3)
    check_launch("tensors", a, impl, st, step=np.array(counts), step_no=0)


def scenario_ranger(impl, alpha, k):
    """Ranger syncs at alpha 0, 0.5, 1 and k 1, 5, 6: tensors at different counts in one launch, two launches."""
    a = Args("ranger", lr=1e-3, weight_decay=1e-2, beta1=0.95, alpha=alpha, k=k)
    numel = [1, 257, 300, 511, 64, 33]
    st = make_step(a, numel, (4,), seed=4)
    step = np.array([1, k, k + 1, 2 * k - 1, 1, 2 * k])
    for s in range(2):
        check_launch("tensors", a, impl, st, step=step, step_no=s)
        step = step + 1
        _fresh_grads(st, 40 + s)


def scenario_sgd(impl, momentum, weight_decay):
    """SGD with momentum 0 (no state touched; the _amp form does not advance the count) and 0.9."""
    a = Args("sgd", lr=1e-2, weight_decay=weight_decay, momentum=momentum)
    numel = [1, 255, 256, 257, 9]
    st = make_step(a, numel, (3,), seed=5)
    step = np.array([1, 2, 1, 1, 7]) if momentum else np.zeros(5, int)
    check_launch("tensors", a, impl, st, step=step, step_no=0)
    _fresh_grads(st, 50)
    count_in = (step if momentum else np.zeros(5, int)).astype(np.int32)
    check_launch("tensors_amp", a, impl, st, step_no=1,
                 amp=dict(scale=2.0 ** 16, found_inf=0.0, count_in=count_in, base=np.maximum(count_in + 1 - 3, 1)))


def amp_bases(count_in, slots):
    """The base that puts count_in + 1 at window slot `slot` for each tensor."""
    return np.asarray(count_in) + 1 - np.asarray(slots)


def _snan_grads(st: Step):
    """SENTINEL (a signalling NaN) in the first, middle and last gradient element of each tensor: a kernel that stores
    g * 1 back quiets it, so at scale 1 these bits show whether the gradient was written."""
    for g in st.grads:
        if g is not None:
            g[[0, g.size // 2, g.size - 1]] = SENTINEL


def scenario_amp(impl, rule, scale):
    """snb_optim_step_tensors_amp: window slots 0 and 7 and tensors at different bases in one launch, then a step with
    found_inf set (nothing but the gradients moves), then one more taken step at other slots.  At scale 1 some
    gradient elements are signalling NaNs, which must come back with their bits."""
    a = Args(rule, lr=1e-3, weight_decay=1e-2, momentum=0.9 if rule == "sgd" else 0.0, k=5)
    numel = [1, 255, 256, 257, 4 * impl.sm_count * BLOCK + 1, 31]
    st = make_step(a, numel, (2,), seed=6)
    count_in = np.array([7, 8, 9, 12, 14, 7], np.int32)
    slots = [[0, 7, 3, 7, 0, 7], [7, 0, 0, 1, 7, 5], [7, 0, 7, 0, 7, 1]]
    for s, found_inf in enumerate([0.0, 1.0, 0.0]):
        if scale == 1.0:
            _snan_grads(st)
        base = amp_bases(count_in, slots[s])
        assert (base >= 1).all(), base
        count_out = check_launch("tensors_amp", a, impl, st, step_no=s,
                                 amp=dict(scale=scale, found_inf=found_inf, count_in=count_in, base=base))
        count_in = np.asarray(count_out, np.int32)
        _fresh_grads(st, 60 + s)


def scenario_nerf(impl, rule, precision=None, weight_decay=1e-2):
    """The 24 NeRF tensors, one without a gradient: two plain steps (snb_adam_step / snb_optim_step; the second at
    counts where RAdam turns adaptive and Ranger syncs, with an lr change), then the _amp form at slot 0, at slot 7
    with a scale of 3000, and a skipped step."""
    a = Args(rule, lr=1e-3, weight_decay=weight_decay, momentum=0.9 if rule == "sgd" else 0.0,
             beta1=0.95 if rule == "ranger" else 0.9, k=6)
    st = make_step(a, NERF_NUMEL, (5,), seed=7)
    if rule == "adam":
        steps = [1, 6]
    else:
        steps = [np.full(24, 1), np.where(np.arange(24) % 2 == 0, 6, 5)]
    for s, step in enumerate(steps):
        check_launch("nerf", a, impl, st, step=step, step_no=s, precision=precision)
        _fresh_grads(st, 70 + s)
        a = a.with_(lr=a.lr * 0.5)
    n_counts = 1 if rule == "adam" else 24
    count_in = np.full(n_counts, 6, np.int32)
    for s, (slot, scale, found_inf) in enumerate([(0, 2.0 ** 16, 0.0), (7, 3000.0, 0.0), (0, 1.0, 1.0)], 2):
        count_out = check_launch("nerf_amp", a, impl, st, step_no=s, precision=precision,
                                 amp=dict(scale=scale, found_inf=found_inf, count_in=count_in,
                                          base=amp_bases(count_in, np.full(n_counts, slot))))
        count_in = np.asarray(count_out, np.int32)
        _fresh_grads(st, 80 + s)


def scenario_nonfinite(impl, rule):
    """NaN and +-inf gradients through the plain forms: every result keeps float64's class."""
    a = Args(rule, lr=1e-3, weight_decay=1e-2, momentum=0.9 if rule == "sgd" else 0.0)
    numel = [257, 1000, 3]
    st = make_step(a, numel, (), seed=8, nonfinite=True)
    check_launch("tensors", a, impl, st, step=np.array([1, 6, 2]), step_no=0)
    rng = np.random.default_rng(9)
    for g in st.grads:
        g[:] = edge_values(g.size, rng, "grad", nonfinite=True)
    check_launch("tensors", a, impl, st, step=np.array([2, 7, 3]), step_no=1)
