"""The fused optimiser steps of sinnerf_b200/csrc/optim.cu, element by element through the C ABI: every launch's
parameters, state buffers, unscaled gradients (_amp) and counts bit for bit against the float32 emulation of
tests/optim_emulation.py, and each stage of each stepped tensor against float64 from the kernel's own float32 inputs to
that stage, within the bound its count of roundings gives (optim_emulation.BOUND_K).

The inputs are synthetic and chosen for the edges: magnitudes across 2^-30 .. 2^30, +-0, zero gradients on zero state,
subnormal gradients, gradients whose square overflows float32, NaN and +-inf (plain forms); numel 1, 255, 256, 257, one
grid sweep +- 1 from the device's SM count, a tensor of more than 2^21 elements, a 32-entry table; tensors without a
gradient interleaved, their parameters and state regions (and every state buffer the rule does not use) filled with a
NaN-payload sentinel that must come back unchanged; counts 1, 2, both sides of the RAdam / Ranger crossings, 1e4 and
1e6, different per tensor in one launch; _amp window slots 0 and 7, scales 1, 2^16 and 3000, and skipped steps.  The
NeRF entry points run in every precision mode: the re-packed image equals a fresh snb_pack_weights of the stepped
parameters, and snb_refresh_weights finds it clean.

test_torch_ops_match_emulation runs the operations the fused steps replace (torch.optim.Adam's single-tensor path, the
oracle's SGD / RAdam / Ranger) on CUDA tensors holding the same inputs and holds them to the same emulation, bit for
bit, so that "operation for operation" is checked rather than assumed.
"""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

from tests import optim_emulation as emu

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NEW_ACTIVATION = 1


class Lib:
    """optim_emulation.StandIn's interface on the C ABI: numpy in, numpy out, tensors on cuda:0 in between."""

    def __init__(self):
        from sinnerf_b200 import _lib
        self._lib, self.lib = _lib, _lib.load()
        sm = C.c_int(0)
        assert self.lib.snb_device_check(C.byref(sm), None, None) == 0, self.lib.snb_last_error()
        self.sm_count = sm.value
        self.images_checked = 0

    def _ok(self, rc):
        assert rc == 0, self.lib.snb_last_error()
        torch.cuda.synchronize()

    @staticmethod
    def _up(x):
        return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)

    @staticmethod
    def _down(dst, src):
        if dst is not None:
            dst[...] = src.cpu().numpy()

    def _upload(self, st):
        return ([self._up(p) for p in st.params], [self._up(g) for g in st.grads],
                [self._up(b) for b in (st.exp_avg, st.exp_avg_sq, st.slow)])

    def _download(self, st, dev, grads=False):
        ps, gs, bufs = dev
        for p, d in zip(st.params, ps):
            self._down(p, d)
        if grads:
            for g, d in zip(st.grads, gs):
                self._down(g, d)
        for b, d in zip((st.exp_avg, st.exp_avg_sq, st.slow), bufs):
            self._down(b, d)

    def _ptrs(self, ts):
        return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])

    def _optim_args(self, a):
        return self._lib.SnbOptimArgs(emu.RULE_ID[a.rule], a.lr, a.weight_decay, a.momentum, a.beta1, a.beta2, a.eps,
                                      a.n_sma_threshold, a.alpha, a.k)

    def _amp(self, scale, found_inf, count_in, base):
        keep = dict(scale=None if scale is None else torch.tensor([scale], dtype=torch.float32, device=DEV),
                    found_inf=None if found_inf is None else torch.tensor([found_inf], dtype=torch.float32,
                                                                          device=DEV),
                    count_in=torch.tensor(np.asarray(count_in), dtype=torch.int32, device=DEV))
        keep["count_out"] = torch.full_like(keep["count_in"], -7)
        b = np.zeros(emu.MAX_TENSORS, np.int64)
        b[:len(base)] = base
        amp = self._lib.SnbAmpStep(self._lib.ptr(keep["scale"]), self._lib.ptr(keep["found_inf"]),
                                   self._lib.ptr(keep["count_in"]), self._lib.ptr(keep["count_out"]),
                                   (C.c_int * emu.MAX_TENSORS)(*[int(x) for x in b]))
        return amp, keep

    def step_tensors(self, a, st, step):
        dev = self._upload(st)
        numel = (C.c_int64 * len(st.params))(*[p.size for p in st.params])
        steps = (C.c_int * len(st.params))(*[int(x) for x in step])
        m, v, s = (self._lib.ptr(b) for b in dev[2])
        args = self._optim_args(a)
        self._ok(self.lib.snb_optim_step_tensors(len(st.params), self._ptrs(dev[0]), self._ptrs(dev[1]), numel, steps,
                                                 m, v, s, C.byref(args), self._lib.stream_ptr(DEV)))
        self._download(st, dev)

    def step_tensors_amp(self, a, st, scale, found_inf, count_in, base):
        dev = self._upload(st)
        numel = (C.c_int64 * len(st.params))(*[p.size for p in st.params])
        m, v, s = (self._lib.ptr(b) for b in dev[2])
        args = self._optim_args(a)
        amp, keep = self._amp(scale, found_inf, count_in, base)
        self._ok(self.lib.snb_optim_step_tensors_amp(len(st.params), self._ptrs(dev[0]), self._ptrs(dev[1]), numel,
                                                     m, v, s, C.byref(args), C.byref(amp), self._lib.stream_ptr(DEV)))
        self._download(st, dev, grads=True)
        assert torch.equal(keep["count_in"].cpu(), torch.tensor(np.asarray(count_in), dtype=torch.int32))
        return keep["count_out"].cpu().numpy()

    # NeRF entry points: the packed image of `precision` (None: no image) is packed from the parameters before the
    # step, handed to the step, and checked after it.
    def _packed(self, params, precision):
        if precision is None:
            return None
        prec = self._lib.precision_id(precision)
        buf = torch.zeros(int(self.lib.snb_packed_weights_bytes(prec)), dtype=torch.uint8, device=DEV)
        self._ok(self.lib.snb_pack_weights(self._ptrs(params), prec, NEW_ACTIVATION, self._lib.ptr(buf),
                                           self._lib.stream_ptr(DEV)))
        return buf

    def _check_image(self, params, precision, packed, before, skipped):
        if packed is None:
            return
        prec = self._lib.precision_id(precision)
        header = packed[:32].cpu().numpy().view(np.int32)
        if skipped:
            assert header[4] == 0, f"{precision}: a skipped step leaves the header dirty"
            assert torch.equal(packed[24:], before[24:]), f"{precision}: a skipped step changed the image"
        fresh = self._packed(params, precision)
        assert torch.equal(packed[256:], fresh[256:]), f"{precision}: image after the step != a fresh pack"
        assert torch.equal(packed[24:32], fresh[24:32]), f"{precision}: stamped checksum != a fresh pack's"
        self._ok(self.lib.snb_refresh_weights(self._ptrs(params), prec, NEW_ACTIVATION, self._lib.ptr(packed),
                                              self._lib.stream_ptr(DEV)))
        assert packed[:32].cpu().numpy().view(np.int32)[4] == 0, f"{precision}: refresh found the image dirty"
        self.images_checked += 1

    def step_nerf(self, a, st, step, precision=None):
        dev = self._upload(st)
        packed = self._packed(dev[0], precision)
        m, v, s = (self._lib.ptr(b) for b in dev[2])
        prec = 0 if precision is None else self._lib.precision_id(precision)
        if a.rule == "adam":
            args = self._lib.SnbAdamArgs(a.lr, a.beta1, a.beta2, a.eps, a.weight_decay, int(step))
            rc = self.lib.snb_adam_step(self._ptrs(dev[0]), self._ptrs(dev[1]), m, v, C.byref(args), prec,
                                        NEW_ACTIVATION, self._lib.ptr(packed), self._lib.stream_ptr(DEV))
        else:
            args = self._optim_args(a)
            args.step = (C.c_int * 24)(*[int(x) for x in step])
            rc = self.lib.snb_optim_step(self._ptrs(dev[0]), self._ptrs(dev[1]), m, v, s, C.byref(args), prec,
                                         NEW_ACTIVATION, self._lib.ptr(packed), self._lib.stream_ptr(DEV))
        self._ok(rc)
        self._check_image(dev[0], precision, packed, None, False)
        self._download(st, dev)

    def step_nerf_amp(self, a, st, scale, found_inf, count_in, base, precision=None):
        dev = self._upload(st)
        packed = self._packed(dev[0], precision)
        skipped = found_inf is not None and found_inf != 0
        if packed is not None and skipped:
            packed[16:20] = torch.tensor([1, 0, 0, 0], dtype=torch.uint8)     # header.dirty = 1: the skip must clear it
        before = None if packed is None else packed.clone()
        m, v, s = (self._lib.ptr(b) for b in dev[2])
        prec = 0 if precision is None else self._lib.precision_id(precision)
        amp, keep = self._amp(scale, found_inf, count_in, base)
        if a.rule == "adam":
            args = self._lib.SnbAdamArgs(a.lr, a.beta1, a.beta2, a.eps, a.weight_decay, 0)
            rc = self.lib.snb_adam_step_amp(self._ptrs(dev[0]), self._ptrs(dev[1]), m, v, C.byref(args), C.byref(amp),
                                            prec, NEW_ACTIVATION, self._lib.ptr(packed), self._lib.stream_ptr(DEV))
        else:
            args = self._optim_args(a)
            rc = self.lib.snb_optim_step_amp(self._ptrs(dev[0]), self._ptrs(dev[1]), m, v, s, C.byref(args),
                                             C.byref(amp), prec, NEW_ACTIVATION, self._lib.ptr(packed),
                                             self._lib.stream_ptr(DEV))
        self._ok(rc)
        self._check_image(dev[0], precision, packed, before, skipped)
        self._download(st, dev, grads=True)
        return keep["count_out"].cpu().numpy()


_lib_obj = []


def lib():
    if not _lib_obj:
        _lib_obj.append(Lib())
    return _lib_obj[0]


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print(f"\noptimiser stages, largest |got - float64| / (u * terms + 2^-149): {emu.measured_report()}",
          file=sys.stderr)


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("rule", emu.RULES)
def test_table(rule, weight_decay):
    emu.scenario_table(lib(), rule, weight_decay)


@pytest.mark.parametrize("rule", emu.RULES)
def test_table32(rule):
    emu.scenario_table32(lib(), rule)


@pytest.mark.parametrize("beta2", [0.9, 0.99, 0.999])
@pytest.mark.parametrize("rule", emu.RULES)
def test_counts(rule, beta2):
    emu.scenario_counts(lib(), rule, beta2)


@pytest.mark.parametrize("k", [1, 5, 6])
@pytest.mark.parametrize("alpha", [0.0, 0.5, 1.0])
def test_ranger_sync(alpha, k):
    emu.scenario_ranger(lib(), alpha, k)


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("momentum", [0.0, 0.9])
def test_sgd(momentum, weight_decay):
    emu.scenario_sgd(lib(), momentum, weight_decay)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 16, 3000.0])
@pytest.mark.parametrize("rule", emu.RULES)
def test_amp(rule, scale):
    emu.scenario_amp(lib(), rule, scale)


@pytest.mark.parametrize("rule", emu.RULES)
def test_nonfinite_gradients(rule):
    emu.scenario_nonfinite(lib(), rule)


@pytest.mark.parametrize("precision", ["fp32", "f16x3", "bf16x3", "bf16", "f16"])
@pytest.mark.parametrize("rule", emu.RULES)
def test_nerf(rule, precision):
    """The NeRF entry points with the image of `precision`: two plain steps, two _amp steps and a skipped one."""
    before = lib().images_checked
    emu.scenario_nerf(lib(), rule, precision)
    assert lib().images_checked - before == 5


# ------------------------------------------------------------------------------------------------ the replaced ops
def _torch_step(rule, a, count, p, g, m, v, slow):
    """One step of the optimiser the fused one replaces, on CUDA fp32 tensors with the given state at count - 1."""
    from oracle import optim_oracle
    tp = torch.from_numpy(p.copy()).to(DEV)
    tp.grad = torch.from_numpy(g.copy()).to(DEV)
    if rule == "adam":
        opt = torch.optim.Adam([tp], lr=a.lr, betas=(a.beta1, a.beta2), eps=a.eps, weight_decay=a.weight_decay,
                               foreach=False)
        state = {"step": torch.tensor(float(count - 1)), "exp_avg": torch.from_numpy(m.copy()).to(DEV),
                 "exp_avg_sq": torch.from_numpy(v.copy()).to(DEV)}
    elif rule == "sgd":
        opt = optim_oracle.SGD([tp], lr=a.lr, momentum=a.momentum, weight_decay=a.weight_decay)
        state = {} if count == 1 else {"momentum_buffer": torch.from_numpy(m.copy()).to(DEV)}
    else:
        cls = optim_oracle.RAdam if rule == "radam" else optim_oracle.Ranger
        kw = dict(alpha=a.alpha, k=a.k, N_sma_threshhold=a.n_sma_threshold) if rule == "ranger" else {}
        opt = cls([tp], lr=a.lr, betas=(a.beta1, a.beta2), eps=a.eps, weight_decay=a.weight_decay, **kw)
        state = {} if count == 1 else {"step": count - 1, "exp_avg": torch.from_numpy(m.copy()).to(DEV),
                                       "exp_avg_sq": torch.from_numpy(v.copy()).to(DEV)}
        if rule == "ranger" and count > 1:
            state["slow_buffer"] = torch.from_numpy(slow.copy()).to(DEV)
    if state:
        opt.state[tp] = state
    opt.step()
    st = opt.state[tp]
    m_out = st.get("exp_avg", st.get("momentum_buffer"))
    return (tp.detach().cpu().numpy(), None if m_out is None else m_out.cpu().numpy(),
            None if "exp_avg_sq" not in st else st["exp_avg_sq"].cpu().numpy(),
            None if "slow_buffer" not in st else st["slow_buffer"].cpu().numpy())


@pytest.mark.parametrize("weight_decay", [0.0, 1e-2])
@pytest.mark.parametrize("rule", emu.RULES)
def test_torch_ops_match_emulation(rule, weight_decay):
    """torch.optim.Adam(foreach=False) and the oracle's SGD / RAdam / Ranger, stage by stage on CUDA: parameters and
    every state tensor equal the emulation's bit for bit at each count of count_set (RAdam / Ranger on both sides of
    the crossing, Ranger on its sync counts), on finite edge values (the replaced optimisers start a tensor's state at
    zeros, so counts past 1 load state as a resumed run would)."""
    a = emu.Args(rule, lr=1e-3, weight_decay=weight_decay, momentum=0.9 if rule == "sgd" else 0.0,
                 beta1=0.95 if rule == "ranger" else 0.9, k=6)
    counts = sorted(set(emu.count_set(a)) | ({6, 12} if rule == "ranger" else set()))
    rng = np.random.default_rng(11)
    c = emu.consts(a)
    for count in counts:
        n = 4099
        p, g = emu.edge_values(n, rng, "param"), emu.edge_values(n, rng, "grad")
        m, v, slow = emu.edge_values(n, rng, "m"), emu.edge_values(n, rng, "v"), emu.edge_values(n, rng, "param")
        if count == 1:
            m, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
        if rule == "adam":
            lr_neg_step, inv = emu.adam_scalars(a, count)
            ep, em, ev = emu.adam32(p, g, m, v, c, lr_neg_step, inv)
            es = None
        else:
            step_lr, flags = emu.rule_scalars(a, count)
            ep, em, ev, es = emu.rule32(rule, p, g, m, v, slow, c, flags, step_lr)
        tp, tm, tv, ts = _torch_step(rule, a, count, p, g, m, v, slow)
        what = f"{rule} wd={weight_decay} count {count}"
        computed = np.ones(n, bool)
        emu._compare_bits(tm, em, computed, what, "exp_avg")
        if rule != "sgd":
            emu._compare_bits(tv, ev, computed, what, "exp_avg_sq")
        emu._compare_bits(tp, ep, computed, what, "param")
        if rule == "ranger":
            emu._compare_bits(ts, es, computed, what, "slow_buffer")
