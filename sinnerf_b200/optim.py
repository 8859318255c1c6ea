"""Fused Adam for the NeRF MLPs (SURVEY 8f-4): `torch.optim.Adam` as the reference's `get_optimizer` configures
it (reference utils/__init__.py:10-31: lr, eps = 1e-8, weight_decay) with the whole update of one model --
all 24 tensors -- in ONE sm_90a kernel, followed on the same stream by the re-pack of the weight image the
field kernels stream, so the next forward finds it up to date (and stamped clean) without re-packing.

`FusedAdam` is a `torch.optim.Optimizer`: `param_groups[0]['lr']` is honoured every step, so the reference's
schedulers (utils/__init__.py:34-58, warm-up included) keep working; under DDP it is stepped after the
gradient all-reduce exactly like torch's Adam (train.py:51-52).  State (`exp_avg`, `exp_avg_sq`) is one flat
fp32 buffer per model; `state_dict()` exposes per-parameter views with torch.optim.Adam's key names.

`FusedSGD`, `FusedRAdam` and `FusedRanger` do the same for the reference's other `--optimizer` choices (torch.optim.SGD,
and the reference's own RAdam and Ranger, utils/optimizers.py), with per-parameter step counts and state keys as
those optimizers keep them, so checkpoints move both ways between them and the fused ones.

All four also step `sinnerf_b200.discriminator.Discriminator` modules, which `get_optimizer(hparams, [self.D],
rate=0.2)` hands them for the adversarial loss (models/sinnerf.py:207-209): every weight_orig of a module in one
launch of snb_optim_step_tensors, with no re-pack (the discriminator derives its GEMM copy of each weight on every
call).  There Adam too keeps a step count per parameter, and every rule creates a parameter's state on its first step,
as torch.optim.Adam / SGD and the reference's RAdam / Ranger do over `D.parameters()`; so `opt_d`'s state dict moves
both ways between them and the fused optimisers.

Under AMP all four set `_step_supports_amp_scaling`, so `scaler.step(opt)` hands them GradScaler's scale and found_inf
as device tensors and does not wait for found_inf on the host: the step kernel unscales each gradient (writing it back
to `.grad`, as GradScaler.unscale_ would) and skips the update itself when found_inf is set.  The update counts the
step-dependent scalars need then live on the device (`_Counts`); `state`, `state_dict()` and `load_state_dict()` read
them back when they are behind, so they return what the plain path returns after the same taken and skipped steps.
`amp_scaling=False` keeps GradScaler's own unscale pass and its host check of found_inf (Lightning refuses gradient
clipping for optimisers that unscale internally).
"""
from __future__ import annotations

import collections
import ctypes as C
from typing import Iterable, Optional

import torch

from . import _lib, config
from .discriminator import Discriminator
from .nerf import NeRF

__all__ = ["FusedAdam", "FusedSGD", "FusedRAdam", "FusedRanger", "get_optimizer"]


def _check_modules(models, who: str):
    """(the modules as a list, whether they are Discriminators); TypeError unless they are all NeRF models or all
    Discriminators."""
    models = list(models)
    for kind in (NeRF, Discriminator):
        if models and all(isinstance(m, kind) for m in models):
            return models, kind is Discriminator
    raise TypeError(f"{who} steps sinnerf_b200.NeRF models or sinnerf_b200.discriminator.Discriminator modules, all "
                    "of one kind (pass the modules, not their parameters)")


def _params(m) -> list:
    """The tensors a step of module m updates: a NeRF's 24 in state-dict order, a Discriminator's weight_orig tensors
    in `parameters()` order (what the reference's get_optimizer hands torch; its convolutions have no bias and its
    InstanceNorms no affine parameters).  Like NeRF._param_list, reads the current Parameter objects from the module
    dicts: `parameters()` walks every submodule and costs ~20 us of host time per step."""
    if isinstance(m, NeRF):
        return m._param_list()
    return [c._parameters["weight_orig"] for c in m.main._modules.values() if "weight_orig" in c._parameters]


def _check_tensors(ps, who: str) -> None:
    for p in ps:
        if p.dtype != torch.float32 or not p.is_contiguous() or (p.grad is not None and not p.grad.is_contiguous()):
            raise ValueError(f"{who}: parameters and gradients must be contiguous fp32 CUDA tensors")
        if p.device != ps[0].device:
            raise ValueError(f"{who}: a module's parameters must be on one device (got {p.device} and {ps[0].device})")


class _Counts:
    """The update counts of one module's tensors (FusedAdam over a NeRF: one count for the module) as GradScaler-native
    steps leave them: on the device, where the kernel advances them only on a taken step, with the host's view a
    step or more behind.

    `host` holds the counts as last read back, `lag` the increments issued since, any of which may have been skipped.
    Each step's kernel reads the counts from one row of `dev` and writes them to the other.  Right after the launch the
    new row is copied to pinned memory without blocking; a later step picks up the newest copy whose event has
    completed.  A step needs lag < OPTIM_WINDOW on every count it advances, because the kernel's table of scalars
    covers the counts host + 1 .. host + OPTIM_WINDOW.  Only when the GPU runs that many steps behind does it wait for
    one copy.  Plain steps and loaded state change `host` directly; the device row is refreshed from it before the
    next GradScaler-native step."""

    def __init__(self, n: int):
        self.host = [0] * n
        self.lag = [0] * n
        self.issued = [0] * n          # increments issued in all, to match a read-back with the steps after it
        self.dev = None                # (2, n) int32 on the module's device
        self.row = 0                   # the row holding the current counts
        self.dev_current = False       # whether the device rows follow `host` (False after a host-side change)
        self.reads = collections.deque()   # in-flight read-backs: (event, pinned row, issued at the copy)
        self.ring = self.events = None
        self.seq = 0

    def exact(self) -> bool:
        return not any(self.lag)

    def poll(self) -> None:
        """Take the newest completed read-back, without waiting."""
        done = None
        while self.reads and self.reads[0][0].query():
            done = self.reads.popleft()
        if done is not None:
            self.host = done[1].tolist()
            self.lag = [a - b for a, b in zip(self.issued, done[2])]

    def settle(self) -> None:
        """Make `host` exact: the newest completed read-back, or one blocking copy when that is behind."""
        self.poll()
        if not self.exact():
            self.host = self.dev[self.row].tolist()
            self.lag = [0] * len(self.host)
        self.reads.clear()

    def load(self, counts) -> None:
        """Counts set on the host (a plain step, a loaded state dict); `host` must be exact."""
        assert self.exact()
        self.host = list(counts)
        self.dev_current = False
        self.reads.clear()

    def prepare(self, advances, dev) -> list:
        """Before a GradScaler-native step: the device rows current and the window in reach of every count the step
        advances.  Returns the window bases."""
        self.poll()
        if any(a and lag >= _lib.OPTIM_WINDOW for a, lag in zip(advances, self.lag)):
            self.settle()
        if not self.dev_current:
            if self.dev is None:
                n = len(self.host)
                self.dev = torch.zeros(2, n, dtype=torch.int32, device=dev)
                self.ring = torch.empty(_lib.OPTIM_WINDOW, n, dtype=torch.int32, pin_memory=True)
                self.events = [torch.cuda.Event() for _ in range(_lib.OPTIM_WINDOW)]
            self.dev[self.row].copy_(torch.tensor(self.host, dtype=torch.int32).pin_memory(), non_blocking=True)
            self.dev_current = True
        return [c + 1 for c in self.host]

    def pointers(self):
        return _lib.ptr(self.dev[self.row]), _lib.ptr(self.dev[self.row ^ 1])

    def advance(self, advances) -> None:
        """After the launch: the kernel's output row is current; start reading it back."""
        self.row ^= 1
        for t, a in enumerate(advances):
            if a:
                self.issued[t] += 1
                self.lag[t] += 1
        if len(self.reads) < _lib.OPTIM_WINDOW:
            k = self.seq % _lib.OPTIM_WINDOW
            self.seq += 1
            self.ring[k].copy_(self.dev[self.row], non_blocking=True)
            self.events[k].record()
            self.reads.append((self.events[k], self.ring[k], list(self.issued)))


def _amp_tensor(t, dev):
    """GradScaler's grad_scale / found_inf as a float32 tensor on dev; None where it is absent.  found_inf is the
    integer 0 when no gradient was checked (nothing to skip for)."""
    if not torch.is_tensor(t):
        return None
    return t.to(device=dev, dtype=torch.float32, non_blocking=True)


class _FusedPerTensor(torch.optim.Optimizer):
    """Shared body of the four fused optimisers: one kernel per model and step, then the re-pack of the weight image on
    the same stream (C ABI snb_optim_step; FusedAdam: snb_adam_step).  For Discriminator modules: one
    snb_optim_step_tensors launch per module and step, nothing to re-pack.

    These rules keep a step count per parameter and skip parameters without a gradient, so the count is tracked per
    tensor (`_counts`, one `_Counts` per module) and passed to the kernel per tensor; FusedAdam over NeRF models keeps
    torch.optim.Adam's one count instead.  State mirrors the reference's exactly: a parameter has a `state` entry only
    once it has been stepped, holding views of the flat buffers the kernel updates."""
    _rule: int
    _buffers: tuple          # state keys of the flat buffers, in snb_optim_step's argument order
    _has_step: bool = True   # the state carries the reference's per-parameter `step`
    _step_supports_amp_scaling = True   # GradScaler passes grad_scale / found_inf instead of unscaling and syncing

    def __init__(self, models: Iterable, defaults: dict, precision: Optional[str], amp_scaling: bool = True):
        self.models, self._disc = _check_modules(models, type(self).__name__)
        super().__init__([p for m in self.models for p in _params(m)], defaults)
        self._precision = precision
        if not amp_scaling:
            self._step_supports_amp_scaling = False
        # FusedAdam over NeRF models: torch.optim.Adam's one step count per model, advanced by every step
        self._one_count = self._rule == _lib.OPTIM_ADAM and not self._disc
        self._flat = []          # per model: the flat state buffers, in _buffers order
        self._views = {}         # parameter -> {state key: view of its slice of the flat buffer}
        self._slot = {}          # parameter -> (model index, tensor index): where its update count is kept
        # the reference's state['step'] per tensor
        self._counts = [_Counts(1 if self._one_count else len(_params(m))) for m in self.models]
        self._stale = False      # GradScaler-native steps ran since `state` was last published

    @property
    def state(self):
        """torch.optim.Optimizer's `state`, brought up to date with the device's update counts first."""
        self._sync()
        return self.__dict__["state"]

    @state.setter
    def state(self, value):
        self.__dict__["state"] = value

    def _sync(self) -> None:
        if self.__dict__.get("_stale"):
            self._stale = False
            for c in self._counts:
                c.settle()
            self._publish()

    def _count(self, p) -> int:
        i, t = self._slot[p]
        return self._counts[i].host[t]

    def _amp_inputs(self, dev):
        """(grad_scale, found_inf) as GradScaler's step() attached them, on dev, or None outside GradScaler-native
        stepping (a plain opt.step(), a disabled scaler, amp_scaling=False).  grad_scale is None after
        scaler.unscale_(opt): the gradients are unscaled already."""
        if not self._step_supports_amp_scaling or not hasattr(self, "found_inf"):
            return None
        return _amp_tensor(getattr(self, "grad_scale", None), dev), _amp_tensor(self.found_inf, dev)

    def _ensure_state(self):
        if self._flat:
            return
        for i, m in enumerate(self.models):
            ps = _params(m)
            _lib.require_device(ps[0], type(self).__name__)
            total = sum(p.numel() for p in ps)
            bufs = [torch.zeros(total, device=ps[0].device, dtype=torch.float32) for _ in self._buffers]
            off = 0
            for t, p in enumerate(ps):
                n = p.numel()
                self._views[p] = {k: b[off:off + n].view_as(p) for k, b in zip(self._buffers, bufs)}
                self._slot[p] = (i, t)
                off += n
            assert self._disc or off == _lib.PARAM_FLOATS
            self._flat.append(bufs)

    def _step_value(self, n: int):
        """The state's `step` entry after n updates, in the type the replaced optimiser keeps it."""
        return n

    def _publish(self):
        state = self.__dict__["state"]
        state.clear()
        for p in self._views:
            n = self._count(p)
            if n > 0:
                state[p] = dict(self._views[p], **({"step": self._step_value(n)} if self._has_step else {}))

    def load_state_dict(self, state_dict):
        """Values are copied INTO the flat buffers (the kernel addresses them by offset); a parameter without state
        starts afresh, as in the reference."""
        self._ensure_state()
        self._sync()
        for c in self._counts:
            c.settle()
        super().load_state_dict(state_dict)
        counts = [list(c.host) for c in self._counts]
        for p, views in self._views.items():
            st = self.state.get(p, {})
            i, t = self._slot[p]
            if all(st.get(k) is not None for k in self._buffers):
                for k, v in views.items():
                    v.copy_(st[k])
                counts[i][t] = int(st["step"]) if self._has_step else 1
            else:
                for v in views.values():
                    v.zero_()
                counts[i][t] = 0
        for c, n in zip(self._counts, counts):
            c.load(n)
        self._publish()

    def _args(self, group) -> "_lib.SnbOptimArgs":
        raise NotImplementedError

    def _advances(self, group) -> bool:
        """Whether a parameter with a gradient advances its count this step."""
        return True

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self._ensure_state()
        lib = _lib.load()
        group = self.param_groups[0]
        args = self._args(group)
        adv = self._advances(group)
        # the entry point: snb_optim_step_tensors (Discriminators), snb_adam_step (FusedAdam over NeRF models) or
        # snb_optim_step, each in its plain and its GradScaler-native (_amp) form
        entry = "snb_optim_step_tensors" if self._disc else "snb_adam_step" if self._one_count else "snb_optim_step"
        n_bufs = 2 if self._one_count else 3
        amp_step = False
        for m, bufs, counts in zip(self.models, self._flat, self._counts):
            ps = _params(m)
            dev = ps[0].device
            _check_tensors(ps, type(self).__name__)
            advances = [True] if self._one_count else [p.grad is not None and adv for p in ps]
            parr = (C.c_void_p * len(ps))(*[p.data_ptr() for p in ps])
            garr = (C.c_void_p * len(ps))(*[(p.grad.data_ptr() if p.grad is not None else None) for p in ps])
            st = [_lib.ptr(b) for b in bufs] + [None] * (n_bufs - len(bufs))
            if self._disc:
                head, tail = [len(ps), parr, garr, (C.c_int64 * len(ps))(*[p.numel() for p in ps])], []
            else:
                prec = config.step_precision(self._precision, getattr(m, "_last_prec", None))
                head, tail = [parr, garr], [prec, int(m.use_new_activation), _lib.ptr(m.packed_image_buffer(prec))]
            amp = self._amp_inputs(dev)
            with torch.cuda.device(dev):
                if amp is not None:
                    amp_step = True
                    ctl = self._amp_ctl(counts, advances, amp, dev)
                    _lib.check(getattr(lib, entry + "_amp")(*head, *st, C.byref(args), C.byref(ctl), *tail,
                                                            _lib.stream_ptr(dev)), entry + "_amp")
                    counts.advance(advances)
                    continue
                counts.settle()
                counts.load([c + 1 if a else c for c, a in zip(counts.host, advances)])
                if self._disc:
                    head.append((C.c_int * len(ps))(*counts.host))
                elif self._one_count:
                    args.step = counts.host[0]
                else:
                    args.step[:len(ps)] = counts.host
                _lib.check(getattr(lib, entry)(*head, *st, C.byref(args), *tail, _lib.stream_ptr(dev)), entry)
        if amp_step:
            self._stale = True
        else:
            self._publish()
        return loss

    @staticmethod
    def _amp_ctl(counts: _Counts, advances, amp, dev) -> "_lib.SnbAmpStep":
        """The SnbAmpStep of one module's GradScaler-native step: the device scale and found_inf, the count rows,
        and the window bases."""
        base = counts.prepare(advances, dev)
        count_in, count_out = counts.pointers()
        ctl = _lib.SnbAmpStep(scale=_lib.ptr(amp[0]), found_inf=_lib.ptr(amp[1]), count_in=count_in,
                              count_out=count_out)
        ctl.base[:len(base)] = base
        return ctl


class FusedAdam(_FusedPerTensor):
    """torch.optim.Adam(lr, betas, eps, weight_decay), amsgrad off.  NeRF models: one step count for the optimiser and
    state for every tensor from the first step, the 24-tensor kernel and the re-pack (snb_adam_step).  Discriminator
    modules: torch's per-parameter `step` (a tensor, as torch keeps it) and lazily created state (the per-tensor body
    above, rule SNB_OPTIM_ADAM)."""
    _rule = _lib.OPTIM_ADAM
    _buffers = ("exp_avg", "exp_avg_sq")

    def __init__(self, models: Iterable, lr: float = 5e-4, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, precision: Optional[str] = None, amp_scaling: bool = True):
        super().__init__(models, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), precision, amp_scaling)

    @property
    def _steps(self) -> int:
        """NeRF models: updates applied so far (one count per model; all models step together)."""
        return self._counts[0].host[0]

    def _step_value(self, n):
        return torch.tensor(float(n))

    def _publish(self):
        if self._disc:
            return super()._publish()
        for st in self.__dict__["state"].values():
            st["step"] = torch.tensor(float(self._steps))

    def _args(self, group):
        if self._one_count:
            return _lib.SnbAdamArgs(float(group["lr"]), float(group["betas"][0]), float(group["betas"][1]),
                                    float(group["eps"]), float(group["weight_decay"]), 0)
        return _lib.SnbOptimArgs(rule=self._rule, lr=float(group["lr"]), weight_decay=float(group["weight_decay"]),
                                 beta1=float(group["betas"][0]), beta2=float(group["betas"][1]), eps=float(group["eps"]),
                                 k=1)

    def _ensure_state(self):
        if self._disc:
            return super()._ensure_state()
        if self._flat:
            return
        for m in self.models:
            ps = m._param_list()
            dev = ps[0].device
            _lib.require_device(ps[0], "FusedAdam")
            ea = torch.zeros(_lib.PARAM_FLOATS, device=dev, dtype=torch.float32)
            es = torch.zeros(_lib.PARAM_FLOATS, device=dev, dtype=torch.float32)
            off = 0
            for p in ps:
                n = p.numel()
                self.__dict__["state"][p] = {"step": torch.tensor(float(self._steps)),
                                             "exp_avg": ea[off:off + n].view_as(p),
                                             "exp_avg_sq": es[off:off + n].view_as(p)}
                off += n
            assert off == _lib.PARAM_FLOATS
            self._flat.append((ea, es))

    def load_state_dict(self, state_dict):
        """Values are copied INTO the flat buffers (the kernel addresses them by offset)."""
        if self._disc:
            return super().load_state_dict(state_dict)
        self._ensure_state()
        views = {id(p): dict(st) for p, st in self.state.items()}
        for c in self._counts:
            c.settle()
        torch.optim.Optimizer.load_state_dict(self, state_dict)
        step = 0
        for p, st in self.state.items():
            keep = views[id(p)]
            for k in ("exp_avg", "exp_avg_sq"):
                keep[k].copy_(st[k])
                st[k] = keep[k]
            step = max(step, int(float(st.get("step", 0))))
        for c in self._counts:
            c.load([step])


class FusedSGD(_FusedPerTensor):
    """torch.optim.SGD(lr, momentum, weight_decay) as get_optimizer builds it (reference utils/__init__.py:15-17):
    dampening 0, no Nesterov, the foreach path's arithmetic.  State: `momentum_buffer`, created on a parameter's
    first step with momentum != 0 as a copy of its gradient."""
    _rule = _lib.OPTIM_SGD
    _buffers = ("momentum_buffer",)
    _has_step = False

    def __init__(self, models: Iterable, lr: float, momentum: float = 0.0, weight_decay: float = 0.0,
                 precision: Optional[str] = None,
                 amp_scaling: bool = True):
        super().__init__(models, dict(lr=lr, momentum=momentum, dampening=0.0, weight_decay=weight_decay,
                                      nesterov=False), precision, amp_scaling)

    def _advances(self, group):
        return group["momentum"] != 0

    def _args(self, group):
        if group["dampening"] != 0 or group["nesterov"]:
            raise NotImplementedError("FusedSGD: dampening and Nesterov momentum are not fused (get_optimizer uses neither)")
        return _lib.SnbOptimArgs(rule=self._rule, lr=float(group["lr"]), weight_decay=float(group["weight_decay"]),
                                 momentum=float(group["momentum"]), k=1)


class FusedRAdam(_FusedPerTensor):
    """The reference's RAdam (utils/optimizers.py:7-106, degenerated_to_sgd = True).  State: `step`, `exp_avg`,
    `exp_avg_sq` per parameter.  The param group carries the reference's `buffer` key (its N_sma cache, unused here)
    so that a state dict saved from this optimizer loads into the reference's RAdam."""
    _rule = _lib.OPTIM_RADAM
    _buffers = ("exp_avg", "exp_avg_sq")

    def __init__(self, models: Iterable, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, precision: Optional[str] = None,
                 amp_scaling: bool = True):
        super().__init__(models, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                      buffer=[[None, None, None] for _ in range(10)]), precision, amp_scaling)

    def _args(self, group):
        return _lib.SnbOptimArgs(rule=self._rule, lr=float(group["lr"]), weight_decay=float(group["weight_decay"]),
                                 beta1=float(group["betas"][0]), beta2=float(group["betas"][1]), eps=float(group["eps"]),
                                 k=1)


class FusedRanger(_FusedPerTensor):
    """The reference's Ranger (utils/optimizers.py:292-439): RAdam moments, N_sma > N_sma_threshhold for the adaptive
    step, weight decay on every step, and every k-th step of a parameter slow += alpha * (p - slow), p = slow.
    State: `step`, `exp_avg`, `exp_avg_sq`, `slow_buffer`; param-group keys as the reference spells them."""
    _rule = _lib.OPTIM_RANGER
    _buffers = ("exp_avg", "exp_avg_sq", "slow_buffer")

    def __init__(self, models: Iterable, lr: float = 1e-3, alpha: float = 0.5, k: int = 6,
                 N_sma_threshhold: float = 5, betas=(0.95, 0.999), eps: float = 1e-5, weight_decay: float = 0.0,
                 precision: Optional[str] = None,
                 amp_scaling: bool = True):
        super().__init__(models, dict(lr=lr, alpha=alpha, k=k, step_counter=0, betas=betas,
                                      N_sma_threshhold=N_sma_threshhold, eps=eps, weight_decay=weight_decay), precision, amp_scaling)

    def _args(self, group):
        return _lib.SnbOptimArgs(rule=self._rule, lr=float(group["lr"]), weight_decay=float(group["weight_decay"]),
                                 beta1=float(group["betas"][0]), beta2=float(group["betas"][1]), eps=float(group["eps"]),
                                 n_sma_threshold=float(group["N_sma_threshhold"]), alpha=float(group["alpha"]),
                                 k=int(group["k"]))


def get_optimizer(hparams, models, rate=1):
    """Drop-in for reference utils/__init__.py:10-31: `hparams.optimizer` sgd / adam / radam / ranger with the
    reference's arguments (lr * rate, eps = 1e-8, momentum for sgd, weight_decay), each fused.  `models` is the NeRF
    models (`self.models`) or the discriminator (`[self.D]`, rate=0.2); any other module raises TypeError."""
    lr, wd = hparams.lr * rate, hparams.weight_decay
    if hparams.optimizer == "sgd":
        return FusedSGD(models, lr=lr, momentum=hparams.momentum, weight_decay=wd)
    if hparams.optimizer == "adam":
        return FusedAdam(models, lr=lr, eps=1e-8, weight_decay=wd)
    if hparams.optimizer == "radam":
        return FusedRAdam(models, lr=lr, eps=1e-8, weight_decay=wd)
    if hparams.optimizer == "ranger":
        return FusedRanger(models, lr=lr, eps=1e-8, weight_decay=wd)
    raise ValueError("optimizer not recognized!")
