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
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional

import torch

from . import _lib, config
from .nerf import NeRF

__all__ = ["FusedAdam", "FusedSGD", "FusedRAdam", "FusedRanger", "get_optimizer"]


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, models: Iterable[NeRF], lr: float = 5e-4, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, precision: Optional[str] = None):
        self.models: List[NeRF] = list(models)
        if not self.models or not all(isinstance(m, NeRF) for m in self.models):
            raise TypeError("FusedAdam steps sinnerf_b200.NeRF models (pass the modules, not their parameters)")
        params = [p for m in self.models for p in m._param_list()]
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._precision = precision
        self._flat = []          # per model: (exp_avg, exp_avg_sq) flat device buffers
        self._steps = 0

    def _ensure_state(self):
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
                self.state[p] = {"step": torch.tensor(float(self._steps)), "exp_avg": ea[off:off + n].view_as(p),
                                 "exp_avg_sq": es[off:off + n].view_as(p)}
                off += n
            assert off == _lib.PARAM_FLOATS
            self._flat.append((ea, es))

    def load_state_dict(self, state_dict):
        """Values are copied INTO the flat buffers (the kernel addresses them by offset)."""
        self._ensure_state()
        views = {id(p): dict(st) for p, st in self.state.items()}
        super().load_state_dict(state_dict)
        step = 0
        for p, st in self.state.items():
            keep = views[id(p)]
            for k in ("exp_avg", "exp_avg_sq"):
                keep[k].copy_(st[k])
                st[k] = keep[k]
            step = max(step, int(float(st.get("step", 0))))
        self._steps = step

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self._ensure_state()
        lib = _lib.load()
        g = self.param_groups[0]
        self._steps += 1
        args = _lib.SnbAdamArgs(float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]),
                                float(g["weight_decay"]), self._steps)
        for m, (ea, es) in zip(self.models, self._flat):
            prec = config.step_precision(self._precision, getattr(m, "_last_prec", None))
            ps = m._param_list()
            dev = ps[0].device
            for p in ps:
                if p.dtype != torch.float32 or not p.is_contiguous() or (p.grad is not None and not p.grad.is_contiguous()):
                    raise ValueError("FusedAdam: parameters and gradients must be contiguous fp32 CUDA tensors")
            image = m.packed_image_buffer(prec)
            parr = (C.c_void_p * 24)(*[p.data_ptr() for p in ps])
            garr = (C.c_void_p * 24)(*[(p.grad.data_ptr() if p.grad is not None else None) for p in ps])
            with torch.cuda.device(dev):
                _lib.check(lib.snb_adam_step(parr, garr, _lib.ptr(ea), _lib.ptr(es), C.byref(args), prec,
                                             int(m.use_new_activation), _lib.ptr(image), _lib.stream_ptr(dev)),
                           "snb_adam_step")
        for st in self.state.values():
            st["step"] = torch.tensor(float(self._steps))
        return loss


class _FusedPerTensor(torch.optim.Optimizer):
    """Shared body of FusedSGD / FusedRAdam / FusedRanger (C ABI snb_optim_step): one kernel per model and step, then
    the re-pack of the weight image on the same stream.

    These rules keep a step count per parameter and skip parameters without a gradient, so the count is tracked per
    tensor (`_count`) and passed to the kernel per tensor.  State mirrors the reference's exactly: a parameter has a
    `state` entry only once it has been stepped, holding views of the flat buffers the kernel updates."""
    _rule: int
    _buffers: tuple          # state keys of the flat buffers, in snb_optim_step's argument order
    _has_step: bool = True   # the state carries the reference's per-parameter `step`

    def __init__(self, models: Iterable[NeRF], defaults: dict, precision: Optional[str]):
        self.models: List[NeRF] = list(models)
        if not self.models or not all(isinstance(m, NeRF) for m in self.models):
            raise TypeError(f"{type(self).__name__} steps sinnerf_b200.NeRF models (pass the modules, not their parameters)")
        super().__init__([p for m in self.models for p in m._param_list()], defaults)
        self._precision = precision
        self._flat = []          # per model: the flat state buffers, in _buffers order
        self._views = {}         # parameter -> {state key: view of its slice of the flat buffer}
        self._count = {}         # parameter -> updates applied so far (the reference's state['step'])

    def _ensure_state(self):
        if self._flat:
            return
        for m in self.models:
            ps = m._param_list()
            _lib.require_device(ps[0], type(self).__name__)
            bufs = [torch.zeros(_lib.PARAM_FLOATS, device=ps[0].device, dtype=torch.float32) for _ in self._buffers]
            off = 0
            for p in ps:
                n = p.numel()
                self._views[p] = {k: b[off:off + n].view_as(p) for k, b in zip(self._buffers, bufs)}
                self._count[p] = 0
                off += n
            assert off == _lib.PARAM_FLOATS
            self._flat.append(bufs)

    def _publish(self):
        self.state.clear()
        for p, n in self._count.items():
            if n > 0:
                self.state[p] = dict(self._views[p], **({"step": n} if self._has_step else {}))

    def load_state_dict(self, state_dict):
        """Values are copied INTO the flat buffers (the kernel addresses them by offset); a parameter without state
        starts afresh, as in the reference."""
        self._ensure_state()
        super().load_state_dict(state_dict)
        for p, views in self._views.items():
            st = self.state.get(p, {})
            if all(st.get(k) is not None for k in self._buffers):
                for k, v in views.items():
                    v.copy_(st[k])
                self._count[p] = int(st["step"]) if self._has_step else 1
            else:
                for v in views.values():
                    v.zero_()
                self._count[p] = 0
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
        for m, bufs in zip(self.models, self._flat):
            prec = config.step_precision(self._precision, getattr(m, "_last_prec", None))
            ps = m._param_list()
            dev = ps[0].device
            for p in ps:
                if p.dtype != torch.float32 or not p.is_contiguous() or (p.grad is not None and not p.grad.is_contiguous()):
                    raise ValueError(f"{type(self).__name__}: parameters and gradients must be contiguous fp32 CUDA tensors")
            for i, p in enumerate(ps):
                if p.grad is not None and adv:
                    self._count[p] += 1
                args.step[i] = self._count[p]
            image = m.packed_image_buffer(prec)
            parr = (C.c_void_p * 24)(*[p.data_ptr() for p in ps])
            garr = (C.c_void_p * 24)(*[(p.grad.data_ptr() if p.grad is not None else None) for p in ps])
            st = [_lib.ptr(b) for b in bufs] + [None] * (3 - len(bufs))
            with torch.cuda.device(dev):
                _lib.check(lib.snb_optim_step(parr, garr, *st, C.byref(args), prec, int(m.use_new_activation),
                                              _lib.ptr(image), _lib.stream_ptr(dev)), "snb_optim_step")
        self._publish()
        return loss


class FusedSGD(_FusedPerTensor):
    """torch.optim.SGD(lr, momentum, weight_decay) as get_optimizer builds it (reference utils/__init__.py:15-17):
    dampening 0, no Nesterov, the foreach path's arithmetic.  State: `momentum_buffer`, created on a parameter's
    first step with momentum != 0 as a copy of its gradient."""
    _rule = _lib.OPTIM_SGD
    _buffers = ("momentum_buffer",)
    _has_step = False

    def __init__(self, models: Iterable[NeRF], lr: float, momentum: float = 0.0, weight_decay: float = 0.0,
                 precision: Optional[str] = None):
        super().__init__(models, dict(lr=lr, momentum=momentum, dampening=0.0, weight_decay=weight_decay,
                                      nesterov=False), precision)

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

    def __init__(self, models: Iterable[NeRF], lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, precision: Optional[str] = None):
        super().__init__(models, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                      buffer=[[None, None, None] for _ in range(10)]), precision)

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

    def __init__(self, models: Iterable[NeRF], lr: float = 1e-3, alpha: float = 0.5, k: int = 6,
                 N_sma_threshhold: float = 5, betas=(0.95, 0.999), eps: float = 1e-5, weight_decay: float = 0.0,
                 precision: Optional[str] = None):
        super().__init__(models, dict(lr=lr, alpha=alpha, k=k, step_counter=0, betas=betas,
                                      N_sma_threshhold=N_sma_threshhold, eps=eps, weight_decay=weight_decay), precision)

    def _args(self, group):
        return _lib.SnbOptimArgs(rule=self._rule, lr=float(group["lr"]), weight_decay=float(group["weight_decay"]),
                                 beta1=float(group["betas"][0]), beta2=float(group["betas"][1]), eps=float(group["eps"]),
                                 n_sma_threshold=float(group["N_sma_threshhold"]), alpha=float(group["alpha"]),
                                 k=int(group["k"]))


def get_optimizer(hparams, models, rate=1):
    """Drop-in for reference utils/__init__.py:10-31: `hparams.optimizer` sgd / adam / radam / ranger with the
    reference's arguments (lr * rate, eps = 1e-8, momentum for sgd, weight_decay), each fused."""
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
