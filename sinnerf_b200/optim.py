"""Fused Adam for the NeRF MLPs (SURVEY 8f-4): `torch.optim.Adam` as the reference's `get_optimizer` configures
it (reference utils/__init__.py:10-31: lr, eps = 1e-8, weight_decay) with the whole update of one model --
all 24 tensors -- in ONE sm_90a kernel, followed on the same stream by the re-pack of the weight image the
field kernels stream, so the next forward finds it up to date (and stamped clean) without re-packing.

`FusedAdam` is a `torch.optim.Optimizer`: `param_groups[0]['lr']` is honoured every step, so the reference's
schedulers (utils/__init__.py:34-58, warm-up included) keep working; under DDP it is stepped after the
gradient all-reduce exactly like torch's Adam (train.py:51-52).  State (`exp_avg`, `exp_avg_sq`) is one flat
fp32 buffer per model; `state_dict()` exposes per-parameter views with torch.optim.Adam's key names.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional

import torch

from . import _lib, config
from .nerf import NeRF

__all__ = ["FusedAdam", "get_optimizer"]


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
        prec = _lib.precision_id(config.get_precision() if self._precision is None else self._precision)
        for m, (ea, es) in zip(self.models, self._flat):
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


def get_optimizer(hparams, models, rate=1):
    """Drop-in for reference utils/__init__.py:10-31 when `hparams.optimizer == 'adam'` (the default, opt.py:45):
    same lr / eps / weight_decay.  The reference's other optimizers (sgd / radam / ranger) are its own Python
    code and keep working on these modules unchanged -- packed_weights() notices their in-place updates."""
    if hparams.optimizer != "adam":
        raise NotImplementedError(f"sinnerf_b200.optim.get_optimizer: '{hparams.optimizer}' is not fused; use the "
                                  "reference's utils.get_optimizer for it")
    return FusedAdam(models, lr=hparams.lr * rate, eps=1e-8, weight_decay=hparams.weight_decay)
