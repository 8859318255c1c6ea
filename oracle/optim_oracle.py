"""Oracle for the optimiser steps `sinnerf_b200.optim` fuses besides Adam: SGD, RAdam and Ranger.

TEST INFRASTRUCTURE ONLY.  A restatement, with plain torch ops in the reference's order, of the rules
`get_optimizer` (reference utils/__init__.py:10-31) builds for `--optimizer sgd|radam|ranger`:
torch.optim.SGD, and the reference's own RAdam and Ranger (utils/optimizers.py).  The reference calls
overloads torch has deprecated (`addcmul_(value, t1, t2)`, `add_(alpha, t)`, `addcdiv_(value, t1, t2)`);
this file uses the keyword forms, which run the same ATen kernels.

Device-agnostic: the optimisers step whatever tensors they are given (CPU for the fixture test, CUDA for the
comparison with the fused kernels).  State uses the reference's key names and layout (per-parameter `step`
as a python int, `exp_avg`, `exp_avg_sq`, `slow_buffer`, `momentum_buffer`; param-group keys as the
reference spells them), so state dicts move between these classes, the reference's and the fused ones.

Parity pin: `tests/golden/make_optim_golden.py` runs the reference's RAdam / Ranger and torch's SGD on seeded
tensors of the NeRF shapes and commits digests of the results as `tests/golden/optim_steps.npz`;
`tests/test_optim_cpu.py` checks this file against them bit for bit.
"""
from __future__ import annotations

import math

import torch
from torch.optim import Optimizer


def rectification(step: int, beta1: float, beta2: float, adaptive_if) -> tuple:
    """(adaptive, step_size) of RAdam's step `step` (utils/optimizers.py:68-86, Ranger :397-411), in python doubles
    and the reference's expression order.  `adaptive_if(N_sma)` is the rule's threshold test; when it fails the step
    degenerates to SGD with momentum (RAdam's default degenerated_to_sgd, Ranger always)."""
    beta2_t = beta2 ** step
    n_sma_max = 2 / (1 - beta2) - 1
    n_sma = n_sma_max - 2 * step * beta2_t / (1 - beta2_t)
    if adaptive_if(n_sma):
        return True, math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_sma_max - 4) * (n_sma - 2) / n_sma * n_sma_max
                               / (n_sma_max - 2)) / (1 - beta1 ** step)
    return False, 1.0 / (1 - beta1 ** step)


def _moments(state, grad, beta1, beta2):
    # utils/optimizers.py:65-66 (Ranger :393-395)
    state["exp_avg_sq"].mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    state["exp_avg"].mul_(beta1).add_(grad, alpha=1 - beta1)


def _rectified_update(p, state, group, adaptive, step_size):
    # utils/optimizers.py:90-104 (Ranger :416-425): decay, then the adaptive or the momentum-only update
    if group["weight_decay"] != 0:
        p.add_(p, alpha=-group["weight_decay"] * group["lr"])
    if adaptive:
        denom = state["exp_avg_sq"].sqrt().add_(group["eps"])
        p.addcdiv_(state["exp_avg"], denom, value=-step_size * group["lr"])
    else:
        p.add_(state["exp_avg"], alpha=-step_size * group["lr"])


class SGD(Optimizer):
    """torch.optim.SGD(lr, momentum, weight_decay) as get_optimizer builds it (utils/__init__.py:15-17): dampening 0,
    no Nesterov; the per-element operations of torch/optim/sgd.py."""

    def __init__(self, params, lr, momentum=0.0, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=0.0, weight_decay=weight_decay,
                                      nesterov=False))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                d = p.grad if group["weight_decay"] == 0 else p.grad.add(p, alpha=group["weight_decay"])
                if group["momentum"] != 0:
                    state = self.state[p]
                    buf = state.get("momentum_buffer")
                    if buf is None:
                        buf = state["momentum_buffer"] = d.clone()
                    else:
                        buf.mul_(group["momentum"]).add_(d, alpha=1 - group["dampening"])
                    d = buf
                p.add_(d, alpha=-group["lr"])


class RAdam(Optimizer):
    """utils/optimizers.py:7-106 with degenerated_to_sgd = True (the default; get_optimizer passes lr, eps,
    weight_decay: utils/__init__.py:22-24)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:                                   # :42-43
                    continue
                state = self.state[p]
                if not state:                                        # :53-56
                    state.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p))
                _moments(state, p.grad, beta1, beta2)
                state["step"] += 1
                adaptive, step_size = rectification(state["step"], beta1, beta2, lambda n: n >= 5)
                _rectified_update(p, state, group, adaptive, step_size)


class Ranger(Optimizer):
    """utils/optimizers.py:292-439: RAdam with Ranger's defaults and a strict threshold, weight decay applied on every
    step, and a lookahead every k-th step of a parameter (get_optimizer passes lr, eps, weight_decay:
    utils/__init__.py:25-27)."""

    def __init__(self, params, lr=1e-3, alpha=0.5, k=6, N_sma_threshhold=5, betas=(0.95, 0.999), eps=1e-5,
                 weight_decay=0.0):
        super().__init__(params, dict(lr=lr, alpha=alpha, k=k, step_counter=0, betas=betas,
                                      N_sma_threshhold=N_sma_threshhold, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:                                   # :360-361
                    continue
                state = self.state[p]
                if not state:                                        # :371-381: the slow copy is taken before the update
                    state.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p),
                                 slow_buffer=p.clone())
                _moments(state, p.grad, beta1, beta2)
                state["step"] += 1
                adaptive, step_size = rectification(state["step"], beta1, beta2,
                                                    lambda n: n > group["N_sma_threshhold"])
                _rectified_update(p, state, group, adaptive, step_size)
                if state["step"] % group["k"] == 0:                  # :431-437
                    slow = state["slow_buffer"]
                    slow.add_(p - slow, alpha=group["alpha"])
                    p.copy_(slow)
