"""Process-wide settings of the sm_90a path."""
import os

import torch

# default: the fp32-parity tensor-core mode (validated against the oracle at <= 1e-4)
_precision = os.environ.get("SINNERF_B200_PRECISION", "f16x3")

# The precision policy: not a mode of its own, it picks one per pass from CUDA autocast (resolve_precision)
AUTOCAST = "autocast"
_AUTOCAST_MODES = {torch.float16: "f16", torch.bfloat16: "bf16"}
_NOW = object()


def set_precision(name: str) -> None:
    """Arithmetic of the field MLP: 'fp32' (FFMA, exact), 'f16x3' / 'bf16x3' (wgmma, split operands,
    fp32-parity), 'bf16' / 'f16' (wgmma single pass; 'f16' is the reference's arithmetic under Lightning's
    precision=16), or 'autocast': per pass, 'f16' inside fp16 CUDA autocast, 'bf16' inside bf16 autocast and
    'f16x3' outside it.  Everything outside the MLP is always fp32."""
    from . import _lib
    if name != AUTOCAST:
        _lib.precision_id(name)
    global _precision
    _precision = name


def get_precision() -> str:
    return _precision


def resolve_precision(precision=None, autocast_dtype=_NOW) -> int:
    """The SNB_PREC_* id a pass runs in: `precision` (a mode name, an id or 'autocast'), else the process setting.
    'autocast' follows `autocast_dtype` (None: autocast off), by default the CUDA autocast state of the calling thread."""
    from . import _lib
    name = _precision if precision is None else precision
    if name == AUTOCAST:
        if autocast_dtype is _NOW:
            autocast_dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else None
        name = _AUTOCAST_MODES.get(autocast_dtype, "f16x3")
    return _lib.precision_id(name)


def step_precision(precision, last_pass) -> int:
    """The SNB_PREC_* id whose weight image a fused optimiser re-packs after its step.  Under 'autocast' that is the
    mode of the model's last pass (`last_pass`, None before the first): the step runs outside the autocast region the
    passes run in (`scaler.step(opt)` after the forward), where the policy would name another image."""
    name = _precision if precision is None else precision
    if name == AUTOCAST and last_pass is not None:
        return last_pass
    return resolve_precision(precision)


# Training path: how the activations the backward needs are kept.  'fp16' (default for the tensor-core modes):
# one fp16 copy in the MMA-ready tile layout + power-of-two scaled fp16 gradients between layers, backward on
# tensor cores (half the HBM traffic and memory; parameter gradients within the 1e-3 parity bar).  'fp32':
# row-major fp32 activations and the fp32-input tensor-core backward (bf16 hi/lo split; the only option of precision
# 'fp32').
_train_storage = os.environ.get("SINNERF_B200_TRAIN_STORAGE", "fp16")


def set_train_storage(name: str) -> None:
    if name not in ("fp16", "fp32"):
        raise ValueError("train storage must be 'fp16' or 'fp32'")
    global _train_storage
    _train_storage = name


def get_train_storage() -> str:
    return _train_storage
