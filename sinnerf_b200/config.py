"""Process-wide settings of the sm_90a path."""
import os

# default: the fp32-parity tensor-core mode (validated against the oracle at <= 1e-4)
_precision = os.environ.get("SINNERF_B200_PRECISION", "f16x3")


def set_precision(name: str) -> None:
    """Arithmetic of the field MLP: 'fp32' (FFMA, exact), 'f16x3' / 'bf16x3' (wgmma, split operands,
    fp32-parity), 'bf16' (wgmma single pass).  Everything outside the MLP is always fp32."""
    from . import _lib
    _lib.precision_id(name)
    global _precision
    _precision = name


def get_precision() -> str:
    return _precision


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
