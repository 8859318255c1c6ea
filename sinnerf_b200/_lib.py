"""ctypes binding of libsinnerf_b200.so (include/sinnerf_b200.h).

There is no CPU or PyTorch fallback anywhere in this package: if the shared library is missing
or the device is not sm_90 (H100), every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
# SNB_LIB_PATH: load another build of the same library (A/B timing of kernel variants by the tools/ scripts)
LIB_PATH = os.environ.get("SNB_LIB_PATH") or os.path.join(_PKG, "libsinnerf_b200.so")

SNB_OK = 0
PRECISIONS = {"fp32": 0, "f16x3": 1, "bf16x3": 2, "bf16": 3}
# Modes kept out of PRECISIONS: the parity tests enumerate that table and hold every mode in it except bf16 / bf16x3 to
# the fp32 bar (1e-4).  The single-product fp16 mode (SNB_PREC_F16, the reference's arithmetic under Lightning's
# precision=16) is not fp32-accurate; it has tests of its own against an oracle with the same operand rounding.
REDUCED_PRECISIONS = {"f16": 4}

c_f = C.c_void_p  # device pointers travel as void*


MAX_PIXEL_DST = 8   # SNB_MAX_PIXEL_DST


class SnbPixelScatter(C.Structure):
    _fields_ = [("dst", c_f * MAX_PIXEL_DST), ("n_dst", C.c_int), ("row_offset", C.c_int64)]


class SnbRenderArgs(C.Structure):
    _fields_ = [
        ("rays", c_f), ("n_rays", C.c_int64), ("n_samples", C.c_int), ("n_importance", C.c_int),
        ("use_disp", C.c_int), ("perturb", C.c_float), ("noise_std", C.c_float), ("white_back", C.c_int),
        ("test_time", C.c_int), ("precision", C.c_int), ("packed_coarse", c_f), ("packed_fine", c_f),
        ("z_steps", c_f), ("u_steps", c_f), ("perturb_u", c_f), ("noise_coarse", c_f), ("pdf_u", c_f),
        ("noise_fine", c_f), ("z_coarse", c_f), ("raw_coarse", c_f), ("rgb_coarse", c_f),
        ("depth_coarse", c_f), ("weights_coarse", c_f), ("z_fine", c_f), ("raw_fine", c_f),
        ("rgb_fine", c_f), ("depth_fine", c_f), ("weights_fine", c_f), ("pixel_scatter", C.POINTER(SnbPixelScatter)),
    ]


class SnbLossSpec(C.Structure):
    _fields_ = [("target_rgb", c_f), ("target_depth", c_f), ("rgb_weight", c_f), ("depth_weight", c_f),
                ("rgb_weight0", C.c_float), ("depth_weight0", C.c_float)]


class SnbAdamArgs(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double), ("step", C.c_int)]


OPTIM_SGD, OPTIM_RADAM, OPTIM_RANGER = 0, 1, 2   # SNB_OPTIM_*


class SnbOptimArgs(C.Structure):
    _fields_ = [("rule", C.c_int), ("lr", C.c_double), ("weight_decay", C.c_double), ("momentum", C.c_double),
                ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_double), ("n_sma_threshold", C.c_double),
                ("alpha", C.c_double), ("k", C.c_int), ("step", C.c_int * 24)]


LOSS_WS_FLOATS = 4096   # SNB_LOSS_WS_FLOATS
PARAM_FLOATS = 595844   # SNB_PARAM_FLOATS

# name -> (restype, argtypes); must list every symbol include/sinnerf_b200.h declares
SIGNATURES = {
    "snb_version": (C.c_int, []),
    "snb_last_error": (C.c_char_p, []),
    "snb_device_check": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "snb_packed_weights_bytes": (C.c_size_t, [C.c_int]),
    "snb_pack_weights": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, c_f, c_f]),
    "snb_refresh_weights": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, c_f, c_f]),
    "snb_sample_coarse": (C.c_int, [c_f, c_f, c_f, C.c_float, C.c_int, C.c_int64, C.c_int, c_f, c_f]),
    "snb_embed": (C.c_int, [c_f, C.c_int64, C.c_int, C.c_int, c_f, c_f]),
    "snb_mlp_forward": (C.c_int, [c_f, C.c_int, c_f, C.c_int64, C.c_int64, C.c_int, c_f, c_f]),
    "snb_field_forward": (C.c_int, [c_f, C.c_int, c_f, c_f, C.c_int64, C.c_int, C.c_int, c_f, c_f]),
    "snb_composite_forward": (C.c_int, [c_f, C.c_int, c_f, c_f, c_f, C.c_float, C.c_int, C.c_int64, C.c_int,
                                        c_f, c_f, c_f, c_f]),
    "snb_composite_forward_scatter": (C.c_int, [c_f, c_f, c_f, c_f, C.c_float, C.c_int, C.c_int64, C.c_int,
                                                c_f, c_f, c_f, C.POINTER(SnbPixelScatter), c_f]),
    "snb_sample_pdf": (C.c_int, [c_f, C.c_int64, c_f, C.c_int64, c_f, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                 C.c_float, c_f, c_f]),
    "snb_importance_merge": (C.c_int, [c_f, c_f, c_f, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_float, c_f,
                                       c_f, c_f]),
    "snb_render_forward": (C.c_int, [C.POINTER(SnbRenderArgs), c_f]),
    "snb_generate_rays": (C.c_int, [C.POINTER(C.c_float)] + [C.c_float] * 6 + [C.c_int] * 6 + [c_f, c_f]),
    "snb_field_forward_train": (C.c_int, [c_f, C.c_int, c_f, c_f, C.c_int64, C.c_int, c_f, c_f, c_f, c_f, c_f, c_f]),
    "snb_composite_backward": (C.c_int, [c_f, c_f, c_f, c_f, C.c_float, C.c_int, c_f, c_f, c_f, C.c_int64, C.c_int,
                                         c_f, c_f]),
    "snb_composite_forward_loss": (C.c_int, [c_f, c_f, c_f, c_f, C.c_float, C.c_int, C.c_int64, C.c_int,
                                             C.POINTER(SnbLossSpec), c_f, c_f, c_f, c_f, c_f, c_f]),
    "snb_composite_backward_loss": (C.c_int, [c_f, c_f, c_f, c_f, C.c_float, C.c_int, c_f, c_f, c_f,
                                              C.POINTER(SnbLossSpec), c_f, c_f, c_f, C.c_int64, C.c_int, c_f, c_f, c_f]),
    "snb_act16_bytes": (C.c_size_t, [C.c_int64]),
    "snb_bwd16_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "snb_field_forward_train16": (C.c_int, [c_f, C.c_int, c_f, c_f, C.c_int64, C.c_int, c_f, c_f, c_f]),
    "snb_field_backward16": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, c_f, c_f, c_f, C.c_int64,
                                       c_f, c_f, c_f]),
    "snb_adam_step": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), c_f, c_f, C.POINTER(SnbAdamArgs),
                                C.c_int, C.c_int, c_f, c_f]),
    "snb_optim_step": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), c_f, c_f, c_f, C.POINTER(SnbOptimArgs),
                                 C.c_int, C.c_int, c_f, c_f]),
    "snb_field_backward": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, c_f, c_f, c_f, c_f, c_f,
                                     c_f, C.c_int64, c_f, c_f, c_f, c_f, c_f, c_f]),
    "snb_field_forward_train_sigma": (C.c_int, [c_f, C.c_int, c_f, c_f, C.c_int64, C.c_int, c_f, c_f, c_f, c_f]),
    "snb_field_forward_train16_sigma": (C.c_int, [c_f, C.c_int, c_f, c_f, C.c_int64, C.c_int, c_f, c_f, c_f]),
    "snb_composite_backward_weights": (C.c_int, [c_f, c_f, c_f, c_f, C.c_float, c_f, C.c_int64, C.c_int, c_f, c_f, c_f]),
    "snb_field_backward_sigma": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), c_f, c_f, c_f, C.c_int64,
                                           c_f, c_f, c_f, c_f]),
    "snb_field_backward16_sigma": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), c_f, c_f, C.c_int64, c_f,
                                             c_f, c_f]),
    "snb_depth_smooth_forward": (C.c_int, [c_f, C.POINTER(C.c_int64), c_f, C.POINTER(C.c_int64), C.c_int64, C.c_int,
                                           C.c_int, C.c_int, c_f, c_f, c_f]),
    "snb_depth_smooth_backward": (C.c_int, [c_f, C.POINTER(C.c_int64), c_f, C.POINTER(C.c_int64), C.c_int64, C.c_int,
                                            C.c_int, C.c_int, c_f, c_f, C.POINTER(C.c_int64), c_f, C.POINTER(C.c_int64),
                                            c_f]),
    "snb_ssim_loss_forward": (C.c_int, [c_f, C.POINTER(C.c_int64), c_f, C.POINTER(C.c_int64), C.c_int64, C.c_int,
                                        C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, c_f, c_f, c_f, c_f]),
    "snb_ssim_loss_backward": (C.c_int, [c_f, C.POINTER(C.c_int64), c_f, C.POINTER(C.c_int64), C.c_int64, C.c_int,
                                         C.c_int, C.c_int, c_f, c_f, c_f, C.POINTER(C.c_int64), c_f]),
    "snb_forward_warp_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int, C.c_int]),
    "snb_forward_warp": (C.c_int, [c_f, c_f, C.c_int, C.c_int, c_f, C.c_int64, C.c_int, c_f, c_f, c_f, c_f, c_f]),
    "snb_vit_pack_bytes": (C.c_size_t, [C.c_int]),
    "snb_vit_pack": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, c_f, c_f]),
    "snb_vit_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "snb_vit_forward": (C.c_int, [c_f, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int),
                                  C.c_int, C.c_int, c_f, c_f, c_f]),
    "snb_vit_backward": (C.c_int, [c_f, C.c_int, C.POINTER(C.c_int), C.c_int, c_f, C.POINTER(C.c_void_p),
                                   C.POINTER(C.c_int64), c_f, c_f]),
}
VIT_N_TENSORS = 148       # SNB_VIT_N_TENSORS
VIT_MAX_IMAGES = 8        # SNB_VIT_MAX_IMAGES
WARP_OCCLUSION = {"zbuffer": 0, "last": 1}   # SNB_WARP_*
BWD_WS_FLOATS = 2 * 128 * 256 + 128   # SNB_BWD_WS_FLOATS

_lib = None


def load() -> C.CDLL:
    """Load the library (once).  Raises if it has not been built -- never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m sinnerf_b200.build` "
                "(sinnerf_b200 has no CPU / PyTorch fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(rc: int, what: str) -> None:
    if rc != SNB_OK:
        msg = load().snb_last_error().decode(errors="replace")
        exc = {-1: ValueError, -3: NotImplementedError}.get(rc, RuntimeError)
        raise exc(f"{what} failed ({rc}): {msg}")


_checked_devices = set()


def require_device(t: torch.Tensor, what: str) -> None:
    """The product path is CUDA sm_90 only; anything else is an error, not a fallback."""
    if not t.is_cuda:
        raise RuntimeError(f"sinnerf_b200.{what}: expected a CUDA tensor, got device '{t.device}' "
                           "(this package has no CPU path)")
    idx = t.device.index if t.device.index is not None else torch.cuda.current_device()
    if idx not in _checked_devices:
        with torch.cuda.device(idx):
            check(load().snb_device_check(None, None, None), "snb_device_check")
        _checked_devices.add(idx)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def precision_id(name) -> int:
    if isinstance(name, int):
        return name
    mode = PRECISIONS.get(name, REDUCED_PRECISIONS.get(name))
    if mode is None:
        raise ValueError(f"unknown precision '{name}'; choose one of {sorted(PRECISIONS) + sorted(REDUCED_PRECISIONS)}")
    return mode
