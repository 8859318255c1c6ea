"""SinNeRF's semantic loss: the DINO ViT-S/16 CLS feature of rendered patches (models/sinnerf.py:162-169, :332-338),
forward and input gradient executed by libsinnerf_b200's sm_90a kernels (csrc/vit.cu).

    from sinnerf_b200.vit import load_dino_weights
    self.ext = load_dino_weights().to(self.device)          # models/sinnerf.py:148-149, no network
    ...
    return self.ext.cls_feature(x)                          # body of get_vit_feature

`DinoViTS16` holds DINO vit_small/16's weights as frozen parameters under the names of the reference's
`VitExtractor` (`model.cls_token`, `model.blocks.0.attn.qkv.weight`, ...), so a SinNeRF checkpoint's `ext.model.*`
entries load with strict=True, and DDP neither reduces nor broadcasts them.  It has no `forward`: the feature is
`cls_feature(x)` (get_vit_feature: nearest resize to 224 x 224, ImageNet normalisation, block 11's output at token 0
of image 0), differentiable in x only, and `semantic_loss(ref, coarse, fine)` runs both rendered patches through one
batched forward and one batched backward.

Inputs are (B, 3, h, w) fp32 CUDA tensors read through their strides (the '(b p q) c -> b c p q' views of
render_rays' ray-major outputs are not copied); only image 0 of each is used, and gradients come back with the input's
strides, zero on images 1..B-1.  The GEMM arithmetic follows `precision=` or the process setting
(config.resolve_precision): 'f16x3', 'bf16x3' and 'fp32' use the fp16 hi + lo three-product split (fp32 parity),
'f16' and 'bf16' one product; under 'autocast', fp16 autocast gives 'f16', the reference's arithmetic under
Lightning's precision=16.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
from torch import nn
import torch.nn.functional as F

from . import _lib
from .config import resolve_precision

__all__ = ["DinoViTS16", "load_dino_weights", "DINO_FILE", "default_weights_path"]

DIM, DEPTH, MLP, TOKENS = 384, 12, 1536, 197
DINO_FILE = "dino_deitsmall16_pretrain.pth"   # the released backbone; torch.hub caches it under checkpoints/


class _Attn(nn.Module):
    def __init__(self):
        super().__init__()
        self.qkv = nn.Linear(DIM, 3 * DIM)
        self.proj = nn.Linear(DIM, DIM)


class _Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(DIM, MLP)
        self.fc2 = nn.Linear(MLP, DIM)


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.norm1 = nn.LayerNorm(DIM, eps=1e-6)
        self.attn = _Attn()
        self.norm2 = nn.LayerNorm(DIM, eps=1e-6)
        self.mlp = _Mlp()


class _PatchEmbed(nn.Module):
    def __init__(self):
        super().__init__()
        self.proj = nn.Conv2d(3, DIM, 16, 16)


class _Backbone(nn.Module):
    """DINO vit_small(patch_size=16) parameter layout (its state-dict keys and order); no forward of its own."""

    def __init__(self):
        super().__init__()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, DIM))
        self.pos_embed = nn.Parameter(torch.zeros(1, TOKENS, DIM))
        self.patch_embed = _PatchEmbed()
        self.blocks = nn.ModuleList([_Block() for _ in range(DEPTH)])
        self.norm = nn.LayerNorm(DIM, eps=1e-6)


def _kernel_params(model: _Backbone):
    """The SNB_VIT_N_TENSORS tensors of the weight image, in the C ABI's order (state-dict order without norm.*)."""
    ps = [model.cls_token, model.pos_embed, model.patch_embed.proj.weight, model.patch_embed.proj.bias]
    for b in model.blocks:
        ps += [b.norm1.weight, b.norm1.bias, b.attn.qkv.weight, b.attn.qkv.bias, b.attn.proj.weight, b.attn.proj.bias,
               b.norm2.weight, b.norm2.bias, b.mlp.fc1.weight, b.mlp.fc1.bias, b.mlp.fc2.weight, b.mlp.fc2.bias]
    assert len(ps) == _lib.VIT_N_TENSORS
    return ps


def _check_image(x, name: str, what: str) -> None:
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"{what}: {name} is not a torch.Tensor (got {type(x)})")
    if x.dim() != 4 or x.shape[0] < 1 or x.shape[1] != 3 or x.shape[2] < 1 or x.shape[3] < 1:
        raise ValueError(f"{what}: invalid {name} shape, we expect Bx3xHxW with B, H, W >= 1. Got: {tuple(x.shape)}")
    _lib.require_device(x, what)
    if x.dtype != torch.float32:
        raise TypeError(f"{what}: {name} must be float32 (got {x.dtype})")


def _arrays(imgs):
    """host arrays of the C ABI for image 0 of each tensor: pointers, (c, h, w) strides, (h, w) sizes"""
    n = len(imgs)
    ptrs = (C.c_void_p * n)(*[x.data_ptr() for x in imgs])
    strides = (C.c_int64 * (3 * n))(*[s for x in imgs for s in x.stride()[1:]])
    sizes = (C.c_int * (2 * n))(*[s for x in imgs for s in x.shape[2:]])
    return ptrs, strides, sizes


class _ClsFeatures(torch.autograd.Function):
    """features (n, 384) of image 0 of each of n tensors; backward to those tensors"""

    @staticmethod
    def forward(ctx, packed, mode, save, *imgs):
        lib = _lib.load()
        n = len(imgs)
        dev = imgs[0].device
        ws = torch.empty(lib.snb_vit_workspace_bytes(n, int(save)), device=dev, dtype=torch.uint8)
        out = torch.empty(n, DIM, device=dev, dtype=torch.float32)
        ptrs, strides, sizes = _arrays(imgs)
        _lib.check(lib.snb_vit_forward(_lib.ptr(packed), mode, ptrs, strides, sizes, n, int(save), _lib.ptr(out),
                                       _lib.ptr(ws), _lib.stream_ptr(dev)), "snb_vit_forward")
        if save:
            ctx.save_for_backward(packed, ws, *imgs)
            ctx.mode = mode
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        packed, ws, *imgs = ctx.saved_tensors
        g = g.detach().to(torch.float32).contiguous()
        # zeros_like keeps the input's strides (a permuted view stays permuted); the kernels write image 0 of each
        grads = [torch.zeros_like(x) for x in imgs]
        n = len(imgs)
        _, _, sizes = _arrays(imgs)
        ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in grads])
        strides = (C.c_int64 * (3 * n))(*[s for t in grads for s in t.stride()[1:]])
        _lib.check(lib.snb_vit_backward(_lib.ptr(packed), ctx.mode, sizes, n, _lib.ptr(g), ptrs, strides, _lib.ptr(ws),
                                        _lib.stream_ptr(g.device)), "snb_vit_backward")
        return (None, None, None, *[gr if need else None for gr, need in zip(grads, ctx.needs_input_grad[3:])])


class DinoViTS16(nn.Module):
    """DINO ViT-S/16 as SinNeRF's VitExtractor uses it: frozen weights under `model.*`, the CLS feature of block 11."""

    def __init__(self):
        super().__init__()
        self.model = _Backbone()
        self.requires_grad_(False)
        self._images = {}      # (device, mode) -> (parameter key, packed image)

    def packed(self, device, mode: int) -> torch.Tensor:
        """The weight image of `mode` on `device`, packed once and re-packed only when a weight tensor's data pointer
        or version counter changes."""
        ps = _kernel_params(self.model)
        for p in ps:
            if p.device != device or p.dtype != torch.float32:
                raise RuntimeError(f"DinoViTS16: weights are {p.dtype} on {p.device}; move the module to {device} "
                                   "(.to(device)) in float32")
        if not all(p.is_contiguous() for p in ps):
            raise RuntimeError("DinoViTS16: weight tensors must be contiguous")
        key = tuple((p.data_ptr(), p._version) for p in ps)
        hit = self._images.get((str(device), mode))
        if hit is not None and hit[0] == key:
            return hit[1]
        lib = _lib.load()
        img = torch.empty(lib.snb_vit_pack_bytes(mode), device=device, dtype=torch.uint8)
        ptrs = (C.c_void_p * len(ps))(*[p.data_ptr() for p in ps])
        _lib.check(lib.snb_vit_pack(ptrs, mode, _lib.ptr(img), _lib.stream_ptr(device)), "snb_vit_pack")
        self._images[(str(device), mode)] = (key, img)
        return img

    def _features(self, imgs, precision):
        what = "DinoViTS16"
        if len(imgs) > _lib.VIT_MAX_IMAGES:
            raise ValueError(f"{what}: at most {_lib.VIT_MAX_IMAGES} images per pass (got {len(imgs)})")
        dev = imgs[0].device
        for x in imgs:
            if x.device != dev:
                raise ValueError(f"{what}: inputs must be on one device. Got: {dev} and {x.device}")
        mode = resolve_precision(precision)
        # under torch.no_grad() (the reference's ref_ refresh) the pass keeps nothing for a backward
        save = torch.is_grad_enabled() and any(x.requires_grad for x in imgs)
        return _ClsFeatures.apply(self.packed(dev, mode), mode, save, *imgs)

    def cls_feature(self, x: torch.Tensor, precision=None) -> torch.Tensor:
        """get_vit_feature(x) (models/sinnerf.py:162-169): x (B, 3, h, w) -> (384,), the block-11 output at token 0
        of image 0 after a nearest resize to 224 x 224 and ImageNet normalisation.  Differentiable in x; under
        torch.no_grad() the pass keeps nothing for a backward."""
        _check_image(x, "x", "cls_feature")
        return self._features([x], precision)[0]

    def semantic_loss(self, ref: torch.Tensor, coarse: torch.Tensor, fine: torch.Tensor, precision=None) -> torch.Tensor:
        """mse(f(coarse), ref) + mse(f(fine), ref) (models/sinnerf.py:332-338) with both features from one batched
        pass (and one batched backward).  ref (384,) is a target (get_vit_feature of the real patch under no_grad)."""
        what = "semantic_loss"
        _check_image(coarse, "coarse", what)
        _check_image(fine, "fine", what)
        if not isinstance(ref, torch.Tensor) or ref.shape != (DIM,):
            raise ValueError(f"{what}: ref must be a ({DIM},) tensor (got {getattr(ref, 'shape', type(ref))})")
        f = self._features([coarse, fine], precision)
        return F.mse_loss(f[0], ref) + F.mse_loss(f[1], ref)


def default_weights_path() -> str:
    return os.path.join(torch.hub.get_dir(), "checkpoints", DINO_FILE)


def _normalise(sd):
    """-> {DINO key: tensor} from DINO's released file, a VitExtractor.model (or DinoViTS16.model) state dict, a
    DinoViTS16 / VitExtractor state dict ('model.' prefix) or a Lightning checkpoint ('state_dict' with 'ext.model.')."""
    if isinstance(sd, dict) and "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    if not isinstance(sd, dict):
        raise TypeError(f"load_dino_weights: expected a path or a state dict (got {type(sd)})")
    for prefix in ("ext.model.", "model."):
        if any(k.startswith(prefix) for k in sd):
            return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    return dict(sd)


def load_dino_weights(src=None) -> DinoViTS16:
    """A DinoViTS16 (on the CPU) holding the weights of `src`: a path to, or the state dict of, DINO's released
    dino_deitsmall16_pretrain.pth; the state_dict() of a VitExtractor.model; or a Lightning checkpoint of SinNeRF
    (entries under 'ext.model.').  With no argument it reads the file torch.hub caches at
    torch.hub.get_dir()/checkpoints/dino_deitsmall16_pretrain.pth, and raises FileNotFoundError naming that path if it
    is not there: nothing is downloaded.  Missing keys (KeyError), extra keys other than head.* (KeyError) and shape
    mismatches (ValueError) raise with the key's name."""
    if src is None:
        src = default_weights_path()
        if not os.path.isfile(src):
            raise FileNotFoundError(f"load_dino_weights: no DINO ViT-S/16 weights at {src} (this library never "
                                    "downloads; put dino_deitsmall16_pretrain.pth there or pass a path / state dict)")
    if isinstance(src, (str, os.PathLike)):
        src = torch.load(src, map_location="cpu", weights_only=True)
    sd = _normalise(src)
    ext = DinoViTS16()
    want = ext.model.state_dict()
    missing = [k for k in want if k not in sd]
    if missing:
        raise KeyError(f"load_dino_weights: missing key {missing[0]!r} ({len(missing)} missing)")
    extra = [k for k in sd if k not in want and not k.startswith("head.")]
    if extra:
        raise KeyError(f"load_dino_weights: unexpected key {extra[0]!r} ({len(extra)} unexpected)")
    for k, v in want.items():
        if tuple(sd[k].shape) != tuple(v.shape):
            raise ValueError(f"load_dino_weights: {k!r} has shape {tuple(sd[k].shape)}, expected {tuple(v.shape)}")
    ext.model.load_state_dict({k: sd[k].detach().to(torch.float32) for k in want}, strict=True)
    return ext
