"""float64 restatement of SinNeRF's get_vit_feature (models/sinnerf.py:162-169) with DINO vit_small/16
(facebookresearch/dino vision_transformer.py: pre-norm blocks, LayerNorm eps 1e-6, qkv laid out (3, heads, 64),
exact GELU, no dropout), differentiable in the input through torch autograd.  The test oracle of sinnerf_b200.vit;
tests/test_vit_cpu.py holds it equal to torchvision's VisionTransformer with the DINO weights mapped onto it."""
import numpy as np
import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
RES = 224


def nearest_index(in_size: int, out_size: int = RES) -> np.ndarray:
    """F.interpolate(mode='nearest') source index of each destination index: min(floor(dst * (float)in / out), in - 1)
    with the scale and the product in float32."""
    scale = np.float32(in_size) / np.float32(out_size)
    dst = np.arange(out_size, dtype=np.float32)
    return np.minimum(np.floor(dst * scale).astype(np.int64), in_size - 1)


def inverse_ranges(in_size: int, out_size: int = RES):
    """[first, last) destination range of every source index under the monotone nearest map (empty when unused)."""
    idx = nearest_index(in_size, out_size)
    first = np.searchsorted(idx, np.arange(in_size), side="left")
    last = np.searchsorted(idx, np.arange(in_size), side="right")
    return first, last


def preprocess(x: torch.Tensor) -> torch.Tensor:
    """image 0 of x (B, 3, h, w) -> (1, 3, 224, 224): nearest resize, then (x - mean) / std"""
    h, w = x.shape[-2:]
    iy, ix = (torch.from_numpy(nearest_index(s)).to(x.device) for s in (h, w))
    y = x[0:1][:, :, iy][:, :, :, ix]
    mean = torch.tensor(MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (y - mean) / std


def block(x, sd, p):
    B, N, Cd = x.shape
    h = F.layer_norm(x, (Cd,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
    qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, N, 3, 6, 64).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    attn = ((q @ k.transpose(-2, -1)) * 64 ** -0.5).softmax(dim=-1)
    o = (attn @ v).transpose(1, 2).reshape(B, N, Cd)
    x = x + F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    h = F.layer_norm(x, (Cd,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
    h = F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
    return x + F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])


def tokens(sd, img224):
    x = F.conv2d(img224, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=16)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat([sd["cls_token"].expand(x.shape[0], -1, -1), x], 1)
    return x + sd["pos_embed"]


def attention_logits(sd, x, b):
    """(heads, 197, 197) scaled logits of block b on token rows x (1, 197, 384)"""
    p = f"blocks.{b}."
    h = F.layer_norm(x, (384,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
    qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(1, 197, 3, 6, 64).permute(2, 0, 3, 1, 4)
    return ((qkv[0] @ qkv[1].transpose(-2, -1)) * 64 ** -0.5)[0]


def cls_feature(sd, x: torch.Tensor) -> torch.Tensor:
    """get_vit_feature(x): block 11's output (before the final norm) at token 0 of image 0, (384,).  sd: DINO keys;
    computed in x's dtype (pass float64 for the oracle)."""
    sd = {k: v.to(x.device, x.dtype) for k, v in sd.items()}
    t = tokens(sd, preprocess(x))
    for b in range(12):
        t = block(t, sd, f"blocks.{b}.")
    return t[0, 0]


def semantic_loss(sd, ref, coarse, fine):
    return F.mse_loss(cls_feature(sd, coarse), ref) + F.mse_loss(cls_feature(sd, fine), ref)
