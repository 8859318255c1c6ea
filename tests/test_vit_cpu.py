"""CPU tests of the semantic-loss path: the float64 oracle (tests/vit_oracle.py) against torchvision's independent
VisionTransformer, the nearest map and its inverse against F.interpolate, weight loading from every accepted source and
its errors, the synthetic weights' logit spread, and C-ABI argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sinnerf_b200 import _lib, build, synthetic
from sinnerf_b200.vit import DinoViTS16, load_dino_weights
from tests import vit_oracle as vo

SHAPES = [(64, 64), (63, 84), (56, 70)]
D = torch.float64


def patch(h, w, seed):
    return torch.rand(2, 3, h, w, generator=torch.Generator().manual_seed(seed), dtype=D)


@pytest.mark.parametrize("hw", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_oracle_matches_torchvision(hw):
    tv = pytest.importorskip("torchvision")
    from torchvision.models.vision_transformer import VisionTransformer
    sd = synthetic.dino_vits16_state_dict(0)
    m = VisionTransformer(224, 16, 12, 6, 384, 1536).double().eval()
    msd = {"class_token": sd["cls_token"], "encoder.pos_embedding": sd["pos_embed"],
           "conv_proj.weight": sd["patch_embed.proj.weight"], "conv_proj.bias": sd["patch_embed.proj.bias"],
           "encoder.ln.weight": sd["norm.weight"], "encoder.ln.bias": sd["norm.bias"]}
    names = {"norm1": "ln_1", "norm2": "ln_2", "attn.qkv": "self_attention.in_proj", "attn.proj": "self_attention.out_proj",
             "mlp.fc1": "mlp.0", "mlp.fc2": "mlp.3"}
    for b in range(12):
        for src, dst in names.items():
            for wb in ("weight", "bias"):
                key = f"encoder.layers.encoder_layer_{b}.{dst}" + ("_" if dst.endswith("in_proj") else ".") + wb
                msd[key] = sd[f"blocks.{b}.{src}.{wb}"]
    msd["heads.head.weight"] = m.heads.head.weight.detach()
    msd["heads.head.bias"] = m.heads.head.bias.detach()
    m.load_state_dict({k: v.double() for k, v in msd.items()}, strict=True)
    got = {}
    m.encoder.layers.encoder_layer_11.register_forward_hook(lambda mod, i, o: got.setdefault("x", o))
    x = patch(*hw, seed=hw[0])
    with torch.no_grad():
        m(vo.preprocess(x))
        want = vo.cls_feature(sd, x)
    tv_feat = got["x"][0, 0]
    assert float((tv_feat - want).norm() / want.norm()) <= 1e-10
    del tv


@pytest.mark.parametrize("size", [64, 63, 84, 56, 70, 1, 5, 111, 112, 224, 225, 300, 513])
def test_nearest_map_and_inverse(size):
    idx = vo.nearest_index(size)
    src = torch.arange(size, dtype=torch.float32).view(1, 1, 1, size)
    want = F.interpolate(src, size=(1, 224)).view(-1).long().numpy()
    assert np.array_equal(idx, want)
    first, last = vo.inverse_ranges(size)
    for s in range(size):
        assert np.array_equal(np.arange(first[s], last[s]), np.nonzero(idx == s)[0])


def test_synthetic_logit_spread():
    sd = {k: v.double() for k, v in synthetic.dino_vits16_state_dict(0).items()}
    x = patch(64, 64, 1)
    t = vo.tokens(sd, vo.preprocess(x))
    for b in range(12):
        L = vo.attention_logits(sd, t, b)
        std = float(L.std(-1).mean())
        assert 1.5 <= std <= 5.0, (b, std)
        t = vo.block(t, sd, f"blocks.{b}.")
    for k in ("norm1.weight", "norm1.bias", "attn.qkv.bias", "mlp.fc2.bias"):
        v = sd["blocks.3." + k]
        assert float((v - v.mean()).abs().max()) > 0.05 and float(v.abs().min()) >= 0.0


def test_synthetic_seeded_and_leaves_rng():
    state = torch.random.get_rng_state()
    a, b = synthetic.dino_vits16_state_dict(3), synthetic.dino_vits16_state_dict(3)
    assert torch.equal(torch.random.get_rng_state(), state)
    assert all(torch.equal(a[k], b[k]) for k in a)


def test_state_dict_names_match_vit_extractor():
    ext = DinoViTS16()
    sd = synthetic.dino_vits16_state_dict(0)
    assert list(ext.state_dict()) == ["model." + k for k in sd]
    assert not any(p.requires_grad for p in ext.parameters())
    ext.load_state_dict({"model." + k: v for k, v in sd.items()}, strict=True)


def _equal(ext, sd):
    return all(torch.equal(ext.model.state_dict()[k], v) for k, v in sd.items())


def test_load_dino_weights_sources(tmp_path):
    sd = synthetic.dino_vits16_state_dict(1)
    path = tmp_path / "dino.pth"
    torch.save(sd, path)
    assert _equal(load_dino_weights(str(path)), sd)                         # DINO's released file
    assert _equal(load_dino_weights(dict(sd, **{"head.weight": torch.zeros(1)})), sd)   # head.* ignored
    assert _equal(load_dino_weights(load_dino_weights(sd).model.state_dict()), sd)      # VitExtractor.model
    ckpt = {"epoch": 3, "state_dict": {**{"ext.model." + k: v for k, v in sd.items()},
                                       "nerf_coarse.xyz_encoding_1.0.weight": torch.zeros(2)}}
    assert _equal(load_dino_weights(ckpt), sd)                             # Lightning checkpoint


def test_load_dino_weights_errors(tmp_path, monkeypatch):
    sd = synthetic.dino_vits16_state_dict(1)
    bad = dict(sd)
    del bad["blocks.4.mlp.fc1.bias"]
    with pytest.raises(KeyError, match="blocks.4.mlp.fc1.bias"):
        load_dino_weights(bad)
    with pytest.raises(KeyError, match="extra_thing"):
        load_dino_weights(dict(sd, extra_thing=torch.zeros(1)))
    bad = dict(sd, **{"blocks.2.attn.qkv.weight": torch.zeros(1152, 383)})
    with pytest.raises(ValueError, match="blocks.2.attn.qkv.weight"):
        load_dino_weights(bad)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    with pytest.raises(FileNotFoundError, match=str(tmp_path / "hub" / "checkpoints" / "dino_deitsmall16_pretrain.pth")):
        load_dino_weights()
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    torch.save(sd, tmp_path / "hub" / "checkpoints" / "dino_deitsmall16_pretrain.pth")
    assert _equal(load_dino_weights(), sd)


def test_cpu_tensors_raise():
    ext = load_dino_weights(synthetic.dino_vits16_state_dict(0))
    with pytest.raises(RuntimeError, match="CUDA"):
        ext.cls_feature(torch.rand(1, 3, 64, 64))
    with pytest.raises(ValueError, match="Bx3xHxW"):
        ext.cls_feature(torch.rand(3, 64, 64))
    with pytest.raises(ValueError, match="Bx3xHxW"):
        ext.semantic_loss(torch.zeros(384), torch.rand(1, 4, 8, 8), torch.rand(1, 3, 8, 8))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_cabi_argument_checks(lib):
    assert lib.snb_vit_pack_bytes(99) == 0
    split, half = lib.snb_vit_pack_bytes(1), lib.snb_vit_pack_bytes(4)
    assert split == lib.snb_vit_pack_bytes(0) == lib.snb_vit_pack_bytes(2) and half == lib.snb_vit_pack_bytes(3)
    n_mat = 384 * 768 + 12 * (1152 * 384 + 384 * 384 + 1536 * 384 + 384 * 1536)
    assert 2 * n_mat * 2 <= split < 2 * n_mat * 2 + (1 << 20) and n_mat * 2 <= half < n_mat * 2 + (1 << 20)
    assert lib.snb_vit_workspace_bytes(0, 0) == 0 and lib.snb_vit_workspace_bytes(_lib.VIT_MAX_IMAGES + 1, 0) == 0
    assert lib.snb_vit_workspace_bytes(2, 1) > lib.snb_vit_workspace_bytes(2, 0) > lib.snb_vit_workspace_bytes(1, 0)
    assert lib.snb_vit_pack(None, 99, None, None) == -3
    assert lib.snb_vit_pack(None, 1, None, None) == -1
    ptrs = (C.c_void_p * 1)(None)
    st = (C.c_int64 * 3)(1, 1, 1)
    sz = (C.c_int * 2)(64, 64)
    assert lib.snb_vit_forward(None, 1, ptrs, st, sz, 1, 0, None, None, None) == -1
    assert b"null image pointer" in lib.snb_last_error()
    assert lib.snb_vit_forward(None, 1, ptrs, st, sz, 0, 0, None, None, None) == -1
    assert b"n_images" in lib.snb_last_error()
    sz0 = (C.c_int * 2)(0, 64)
    ptrs1 = (C.c_void_p * 1)(16)
    assert lib.snb_vit_forward(None, 1, ptrs1, st, sz0, 1, 0, None, None, None) == -1
    assert b"size" in lib.snb_last_error()
    assert lib.snb_vit_backward(None, 7, sz, 1, None, ptrs1, st, None, None) == -3
