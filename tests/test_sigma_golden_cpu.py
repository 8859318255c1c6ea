"""The oracle's sigma-only passes under autograd against the reference's own gradients (tests/golden/sigma_train.npz,
made by tests/golden/make_sigma_golden.py): render_rays(test_time=True) with and without the random draws, and
eval_points (reference models/rendering.py:64-123 = the fine model's sigma of the embedded points)."""
import numpy as np
import pytest
import torch

from oracle import render_oracle as orc
from tests._common import load_npz, rel_l2, room_params

TT_KEYS = ("opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")
GRAD_BAR = 2e-4


@pytest.fixture(scope="module")
def gold():
    return load_npz("sigma_train.npz")


def check(gold, prefix, params):
    for k, v in params.items():
        key = f"{prefix}_grad_{k}"
        if key + "_norm" not in gold:
            assert v.grad is None, (prefix, k)
            continue
        g = v.grad.flatten()
        idx = torch.from_numpy(gold[key + "_idx"].astype(np.int64))
        norm = float(gold[key + "_norm"])
        assert abs(float(g.double().norm()) - norm) <= GRAD_BAR * norm, (prefix, k)
        assert rel_l2(g[idx], torch.from_numpy(gold[key + "_val"])) <= GRAD_BAR, (prefix, k)


@pytest.mark.parametrize("case,perturb,noise_std", [("det", 0.0, 0.0), ("rand", 1.0, 1.0)])
def test_test_time_render_gradients_equal_reference(gold, case, perturb, noise_std):
    rays = torch.from_numpy(gold[f"{case}_rays"])
    rng = {k[len(case) + 5:]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(f"{case}_rng_")}
    pc = {k: v.clone().requires_grad_(True) for k, v in room_params("coarse").items()}
    pf = {k: v.clone().requires_grad_(True) for k, v in room_params("fine").items()}
    out = orc.render_rays(pc, pf, rays, N_samples=64, N_importance=64, perturb=perturb, noise_std=noise_std, rng=rng,
                          test_time=True)
    assert set(out) == set(TT_KEYS)
    for k in TT_KEYS:
        assert rel_l2(out[k].detach(), torch.from_numpy(gold[f"{case}_out_{k}"])) <= 1e-5, k
    sum((out[k] * torch.from_numpy(gold[f"{case}_proj_{k}"])).sum() for k in TT_KEYS).backward()
    check(gold, f"{case}_coarse", pc)
    check(gold, f"{case}_fine", pf)
    # the sigma-only coarse pass reaches layers 1-8 and the sigma head only
    assert {k for k, v in pc.items() if v.grad is None} == {k for k in pc if k.startswith(("xyz_encoding_final",
                                                                                            "dir_encoding", "rgb"))}


def test_eval_points_gradients_equal_reference(gold):
    pts = torch.from_numpy(gold["pts"])
    pf = {k: v.clone().requires_grad_(True) for k, v in room_params("fine").items()}
    sigma = orc.field_mlp(pf, orc.embed(pts, orc.N_XYZ_FREQS), None, sigma_only=True)
    assert sigma.shape == (pts.shape[0], 1)
    assert rel_l2(sigma.detach(), torch.from_numpy(gold["pts_sigma"])) <= 1e-5
    (sigma * torch.from_numpy(gold["pts_proj"])).sum().backward()
    check(gold, "pts_fine", pf)
