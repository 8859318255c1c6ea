"""Randomised differential test: the CPU oracle against what the REFERENCE ITSELF computed on the same inputs.

The reference's outputs were recorded by running it (tests/golden/make_golden.py, `live_golden`) and stored in
tests/golden/reference_live.npz; the inputs are regenerated here from the same seeds.  Seeds, sizes and option
combinations beyond the other goldens: use_disp, white_back, perturb/noise (the reference draws from the global
generator in the order rand, randn, rand, randn -- the oracle must consume it identically), N_importance = 0,
test_time.  Gradients are stored as a seeded sample of each tensor plus the tensor's norm (file size).
"""
import os

import numpy as np
import pytest
import torch

from oracle import render_oracle as orc
from sinnerf_b200 import synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.npz")

CASES = [
    # shape, n, S, Ni, use_disp, perturb, noise_std, white_back, seed
    ("lego", 33, 64, 64, False, 0.0, 0.0, True, 1),
    ("llff", 20, 48, 24, False, 1.0, 1.0, False, 2),
    ("dtu", 17, 32, 16, True, 1.0, 0.0, True, 3),
    ("lego", 9, 64, 0, False, 0.0, 1.0, False, 4),
    ("llff", 5, 16, 40, True, 0.0, 0.0, False, 5),
]


GRAD_SAMPLE = 512


def grad_case_inputs():
    """rays, coarse / fine parameters and the projection seed of the autograd case."""
    return synthetic.random_rays("llff", 14, seed=21), orc.default_init_params(31), orc.default_init_params(32), 5


def grad_sample_index(numel, k):
    """Fixed, seeded sample of flat indices of a tensor (all of them when it is small)."""
    if numel <= k:
        return torch.arange(numel)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(numel))[:k].sort().values


@pytest.fixture(scope="module")
def ref():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def stored(ref, prefix):
    return {k[len(prefix):]: torch.from_numpy(v) for k, v in ref.items() if k.startswith(prefix)}


@pytest.mark.parametrize("shape,n,S,Ni,use_disp,perturb,noise_std,white_back,seed", CASES)
def test_render_rays_oracle_equals_live_reference(ref, shape, n, S, Ni, use_disp, perturb, noise_std, white_back, seed):
    case = CASES.index((shape, n, S, Ni, use_disp, perturb, noise_std, white_back, seed))   # key of the recorded outputs
    rays = synthetic.random_rays(shape, n, seed=seed)
    pc, pf = orc.default_init_params(10 + seed), orc.default_init_params(20 + seed)
    want = stored(ref, f"case{case}/")
    assert want
    with torch.no_grad():
        torch.manual_seed(100 + seed)
        got = orc.render_rays(pc, pf if Ni > 0 else None, rays, N_samples=S, N_importance=Ni, use_disp=use_disp, perturb=perturb,
                              noise_std=noise_std, white_back=white_back)
    for k, v in want.items():
        assert k in got, k
        assert got[k].shape == v.shape, k
        err = float((got[k] - v).abs().max())
        scale = max(float(v.abs().max()), 1e-6)
        assert err <= 2e-5 * scale, (k, err, scale)


def test_test_time_keys_and_values(ref):
    rays = synthetic.random_rays("lego", 12, seed=9)
    pc, pf = orc.default_init_params(1), orc.default_init_params(2)
    want = stored(ref, "testtime/")
    with torch.no_grad():
        got = orc.render_rays(pc, pf, rays, N_samples=64, N_importance=64, noise_std=0.0, white_back=True, test_time=True)
    assert set(k for k in got if not k.startswith("_")) == set(want)
    for k, v in want.items():
        assert float((got[k] - v).abs().max()) <= 2e-5 * max(float(v.abs().max()), 1e-6), k


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_sample_pdf_oracle_equals_live_reference(ref, seed):
    g = torch.Generator().manual_seed(seed)
    n, m, ni = 19, 23 + seed, 31
    bins = torch.sort(torch.rand(n, m + 1, generator=g) * 4 + 2, dim=-1).values
    w = torch.rand(n, m, generator=g) ** 3
    w[0] = 0.0                                    # all-zero weights row (the eps path)
    want = torch.from_numpy(ref[f"pdf{seed}"])
    got = orc.sample_pdf(bins, w, ni, det=True)
    # identical arithmetic; allow the inverse-CDF's knot discontinuity (SURVEY hard part 3) on a few samples
    diff = (got - want).abs()
    assert float(diff.median()) == 0.0
    assert int((diff > 1e-5).sum()) <= 4


def test_autograd_oracle_equals_live_reference(ref):
    """Gradients of a random projection of all outputs w.r.t. all 48 parameter tensors: reference autograd vs
    autograd through the oracle (perturb and noise on: the sample_pdf detach and the RNG order both matter)."""
    rays, pc, pf, _ = grad_case_inputs()
    oc = {k: v.clone().requires_grad_(True) for k, v in pc.items()}
    of = {k: v.clone().requires_grad_(True) for k, v in pf.items()}
    torch.manual_seed(77)
    got = orc.render_rays(oc, of, rays, N_samples=32, N_importance=24, perturb=1.0, noise_std=1.0, white_back=False)
    proj = stored(ref, "proj/")          # the random projection the reference's outputs were reduced with
    assert proj
    sum((got[k] * v).sum() for k, v in proj.items()).backward()
    n_checked = 0
    for tag, params in (("coarse", oc), ("fine", of)):
        for k, v in params.items():
            norm_key, sample_key = f"grad/{tag}/{k}/norm", f"grad/{tag}/{k}/sample"
            if norm_key not in ref:
                assert v.grad is None or float(v.grad.abs().sum()) == 0.0, k
                continue
            b_norm = float(ref[norm_key])
            if v.grad is None:
                assert b_norm == 0.0, k
                continue
            a = v.grad.reshape(-1)[grad_sample_index(v.numel(), GRAD_SAMPLE)]
            b = torch.from_numpy(ref[sample_key])
            assert abs(float(v.grad.double().norm()) - b_norm) <= 2e-4 * max(b_norm, 1e-12), (k, float(v.grad.norm()), b_norm)
            assert float((a - b).norm()) <= 2e-4 * max(float(b.norm()), 1e-12), (k, float((a - b).norm() / b.norm()))
            n_checked += 1
    assert n_checked > 0
