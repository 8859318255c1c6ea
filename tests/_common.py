"""Shared helpers for the test-suite: golden loading and tolerance checks."""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

RENDER_CASES = ["c1_seed0_64p0", "c1_full_seed0_64p0", "lego_seed0_64p64_wb", "llff_room_64p64", "llff_room_64p64_train",
                "dtu_seed0_64p64_disp", "lego_room_testtime", "lego_seed0_32p16_odd"]


def load_npz(name):
    with np.load(os.path.join(GOLDEN, name), allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


_room = None


def room_params(which):
    """'coarse' | 'fine' -> {state-dict key: fp32 tensor} of the reference's trained checkpoint."""
    global _room
    if _room is None:
        # stored in parts of < 1 MB each: room_weights_0.npz, room_weights_1.npz, ...
        _room = {}
        i = 0
        while os.path.exists(os.path.join(GOLDEN, f"room_weights_{i}.npz")):
            _room.update(load_npz(f"room_weights_{i}.npz"))
            i += 1
        assert _room, "tests/golden/room_weights_*.npz missing"
    pre = which + "/"
    return {k[len(pre):]: torch.from_numpy(v.copy()) for k, v in _room.items() if k.startswith(pre)}


def case_params(case):
    """(coarse, fine) parameter dicts a render golden was generated with."""
    from oracle.render_oracle import default_init_params
    tag = str(case["weights_tag"])
    if tag == "room":
        return room_params("coarse"), room_params("fine")
    assert tag == "seed0"
    return default_init_params(0), default_init_params(1)


def case_cfg(case):
    c = case["cfg"]
    return dict(N_samples=int(c[0]), N_importance=int(c[1]), use_disp=bool(c[2]), perturb=float(c[3]),
                noise_std=float(c[4]), white_back=bool(c[5]), test_time=bool(c[6]))


def case_rng(case):
    return {k[4:]: torch.from_numpy(v.copy()) for k, v in case.items() if k.startswith("rng_")}


def rel_l2(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).flatten()
    b = torch.as_tensor(b, dtype=torch.float64).flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def max_rel(a, b):
    """max |a-b| / max |b|  (the 'max-abs <= tol * max|ref|' form of SURVEY.md 8c)."""
    a = torch.as_tensor(a, dtype=torch.float64).flatten()
    b = torch.as_tensor(b, dtype=torch.float64).flatten()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def assert_close(a, b, tol, what=""):
    r, m = rel_l2(a, b), max_rel(a, b)
    assert r <= tol and m <= tol, f"{what}: rel_l2={r:.3e} max_rel={m:.3e} > tol={tol:.1e}"
