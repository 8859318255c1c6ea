#!/usr/bin/env python
"""Generate tests/golden/optim_steps.npz by running the REFERENCE's optimisers.

Run in the build container only (needs /root/reference; the GPU box has none):

    python tests/golden/make_optim_golden.py

Steps the reference's own RAdam and Ranger (``utils/optimizers.py``, unmodified,
from /root/reference) and torch.optim.SGD -- the three non-Adam choices of the
reference's ``get_optimizer`` (``utils/__init__.py:10-31``) -- on CPU/fp32 over the
cases of tests/test_optim_cpu.py, and records sha256 digests of every final
parameter and state tensor plus the per-parameter step counts.  Nothing here is
used at run time by the product; tests/test_optim_cpu.py compares the oracle
(oracle/optim_oracle.py) against this file bit for bit.
"""
import importlib.util
import os
import sys
import types
import warnings

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.test_optim_cpu import OPTIM_CASES, optim_digests, run_optim_case  # noqa: E402


def reference_optimizers():
    """utils/optimizers.py loaded on its own (the package's __init__ pulls in plotting dependencies)."""
    spec = importlib.util.spec_from_file_location("ref_optimizers", os.path.join(REF, "utils", "optimizers.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    return types.SimpleNamespace(SGD=torch.optim.SGD, RAdam=ref.RAdam, Ranger=ref.Ranger)


def main():
    mod = reference_optimizers()
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)       # the reference's deprecated addcmul_ / add_ overloads
        for rule, wd in OPTIM_CASES:
            out.update(optim_digests(f"{rule}_wd{wd:g}", *run_optim_case(mod, rule, wd)))
    path = os.path.join(HERE, "optim_steps.npz")
    np.savez_compressed(path, **{k: np.int64(v) if k.endswith("/step") else np.frombuffer(bytes.fromhex(v), np.uint8)
                                 for k, v in out.items()})
    print("wrote", path, len(out), "digests")


if __name__ == "__main__":
    main()
