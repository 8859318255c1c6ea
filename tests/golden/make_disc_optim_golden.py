#!/usr/bin/env python
"""Generate tests/golden/disc_optim_steps.npz by running the REFERENCE's get_optimizer on a discriminator.

Needs a checkout of the reference SinNeRF repository at REF (below); the tests only read the .npz it writes:

    python tests/golden/make_disc_optim_golden.py

Calls the reference's own ``get_optimizer(hparams, [D], rate=0.2)`` (``utils/__init__.py:10-31``, unmodified, as
``models/sinnerf.py:208`` calls it for the adversarial loss) for sgd / adam / radam / ranger over the cases of
tests/test_disc_optim_cpu.py -- a Discriminator of imsize 64 and -1 with seeded weights, 14 steps of seeded gradients,
one tensor without a gradient on two steps -- on CPU/fp32, and records sha256 digests of every final parameter and
state tensor plus the per-parameter step counts.  Nothing here is used at run time by the product;
tests/test_disc_optim_cpu.py compares the oracle (oracle/optim_oracle.py, and torch's single-tensor Adam) against this
file bit for bit.
"""
import importlib.util
import os
import sys
import types
import warnings

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.test_disc_optim_cpu import DISC_CASES, case_tag, run_disc_case  # noqa: E402
from tests.test_optim_cpu import optim_digests  # noqa: E402


def reference_get_optimizer():
    """utils/__init__.py as the package `ref_utils`, its optimizers.py and warmup_scheduler.py loaded from the
    reference; visualization.py (plotting dependencies, nothing get_optimizer uses) is left empty."""
    utils_dir = os.path.join(REF, "utils")
    sys.modules["ref_utils.visualization"] = types.ModuleType("ref_utils.visualization")
    spec = importlib.util.spec_from_file_location("ref_utils", os.path.join(utils_dir, "__init__.py"),
                                                  submodule_search_locations=[utils_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_utils"] = mod
    spec.loader.exec_module(mod)
    return mod.get_optimizer


def main():
    get_optimizer = reference_get_optimizer()
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)       # the reference's deprecated addcmul_ / add_ overloads
        for rule, imsize, wd in DISC_CASES:
            out.update(optim_digests(case_tag(rule, imsize, wd), *run_disc_case(get_optimizer, rule, imsize, wd)))
    path = os.path.join(HERE, "disc_optim_steps.npz")
    np.savez_compressed(path, **{k: np.int64(v) if k.endswith("/step") else np.frombuffer(bytes.fromhex(v), np.uint8)
                                 for k, v in out.items()})
    print("wrote", path, len(out), "digests")


if __name__ == "__main__":
    main()
