"""Generate the weight-decay golden vectors in this directory by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_wd.py

The recipes are those of make_golden.py, on the same seeds and states as the undecayed fixture of the same name without
"_wd", with one difference: the optimiser is `torch.optim.Adam(lr=4e-4, eps=1e-5, weight_decay=WD)`, as a cfg with
`weightdecay: WD` makes the reference build it (urban_planning_agent.py:145-149).  Each file also stores `weight_decay`.

  * small_mixed_wd   mixed stages, 3 steps, the first one clipped by the reference's own clip_policy_grad;
  * hlg_wd           land-use only: the road head has grad None, so Adam skips it and it must not decay;
  * mlp_small_wd     the rl-mlp model;
  * update_small_wd  the reference's whole update_params iteration.
"""
from __future__ import annotations

import contextlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (installs the reference shim, sets up the paths)
import torch  # noqa: E402

WD = 1e-2
FIXTURES = [
    # name, community, seed, count, rl-mlp
    ("small_mixed_wd", "small", 5, 8, False),
    ("hlg_wd", "hlg", 111, 4, False),
    ("mlp_small_wd", "small", 5, 12, True),
]


@contextlib.contextmanager
def adam_weight_decay(wd):
    """Every torch.optim.Adam built inside the block gets weight_decay=wd (make_golden.py builds it with 0.0)."""
    base = torch.optim.Adam

    class DecayedAdam(base):
        def __init__(self, params, **kw):
            assert kw.get("weight_decay", 0.0) == 0.0, kw
            kw["weight_decay"] = wd
            super().__init__(params, **kw)

    torch.optim.Adam = DecayedAdam
    try:
        yield
    finally:
        torch.optim.Adam = base


def record_weight_decay(name, wd):
    path = os.path.join(HERE, f"{name}.npz")
    z = dict(np.load(path))
    z["weight_decay"] = np.float64(wd)
    np.savez_compressed(path, **z)


if __name__ == "__main__":
    only = set(sys.argv[1:])
    with adam_weight_decay(WD):
        for name, community, seed, count, mlp in FIXTURES:
            if not only or name in only:
                MG.run_fixture(name, community, seed, count, mlp=mlp)
                record_weight_decay(name, WD)
        if not only or "update_small_wd" in only:
            MG.run_update_params(name="update_small_wd")
            record_weight_decay("update_small_wd", WD)
