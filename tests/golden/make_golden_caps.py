"""Generate the concept-cap golden vectors in this directory by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_caps.py

The recipe is make_golden.py's run_fixture on the shipped hlg_concept caps (1500 nodes, 4000 edges), with its `case`
hook swapping in the concept-cap graphs of tests/cap_cases.py (every edge a candidate at e = 4000, every node a road
candidate at n = 1500, one past each hlg cap at 1001 / 3001 / 3001, a hub row of degree 1499), each followed by an
ordinary concept graph.  The states are stored in the fixture.

  * caps_concept       the rl-sgnn model;
  * mlp_caps_concept   the rl-mlp model.

The graphs at the blob format's 65535 / 32767 limits are not recorded: the padded reference would hold 65535-wide
tensors per state, and those cases rest on the float64 oracles (tests/test_gpu_caps.py).
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (installs the reference shim, sets up the paths)

import cap_cases as CC  # noqa: E402

COUNT = 2 * len(CC.CONCEPT_CASES)


def concept_caps(flat, states, actions, adv, ret, exps):
    st, act, _ = CC.concept_batch()
    assert len(st) == len(states) == COUNT
    return dict(states=st, actions=act)


if __name__ == "__main__":
    MG.run_fixture("caps_concept", "hlg_concept", 23, COUNT, case=concept_caps)
    MG.run_fixture("mlp_caps_concept", "hlg_concept", 23, COUNT, mlp=True, case=concept_caps)
