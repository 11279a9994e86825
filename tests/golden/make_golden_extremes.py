"""Generate the golden vectors of the magnitude regimes in this directory by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_extremes.py [name ...]

make_golden.run_fixture's recipe (states stored), with its `case` hook applying the parameter transform and building
the minibatch of each regime (tests/extreme_cases.py) before the reference model records anything:

  * extreme_clamp      GCN node factors beyond exp2a's clamp, moderate edge pre-activations, large and fast graphs;
  * extreme_attention  attention logits spanning more than 104, two nodes tied at the maximum;
  * extreme_heads      peaked policy heads with arg-max, zero-probability and masked actions, every side of the clip;
  * extreme_tanh       saturated numeric-encoder, value-head and policy-head hidden units;
  * mlp_extreme_heads, mlp_extreme_tanh   the rl-mlp model in the same two regimes.

The float64 oracles agree with these vectors to the reference's own fp32 rounding (tests/test_oracle_extremes.py); the
GPU tests take each tensor's bar from the reference's deviation from float64 where it exceeds the suite's 1e-4.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (installs the reference shim, sets up the paths)
import extreme_cases as EC  # noqa: E402

if __name__ == "__main__":
    only = set(sys.argv[1:])
    for name, community, mlp, case in EC.FIXTURES:
        if not only or name in only:
            MG.run_fixture(name, community, 0, 8, mlp=mlp, case=case)
