"""CPU: UrbanPlanningPolicy.forward (policy.py:45-65) of both drop-in models against the distributions the unmodified
reference recorded (tests/golden/make_golden_logits.py): the `logits` and `probs` of both Categoricals and `stage`.

Masked entries are compared bit for bit: a row with a candidate normalises the fill value -2^32+1 back to itself
(the log-sum-exp is far below its ulp of 512) with probability 0, and a row without one (edge_empty) is 0 everywhere
with probability 1 / width.  Candidate entries meet the suite's per-tensor bar of 1e-4 (max|delta| / max|reference|)."""
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200.model import MASK_FILL
from harness import tensorfy
from policy_cases import LOGIT_FIXTURES as FIXTURES, check_distribution, load_policy


def test_fixtures_cover_both_stages_empty_masks_and_zero_probabilities(golden_dir):
    """The recorded set holds what the GPU tests rely on: both stages, all-masked rows, zero-probability candidates."""
    ref = {name: np.load(os.path.join(golden_dir, name + "_logits.npz")) for name in FIXTURES}
    assert all(k in ref["small_mixed"] for k in ("lu_logits", "rd_logits"))
    assert "rd_logits" not in ref["hlg"] and ref["concept"]["lu_logits"].shape[1] == 4000
    empty = ref["edge_empty"]
    assert (empty["lu_logits"] == 0).all(axis=1).any() and (empty["rd_logits"] == 0).all(axis=1).any()
    for name in ("extreme_heads", "mlp_extreme_heads"):
        z = ref[name]["lu_logits"]
        assert ((ref[name]["lu_probs"] == 0) & (z != np.float32(MASK_FILL))).any(), name


@pytest.mark.parametrize("name", list(FIXTURES))
def test_cpu_forward_matches_reference_distributions(name, golden_dir):
    z, ref, states, policy_net = load_policy(name, golden_dir)
    with torch.no_grad():
        d0, d1, stage = policy_net(tensorfy(states))
    assert np.array_equal(stage.numpy(), ref["stage"])
    check_distribution("lu", d0, ref)
    check_distribution("rd", d1, ref)
