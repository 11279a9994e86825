"""CPU: UrbanPlanningPolicy.forward (policy.py:45-65) of both drop-in models against the distributions the unmodified
reference recorded (tests/golden/make_golden_logits.py): the `logits` and `probs` of both Categoricals and `stage`.

Masked entries are compared bit for bit: a row with a candidate normalises the fill value -2^32+1 back to itself
(the log-sum-exp is far below its ulp of 512) with probability 0, and a row without one (edge_empty) is 0 everywhere
with probability 1 / width.  Candidate entries meet the suite's per-tensor bar of 1e-4 (max|delta| / max|reference|)."""
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.model import MASK_FILL, ActorCritic
from fixtures_io import expand_states

TOL = 1e-4
# fixture -> rl-mlp
FIXTURES = {"small_mixed": False, "hlg": False, "concept": False, "edge_empty": False, "extreme_heads": False,
            "mlp_small": True, "mlp_extreme_heads": True}


class Cfg:
    def __init__(self, n, e):
        self.state_encoder_specs = dict(state_encoder_hidden_size=[64, 16], gcn_node_dim=16, num_gcn_layers=2,
                                        num_edge_fc_layers=1, max_num_nodes=n, max_num_edges=e, num_attention_heads=1)
        self.policy_specs = dict(policy_land_use_head_hidden_size=[32, 1], policy_road_head_hidden_size=[32, 1])
        self.value_specs = dict(value_head_hidden_size=[32, 32, 1])


class Agent:
    node_dim, numerical_feature_size, dtype = 23, 52, torch.float32


def load(name, golden_dir):
    """(fixture, recorded logits, the fixture's states, policy_net holding the fixture's parameters on the CPU)."""
    from drl_urban_planning_b200.mlp import create_mlp_model
    from drl_urban_planning_b200.model import create_sgnn_model
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    ref = np.load(os.path.join(golden_dir, name + "_logits.npz"))
    mlp = FIXTURES[name]
    policy_net, value_net = (create_mlp_model if mlp else create_sgnn_model)(Cfg(int(z["n_cap"]), int(z["e_cap"])),
                                                                          Agent())
    sd = (PL.MLP if mlp else PL.SGNN).to_state_dict(np.asarray(z["params"], np.float32))
    ActorCritic(policy_net, value_net).load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return z, ref, expand_states(z), policy_net


def tensorfy(states):
    return [[torch.tensor(x) for x in s] for s in states]


def check_distribution(tag, d, ref):
    """d: a Categorical (or None) against the recorded `<tag>_logits` / `<tag>_probs` (absent when the reference's was
    None): shape, masked entries bit for bit, candidates at the per-tensor bar."""
    if f"{tag}_logits" not in ref:
        assert d is None, tag
        return
    want_z, want_p = ref[f"{tag}_logits"], ref[f"{tag}_probs"]
    z, p = d.logits.detach().cpu().numpy(), d.probs.detach().cpu().numpy()
    assert z.shape == want_z.shape and p.shape == want_p.shape, (tag, z.shape, want_z.shape)
    masked = (want_z == np.float32(MASK_FILL)) | np.all(want_z == 0.0, axis=1, keepdims=True)
    assert np.array_equal(z[masked], want_z[masked]) and np.array_equal(p[masked], want_p[masked]), tag
    cand = ~masked
    if cand.any():
        dz = np.abs(z[cand].astype(np.float64) - want_z[cand]).max() / np.abs(want_z[cand]).max()
        assert dz < TOL, (tag, "logits", dz)
    dp = np.abs(p.astype(np.float64) - want_p).max() / np.abs(want_p).max()
    assert dp < TOL, (tag, "probs", dp)


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
    z, ref, states, policy_net = load(name, golden_dir)
    with torch.no_grad():
        d0, d1, stage = policy_net(tensorfy(states))
    assert np.array_equal(stage.numpy(), ref["stage"])
    check_distribution("lu", d0, ref)
    check_distribution("rd", d1, ref)
