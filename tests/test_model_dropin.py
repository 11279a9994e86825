"""CPU: the drop-in modules keep the reference's parameter names, seeded initialisation, checkpoint keys and
rollout-time behaviour (select_action / get_log_prob_entropy / value on the CPU path)."""
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL
from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
from fixtures_io import expand_states
from harness import Agent, Cfg, rel, tensorfy


def build(n, e, seed=111):
    torch.manual_seed(seed)
    p, v = create_sgnn_model(Cfg(n, e), Agent())
    return p, v, ActorCritic(p, v)


@pytest.mark.parametrize("name", ["tiny_mixed", "small_mixed"])
def test_seeded_init_and_keys_match_reference(name, golden_dir):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    p, v, ac = build(int(z["n_cap"]), int(z["e_cap"]))
    sd = ac.state_dict()
    want = [k for s in PL.SLOTS.values() for k in PL.state_dict_keys(s)]
    assert sorted(sd.keys()) == sorted(want) and len(sd) == 52
    # same layers, same order, same seed as create_sgnn_model of the reference -> bit-identical weights
    assert np.array_equal(ac.flat_parameters(), z["params"])
    assert sum(q.numel() for q in ac.parameters()) == PL.NUM_PARAMS


@pytest.mark.parametrize("name", ["tiny_mixed", "small_mixed"])
def test_cpu_rollout_path_matches_reference(name, golden_dir):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    states = expand_states(z)
    p, v, ac = build(int(z["n_cap"]), int(z["e_cap"]))
    ts = tensorfy(states)
    with torch.no_grad():
        val = v(ts)
        lp, ent = p.get_log_prob_entropy(ts, torch.tensor(z["actions"]))
        greedy = p.select_action(ts, mean_action=True)
        one = p.select_action([ts[0]], mean_action=True)          # the B=1 call of sample_worker / eval_agent
        sampled = p.select_action(ts, mean_action=False)
    assert val.shape == (len(states), 1) and rel(val.numpy(), z["values"]) < 1e-5
    assert rel(lp.numpy(), z["log_probs"]) < 1e-5 and rel(ent.numpy(), z["entropies"]) < 1e-5
    assert np.array_equal(greedy.numpy(), z["greedy"])            # integer actions: bit-exact
    assert one.shape == (1, 2) and np.array_equal(one.numpy()[0], z["greedy"][0])
    # sampled actions are feasible (inside the mask of the active stage)
    for i, st in enumerate(states):
        sid = int(st[8][:2].argmax())
        assert (st[6] if sid == 0 else st[7])[int(sampled[i, sid])]


def test_checkpoint_roundtrip_and_flat_io(golden_dir):
    z = np.load(os.path.join(golden_dir, "tiny_mixed.npz"))
    p, v, ac = build(int(z["n_cap"]), int(z["e_cap"]), seed=5)
    ac.load_flat_parameters(z["params"])
    assert np.array_equal(ac.flat_parameters(), z["params"])
    p2, v2, ac2 = build(int(z["n_cap"]), int(z["e_cap"]), seed=6)
    ac2.load_state_dict(ac.state_dict())                           # reference-style checkpoint exchange
    assert np.array_equal(ac2.flat_parameters(), z["params"])
    # the encoder is shared: both views of a key are the same storage
    sd = ac.state_dict()
    k = "shared_net.node_encoder.weight"
    assert sd["actor_net." + k].data_ptr() == sd["value_net." + k].data_ptr()


def test_unsupported_shapes_are_rejected():
    cfg = Cfg(10, 10)
    cfg.state_encoder_specs["gcn_node_dim"] = 32
    with pytest.raises(NotImplementedError):
        create_sgnn_model(cfg, Agent())
