"""CPU: pin both oracles (padded fp32 torch port, unpadded f64 numpy restatement) to the golden vectors that
`tests/golden/make_golden.py` produced by running the unmodified reference."""
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL
from fixtures_io import expand_states
from harness import per_tensor_rel, rel
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP

FIXTURES = ["tiny_mixed", "small_mixed", "hlg", "concept", "caps_concept"]


@pytest.fixture(scope="module", params=FIXTURES)
def fx(request, golden_dir):
    z = np.load(os.path.join(golden_dir, request.param + ".npz"))
    return request.param, z, expand_states(z)


def test_torch_port_forward_matches_reference(fx):
    name, z, states = fx
    P = TP.params_from_flat(torch.tensor(z["params"]))
    b = TP.stack_states(states)
    with torch.no_grad():
        v = TP.value(P, b)
        lp, ent = TP.log_prob_entropy(P, b, torch.tensor(z["actions"]))
        greedy = TP.greedy_action(P, b)
    assert rel(v.numpy(), z["values"]) < 2e-6
    assert rel(lp.numpy(), z["log_probs"]) < 2e-6
    assert rel(ent.numpy(), z["entropies"]) < 2e-6
    assert np.array_equal(greedy.numpy(), z["greedy"])          # integer action indices: bit-exact


def test_torch_port_steps_match_reference(fx):
    name, z, states = fx
    agent = TP.PortAgent(z["params"])
    b = TP.stack_states(states)
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    args = (b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
            torch.tensor(z["fixed_log_probs"]), ind)
    for k in range(3):
        losses = agent.backward(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert per_tensor_rel(agent.flat_grad(), z["grads"][k])[0] < 5e-5
        agent.clip()
        agent.opt.step()
        agent.steps_done += 1
        assert rel(agent.flat(), z["params_after"][k]) < 5e-6


def test_numpy_oracle_matches_reference(fx):
    name, z, states = fx
    r = ON.ppo_minibatch(z["params"], states, z["actions"], z["advantages"], z["returns"],
                         z["fixed_log_probs"], z["exps"])
    assert rel(r["value"], z["values"].reshape(-1)) < 2e-5
    assert rel(r["log_prob"], z["log_probs"].reshape(-1)) < 2e-5
    assert rel(r["entropy"], z["entropies"].reshape(-1)) < 2e-5
    got = [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]]
    assert np.allclose(got, z["losses"][0], rtol=2e-5, atol=2e-6)
    assert per_tensor_rel(r["grad"], z["grads"][0])[0] < 1e-4
    # greedy actions, bit-exact
    P = ON._p64(z["params"])
    for i, st in enumerate(states):
        g = ON.unpad(st)
        fw = ON.forward(P, g)
        sid = fw["stage_id"]
        assert fw["greedy"] == int(z["greedy"][i, sid])


def test_numpy_oracle_first_step_clip_and_adam(fx):
    """First optimiser step of the agent's life: clip policy group then value group, then Adam."""
    name, z, states = fx
    r = ON.ppo_minibatch(z["params"], states, z["actions"], z["advantages"], z["returns"],
                         z["fixed_log_probs"], z["exps"])
    g = ON.clip_groups(r["grad"])
    live = ON.live_mask(states)
    zero = np.zeros(PL.NUM_PARAMS)
    flat, m, v, t = ON.adam_step(z["params"], zero, zero, zero, g, live)
    assert rel(flat, z["params_after"][0]) < 5e-6
    # entries of an unused head must not move at all
    assert np.array_equal(flat[~live].astype(np.float32), z["params"][~live])


def test_gae_matches_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "gae.npz"))
    for tag, (gamma, tau) in {"g1t0": (1.0, 0.0), "g99t95": (0.99, 0.95)}.items():
        a, r = ON.estimate_advantages(z["rewards"], z["masks"], z["values"], gamma, tau)
        assert np.array_equal(a, z[f"adv_{tag}"]), tag      # same fp32 operation order -> bit-exact
        assert np.array_equal(r, z[f"ret_{tag}"]), tag
        a2, r2 = TP.estimate_advantages(torch.tensor(z["rewards"]), torch.tensor(z["masks"]),
                                        torch.tensor(z["values"]), gamma, tau)
        assert np.array_equal(a2.numpy(), z[f"adv_{tag}"])
        assert np.array_equal(r2.numpy(), z[f"ret_{tag}"])


def test_gae_known_answer():
    """gamma=1, tau=0 (every shipped cfg): A_t = r_t + V_{t+1} m_t - V_t, R_t = r_t + V_{t+1} m_t."""
    r = np.array([1.0, 2.0, 3.0, 4.0], np.float32)
    m = np.array([1.0, 0.0, 1.0, 0.0], np.float32)
    v = np.array([0.5, 0.25, -1.0, 2.0], np.float32)
    a, R = ON.estimate_advantages(r, m, v, 1.0, 0.0)
    assert np.allclose(a.ravel(), [1 + 0.25 - 0.5, 2 - 0.25, 3 + 2 + 1, 4 - 2])
    assert np.allclose(R.ravel(), [1.25, 2.0, 5.0, 4.0])


@pytest.mark.parametrize("name", ["hlg256", "dhm256", "grid64"])
def test_numpy_oracle_matches_reference_at_baseline_sizes(name, golden_dir):
    """BASELINE.json sizes: the f64 oracle against the reference-generated vectors of a 256-graph HLG / DHM minibatch
    and the two-stage grid community (states regenerated from the seed; the digest guards the generator)."""
    from drl_urban_planning_b200 import synth
    from fixtures_io import states_digest
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    states, actions = synth.make_states(int(z["seed"]), str(z["community"]), int(z["count"]))
    assert states_digest(states) == str(z["digest"])
    r = ON.ppo_minibatch(z["params"], states, z["actions"], z["advantages"], z["returns"],
                         z["fixed_log_probs"], z["exps"])
    assert rel(r["value"], z["values"].reshape(-1)) < 2e-5
    assert rel(r["log_prob"], z["log_probs"].reshape(-1)) < 2e-5
    assert rel(r["entropy"], z["entropies"].reshape(-1)) < 2e-5
    got = [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]]
    assert np.allclose(got, z["losses"][0], rtol=2e-5, atol=2e-6)
    assert per_tensor_rel(r["grad"], z["grads"][0])[0] < 1e-4


def test_torch_port_update_policy_matches_reference(golden_dir):
    """The multi-epoch trajectory of the unmodified reference's update_params / update_policy (composed epoch
    permutations, urban_planning_agent.py:306-312) reproduced by the oracle port driven the same way."""
    import math
    z = np.load(os.path.join(golden_dir, "update_small.npz"))
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    states = expand_states(z)
    agent = TP.PortAgent(z["params"])
    b_all = TP.stack_states(states)
    act = torch.tensor(z["actions"])
    with torch.no_grad():
        values = TP.value(agent.params(), b_all)
    adv, ret = TP.estimate_advantages(torch.tensor(z["rewards"]), torch.tensor(z["masks"]), values,
                                      float(z["gamma_tau"][0]), float(z["gamma_tau"][1]))
    with torch.no_grad():
        fixed, _ = TP.log_prob_entropy(agent.params(), b_all, act)
    exps_t = torch.tensor(z["exps"])
    np.random.seed(np_seed)
    order, losses = np.arange(T), []
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(int(math.floor(T / B))):
            idx = order[i * B:(i + 1) * B]
            b = TP.stack_states([states[j] for j in idx])
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(agent.step(b, act[idx], adv[idx], ret[idx], fixed[idx], ind))
    assert np.allclose(np.array(losses), z["losses"], rtol=2e-5, atol=2e-6)
    assert rel(agent.flat(), z["params_after"]) < 5e-6


def test_empty_action_masks_match_reference(golden_dir):
    """All logits equal to the fill value: the reference's fp32 log-softmax yields log_prob = 0 and entropy = 0 (not the
    -log(width) / log(width) of exact arithmetic), arg-max = first index."""
    z = np.load(os.path.join(golden_dir, "edge_empty.npz"))
    states = expand_states(z)
    assert z["log_probs"].ravel()[1] == 0.0 and z["log_probs"].ravel()[2] == 0.0
    assert abs(z["entropies"].ravel()[1]) == 0.0 and abs(z["entropies"].ravel()[2]) == 0.0
    r = ON.ppo_minibatch(z["params"], states, z["actions"], np.zeros((3, 1), np.float32), np.zeros((3, 1), np.float32),
                         np.zeros((3, 1), np.float32), np.ones(3, np.float32), want_grad=False)
    assert np.allclose(r["log_prob"], z["log_probs"].ravel(), rtol=2e-5, atol=1e-7)
    assert np.allclose(r["entropy"], z["entropies"].ravel(), rtol=2e-5, atol=1e-7)
    b = TP.stack_states(states)
    with torch.no_grad():
        lp, ent = TP.log_prob_entropy(TP.params_from_flat(torch.tensor(z["params"])), b, torch.tensor(z["actions"]))
    assert np.allclose(lp.numpy(), z["log_probs"], rtol=2e-6, atol=1e-7) and np.allclose(ent.numpy(), z["entropies"], atol=1e-6)
