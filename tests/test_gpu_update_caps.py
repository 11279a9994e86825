"""GPU (H100): one whole update_params iteration of PPOUpdater on the shipped concept caps (1500 nodes, 4000 edges), with
the concept-cap graphs of tests/cap_cases.py (every edge or every node a candidate, one past each hlg cap, a hub row)
mixed into ordinary hlg_concept / dhm_concept rollout states, on both models, against the padded eager-PyTorch oracle
ports driven by the same np.random permutations (as tests/test_gpu_update.py does on small caps)."""
import math

import numpy as np
import pytest
import torch

import cap_cases as CC
from drl_urban_planning_b200 import _lib, params as PL, synth
from harness import rel
from oracle import mlp_port as MP
from oracle import torch_port as TP
from test_gpu_update import port_update_params

pytestmark = pytest.mark.gpu

T, B, EPOCHS, SEED = 512, 128, 1, 29


def rollout():
    """T states: the concept-cap batch spread over the rollout, the rest ordinary concept states; rewards, episode
    ends every 50 states, and exps = 0 on a few."""
    caps, caps_actions, _ = CC.concept_batch()
    rest, rest_actions = synth.make_mixed_states(SEED, ["hlg_concept", "dhm_concept"], T - len(caps))
    at = np.linspace(3, T - 5, len(caps)).astype(int)
    states, actions, j = [], np.zeros((T, 2), np.float32), 0
    for i in range(T):
        if i in at:
            k = int(np.flatnonzero(at == i)[0])
            states.append(caps[k]); actions[i] = caps_actions[k]
        else:
            states.append(rest[j]); actions[i] = rest_actions[j]; j += 1
    rng = np.random.default_rng(SEED)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[49::50] = 0.0
    exps = np.ones(T, np.float32); exps[7::97] = 0.0
    return states, actions, rewards, masks, exps, at


def mlp_port_update(flat, states, actions, rewards, masks, exps, seed):
    """The reference's update_params / update_policy control flow on the rl-mlp port (CPU)."""
    agent = MP.MLPPortAgent(flat)
    act = torch.tensor(actions)
    with torch.no_grad():
        values = torch.cat([MP.value(agent.P, MP.stack_states(states[i:i + B])) for i in range(0, T, B)])
        fixed = torch.cat([MP.log_prob_entropy(agent.P, MP.stack_states(states[i:i + B]), act[i:i + B])[0]
                           for i in range(0, T, B)])
    adv, ret = TP.estimate_advantages(torch.tensor(rewards), torch.tensor(masks), values, 0.99, 0.95)
    exps_t = torch.tensor(exps)
    np.random.seed(seed)
    order, losses = np.arange(T), []
    for _ in range(EPOCHS):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]
        for i in range(int(math.floor(T / B))):
            idx = order[i * B:(i + 1) * B]
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(agent.step(MP.stack_states([states[j] for j in idx]), act[idx], adv[idx], ret[idx],
                                     fixed[idx], ind))
    return agent.flat(), np.array(losses), adv.numpy(), fixed.numpy()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_update_params_at_the_concept_caps_matches_oracle_port(model):
    from drl_urban_planning_b200.ppo import PPOUpdater
    dev = torch.device("cuda", 0)
    states, actions, rewards, masks, exps, at = rollout()
    n = np.array([int(st[4].sum()) for st in states])
    assert sorted(n[at][n[at] > 1000].tolist()) == [1001, 1500, 1500, 1500] and (np.delete(n, at) <= 470).all()
    flat = PL.default_init(SEED) if model == "sgnn" else PL.MLP.default_init(SEED)
    if model == "sgnn":
        want, want_losses, adv, _, fixed = port_update_params(flat, states, actions, rewards, masks, exps, 0.99, 0.95,
                                                              EPOCHS, B, seed=7)
    else:
        want, want_losses, adv, fixed = mlp_port_update(flat, states, actions, rewards, masks, exps, seed=7)
    spec = synth.COMMUNITIES["hlg_concept"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, gamma=0.99, tau=0.95, opt_num_epochs=EPOCHS,
                    mini_batch_size=B, clip_mode=_lib.CLIP_REFERENCE, model=model)
    logged = []
    np.random.seed(7)
    up.update_params(states, actions, rewards, masks, exps, log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    assert rel(up.advantages.cpu().numpy(), adv.ravel()) < 1e-5
    assert rel(up.fixed_log_probs.cpu().numpy(), fixed.ravel()) < 1e-5
    got = np.array([v for tag, v, s in logged if tag == "loss/loss"])
    assert got.shape[0] == EPOCHS * (T // B)
    assert np.allclose(got, want_losses[:, 0], rtol=2e-4, atol=2e-5), (got, want_losses[:, 0])
    assert rel(up.flat_params(), want) < 2e-5
