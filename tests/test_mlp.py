"""rl-mlp ablation (reference create_mlp_model, urban_planning/models/model.py:22-33; MLPStateEncoder,
state_encoder.py:217-308).  CPU: the oracle restatement and the drop-in modules against golden vectors produced by the
unmodified reference; GPU: the CUDA path (k_mlp) through the C ABI against the same vectors."""
import os

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from fixtures_io import expand_states
from harness import Agent, Cfg, per_tensor_rel, rel, tensorfy
from oracle import mlp_port as MP

FIXTURES = ["mlp_small", "mlp_hlg", "mlp_caps_concept"]
L = PL.MLP


@pytest.fixture(scope="module", params=FIXTURES)
def fx(request, golden_dir):
    z = np.load(os.path.join(golden_dir, request.param + ".npz"))
    return request.param, z, expand_states(z)


def test_mlp_port_matches_reference(fx):
    name, z, states = fx
    b = MP.stack_states(states)
    P = MP.params_from_flat(z["params"])
    with torch.no_grad():
        v = MP.value(P, b)
        lp, ent = MP.log_prob_entropy(P, b, torch.tensor(z["actions"]))
        greedy = MP.greedy_action(P, b)
    assert rel(v.numpy(), z["values"]) < 2e-6 and rel(lp.numpy(), z["log_probs"]) < 2e-6
    assert rel(ent.numpy(), z["entropies"]) < 2e-6
    assert np.array_equal(greedy.numpy(), z["greedy"])
    agent = MP.MLPPortAgent(z["params"])
    ind = torch.tensor(z["exps"]).nonzero(as_tuple=False).squeeze(1)
    args = (b, torch.tensor(z["actions"]), torch.tensor(z["advantages"]), torch.tensor(z["returns"]),
            torch.tensor(z["fixed_log_probs"]), ind)
    for k in range(3):
        losses = agent.step(*args)
        assert np.allclose(losses, z["losses"][k], rtol=2e-5, atol=2e-6), (k, losses, z["losses"][k])
        assert rel(agent.flat(), z["params_after"][k]) < 5e-6
    agent2 = MP.MLPPortAgent(z["params"])
    agent2.backward(*args)
    assert per_tensor_rel(agent2.flat_grad(), z["grads"][0], L)[0] < 5e-5


def test_mlp_dropin_modules_match_reference(fx):
    """create_mlp_model: same keys, bit-identical seeded init, CPU rollout path."""
    from drl_urban_planning_b200.mlp import ActorCritic, create_mlp_model
    name, z, states = fx
    torch.manual_seed(111)
    p, v = create_mlp_model(Cfg(int(z["n_cap"]), int(z["e_cap"])), Agent())
    ac = ActorCritic(p, v)
    want = [k for s in L.slots.values() for k in PL.state_dict_keys(s)]
    assert sorted(ac.state_dict().keys()) == sorted(want)
    assert np.array_equal(L.from_state_dict(ac.state_dict()), z["params"])
    assert sum(q.numel() for q in ac.parameters()) == L.num_params
    ts = tensorfy(states)
    with torch.no_grad():
        val = v(ts)
        lp, ent = p.get_log_prob_entropy(ts, torch.tensor(z["actions"]))
        greedy = p.select_action(ts, mean_action=True)
    assert rel(val.numpy(), z["values"]) < 1e-5 and rel(lp.numpy(), z["log_probs"]) < 1e-5
    assert rel(ent.numpy(), z["entropies"]) < 1e-5
    assert np.array_equal(greedy.numpy(), z["greedy"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_mlp_cuda_path_matches_reference(name, golden_dir):
    from drl_urban_planning_b200.engine import Engine
    from drl_urban_planning_b200.packing import pack_states
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    states = expand_states(z)
    dev = torch.device("cuda", 0)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)
    B = len(states)
    blob = pack_states(states).to(dev)
    eng = Engine(dev, blob.n_cap, blob.e_cap, clip_mode=_lib.CLIP_REFERENCE, model="mlp")
    params = t(z["params"]).clone()
    value, logp, ent, greedy = eng.forward(blob, params, t(z["actions"]), want_greedy=True)
    assert rel(value.cpu().numpy(), z["values"].ravel()) < 1e-4
    assert rel(logp.cpu().numpy(), z["log_probs"].ravel()) < 1e-4
    assert rel(ent.cpu().numpy(), z["entropies"].ravel()) < 1e-4
    stage = z["stage"][:, :2].argmax(1)
    assert np.array_equal(greedy.cpu().numpy().astype(np.int64), z["greedy"][np.arange(B), stage].astype(np.int64))
    n_ind = int((z["exps"] != 0).sum())
    args = (t(z["actions"]), t(z["advantages"]), t(z["returns"]), t(z["fixed_log_probs"]), t(z["exps"]))
    for k in range(3):
        grad = eng.ppo_grad(blob, params, *args, 1.0 / B, 1.0 / n_ind)
        losses = eng.read_losses(grad)
        g = grad.cpu().numpy()
        assert np.allclose(losses, z["losses"][k], rtol=1e-4, atol=1e-5), (k, losses, z["losses"][k])
        worst, where = per_tensor_rel(g[:L.num_params], z["grads"][k], L)
        assert worst < 1e-4, (k, worst, where)
        eng.apply(params, grad)
        torch.cuda.synchronize()
        assert rel(params.cpu().numpy(), z["params_after"][k]) < 1e-5, k


@pytest.mark.gpu
def test_mlp_update_params_runs_on_the_updater():
    """The whole iteration (PPOUpdater with model="mlp": forward sweep, GAE, epochs x minibatches on the two-call path)
    against the oracle port driven the same way."""
    import math
    from drl_urban_planning_b200.ppo import PPOUpdater
    dev = torch.device("cuda", 0)
    T, B, epochs = 48, 16, 2
    states, actions = synth.make_states(71, "small", T)
    rng = np.random.default_rng(71)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    flat = L.default_init(71)
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, gamma=0.99, tau=0.95, opt_num_epochs=epochs,
                    mini_batch_size=B, model="mlp")
    np.random.seed(4)
    up.update_params(states, actions, rewards, masks)
    # oracle port, same control flow
    from oracle import torch_port as TP
    agent = MP.MLPPortAgent(flat)
    b_all = MP.stack_states(states)
    act = torch.tensor(actions)
    with torch.no_grad():
        values = MP.value(agent.P, b_all)
        fixed, _ = MP.log_prob_entropy(agent.P, b_all, act)
    adv, ret = TP.estimate_advantages(torch.tensor(rewards), torch.tensor(masks), values, 0.99, 0.95)
    np.random.seed(4)
    order = np.arange(T)
    for _ in range(epochs):
        perm = np.arange(T); np.random.shuffle(perm)
        order = order[perm]
        for i in range(int(math.floor(T / B))):
            idx = order[i * B:(i + 1) * B]
            agent.step(MP.stack_states([states[j] for j in idx]), act[idx], adv[idx], ret[idx], fixed[idx],
                       torch.arange(B))
    assert rel(up.flat_params(), agent.flat()) < 2e-5


@pytest.mark.gpu
def test_mlp_large_graphs_and_edge_cases_match_oracle_port():
    """k_mlp beyond its shared-memory budget (n > 464 or 2e > 5632: the global-scratch path), both stages, an empty
    action mask and exps = 0 rows, against the oracle port (autograd) on the same padded states."""
    from drl_urban_planning_b200.engine import Engine
    from drl_urban_planning_b200.packing import pack_states
    dev = torch.device("cuda", 0)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)
    sizes = [600, 40, 900, 470, 300, 12]
    stages = [0, 1, 0, 1, 0, 0]
    states, actions = synth.make_states(13, "hlg", len(sizes), sizes=sizes, stages=stages)
    states[5][6][:] = False                                   # empty land-use mask: uniform over the padded width
    count = len(states)
    adv, ret, exps = synth.make_ppo_targets(13, count)
    exps[1] = 0.0
    fixed = np.full((count, 1), -3.3, np.float32)
    flat = L.default_init(13)
    blob = pack_states(states).to(dev)
    assert (blob.info[:, 0] > 464).sum() >= 2
    eng = Engine(dev, blob.n_cap, blob.e_cap, model="mlp")
    params = t(flat)
    value, logp, ent, greedy = eng.forward(blob, params, t(actions), want_greedy=True)
    n_ind = int((exps != 0).sum())
    grad = eng.ppo_grad(blob, params, t(actions), t(adv), t(ret), t(fixed), t(exps), 1.0 / count, 1.0 / n_ind)
    torch.cuda.synchronize()
    agent = MP.MLPPortAgent(flat)
    b = MP.stack_states(states)
    act = torch.tensor(actions)
    ind = torch.tensor(exps).nonzero(as_tuple=False).squeeze(1)
    with torch.no_grad():
        v_ref = MP.value(agent.P, b).numpy().ravel()
        lp_ref, en_ref = MP.log_prob_entropy(agent.P, b, act)
        gr_ref = MP.greedy_action(agent.P, b).numpy()
    losses = agent.backward(b, act, torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    assert rel(value.cpu().numpy(), v_ref) < 1e-4
    assert rel(logp.cpu().numpy(), lp_ref.numpy().ravel()) < 1e-4
    assert rel(ent.cpu().numpy(), en_ref.numpy().ravel()) < 1e-4
    st = np.array(stages)
    keep = np.arange(count) != 5                              # the empty mask has no defined arg-max
    assert np.array_equal(greedy.cpu().numpy()[keep], gr_ref[np.arange(count), st][keep].astype(np.int64))
    assert np.allclose(eng.read_losses(grad), losses, rtol=1e-4, atol=1e-5)
    worst, where = per_tensor_rel(grad.cpu().numpy()[:L.num_params], agent.flat_grad(), L)
    assert worst < 1e-4, (worst, where)
