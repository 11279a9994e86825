"""GPU (H100): action selection through the drop-in modules and the inference server, for both models.  The
rl-mlp drop-in against its CPU path (the counterpart of test_gpu_update.py::test_dropin_modules_dispatch_to_cuda);
sampled selection with caller-supplied uniforms, and the server's sampled replies, against Engine.select_action on the
same uniforms."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states
from drl_urban_planning_b200.server import InferenceServer
from harness import Agent, Cfg, dev, rel, run_clients, t, tensorfy

pytestmark = pytest.mark.gpu

SPEC = synth.COMMUNITIES["small"]


def build(model, seed=3):
    from drl_urban_planning_b200.mlp import create_mlp_model
    from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
    torch.manual_seed(seed)
    p, v = (create_sgnn_model if model == "sgnn" else create_mlp_model)(Cfg(SPEC.max_num_nodes, SPEC.max_num_edges),
                                                                         Agent())
    return p, v, ActorCritic(p, v)


def test_mlp_dropin_modules_dispatch_to_cuda(dev):
    states, actions = synth.make_states(5, "small", 12)
    p, v, ac = build("mlp")
    ts = tensorfy(states)
    with torch.no_grad():
        val_c = v(ts)
        lp_c, ent_c = p.get_log_prob_entropy(ts, torch.tensor(actions))
        gr_c = p.select_action(ts, True)
    ac.to(dev)
    assert p.shared_net.model_kind == "mlp"
    val_g = v(states)
    lp_g, ent_g = p.get_log_prob_entropy([[x.to(dev) for x in s] for s in ts], torch.tensor(actions).to(dev))
    gr_g = p.select_action(states, mean_action=True)
    assert p._engine(dev).model == "mlp" and val_g.is_cuda and val_g.shape == (12, 1)
    assert rel(val_g.cpu().numpy(), val_c.numpy()) < 1e-4
    assert rel(lp_g.cpu().numpy(), lp_c.numpy()) < 1e-4 and rel(ent_g.cpu().numpy(), ent_c.numpy()) < 1e-4
    assert np.array_equal(gr_g.cpu().numpy(), gr_c.numpy())
    ac.to("cpu")
    assert np.array_equal(p.select_action(ts, True).numpy(), gr_c.numpy())


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_dropin_sampling_with_uniforms_matches_the_engine(model, dev):
    """UrbanPlanningPolicy.select_action(mean_action=False, uniforms=u) on CUDA: the engine's picks for u, written
    into the column of each state's stage."""
    states, _ = synth.make_states(6, "small", 16)
    p, v, ac = build(model)
    ac.to(dev)
    u = np.random.default_rng(6).random(16).astype(np.float32)
    u[:2] = [0.0, 1.0 - 2.0 ** -24]
    out = p.select_action(states, mean_action=False, uniforms=t(u, dev)).cpu().numpy()
    flat = (PL if model == "sgnn" else PL.MLP).from_state_dict(ac.state_dict())
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model=model)
    want = eng.select_action(pack_states(states).to(dev), t(flat, dev), uniforms=t(u, dev)).cpu().numpy()
    sid = np.array([int(np.argmax(s[8][:2])) for s in states])
    assert np.array_equal(out[np.arange(16), sid], want.astype(np.float32))
    assert not out[np.arange(16), 1 - sid].any()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_server_sampled_replies_match_the_engine(model, dev):
    """InferenceServer.for_engine serving sampled requests from forked workers seeded by client.seed: the parent
    regenerates each worker's uniform stream, converts it as the server does (float32, kept below 1), and every reply
    must equal engine.select_action on those uniforms."""
    states, _ = synth.make_states(33, "small", 24)
    flat = PL.default_init(33) if model == "sgnn" else PL.MLP.default_init(33)
    eng = Engine(dev, SPEC.max_num_nodes, SPEC.max_num_edges, model=model)
    params = t(flat, dev)
    per_worker = [states[6 * w:6 * w + 6] for w in range(4)]
    u = np.concatenate([np.random.default_rng(100 + w).random(6) for w in range(4)])      # run_clients seeds worker w with 100 + w
    u = np.minimum(u.astype(np.float32), np.nextafter(np.float32(1), np.float32(0)))
    want = eng.select_action(pack_states(states).to(dev), params, uniforms=t(u, dev)).cpu().numpy()
    server = InferenceServer.for_engine(eng, params, SPEC.max_num_nodes, SPEC.max_num_edges, num_workers=4,
                                        max_wait_s=5e-3)
    with server:
        sampled = run_clients(server, per_worker, False)
    assert server.error is None
    for w in range(4):
        for j in range(6):
            i = 6 * w + j
            sid = int(np.argmax(states[i][8][:2]))
            assert sampled[w][j, sid] == want[i] and sampled[w][j, 1 - sid] == 0, (w, j)
    assert max(server.batches) >= 2
