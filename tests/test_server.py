"""Batching inference server for the forked rollout workers (SURVEY 8(f)-2).  CPU: the multi-process plumbing with a
plain-PyTorch policy as `infer_fn`; GPU: the real engine behind it (greedy actions bit-exact)."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import synth
from drl_urban_planning_b200.server import InferenceServer
from harness import Agent, Cfg, run_clients


def test_server_batches_requests_from_forked_workers():
    from drl_urban_planning_b200.model import create_sgnn_model
    spec = synth.COMMUNITIES["tiny"]
    torch.manual_seed(2)
    policy, _ = create_sgnn_model(Cfg(spec.max_num_nodes, spec.max_num_edges), Agent())
    states, _ = synth.make_states(8, "tiny", 12)
    tens = lambda sts: [[torch.tensor(np.array(x)) for x in s] for s in sts]

    def infer(sts, uniforms):                      # CPU stand-in for upb_select_action (greedy only)
        assert np.isnan(uniforms).all()
        with torch.no_grad():
            a = policy.select_action(tens(sts), mean_action=True).numpy()
        stage = np.array([int(np.argmax(s[8][:2])) for s in sts])
        return a[np.arange(len(sts)), stage].astype(np.int64)

    with InferenceServer(infer, spec.max_num_nodes, spec.max_num_edges, num_workers=3, max_wait_s=5e-3) as server:
        per_worker = [states[0:4], states[4:8], states[8:12]]
        res = run_clients(server, per_worker, True)
    assert server.error is None
    with torch.no_grad():
        want = policy.select_action(tens(states), mean_action=True).numpy()
    for w in range(3):
        assert np.array_equal(res[w], want[4 * w:4 * w + 4])
    assert sum(server.batches) == 12 and max(server.batches) >= 2          # requests were served in batches


def test_server_rejects_wrong_padding_and_survives_errors():
    spec = synth.COMMUNITIES["tiny"]
    states, _ = synth.make_states(8, "tiny", 2)

    def infer(sts, uniforms):
        raise RuntimeError("boom")
    with InferenceServer(infer, spec.max_num_nodes, spec.max_num_edges, num_workers=1) as server:
        c = server.client(0)
        with pytest.raises(RuntimeError):
            c.select_action([states[0]], True)            # the worker is released, not left blocked
        small, _ = synth.make_states(1, "small", 1)
        with pytest.raises(ValueError):
            c.select_action([small[0]], True)             # padded to other widths than the server's
    assert isinstance(server.error, RuntimeError)


@pytest.mark.gpu
def test_server_on_the_gpu_engine_matches_direct_calls():
    from drl_urban_planning_b200 import params as PL
    from drl_urban_planning_b200.engine import Engine
    from drl_urban_planning_b200.packing import pack_states
    dev = torch.device("cuda", 0)
    spec = synth.COMMUNITIES["small"]
    states, actions = synth.make_states(33, "small", 24)
    eng = Engine(dev, spec.max_num_nodes, spec.max_num_edges)
    params = torch.as_tensor(PL.default_init(33), device=dev)
    blob = pack_states(states).to(dev)
    greedy = eng.select_action(blob, params).cpu().numpy()
    server = InferenceServer.for_engine(eng, params, spec.max_num_nodes, spec.max_num_edges, num_workers=4,
                                        max_wait_s=5e-3)
    with server:
        per_worker = [states[6 * w:6 * w + 6] for w in range(4)]
        res = run_clients(server, per_worker, True)
        sampled = run_clients(server, per_worker, False)
    assert server.error is None
    for w in range(4):
        for j in range(6):
            i = 6 * w + j
            sid = int(np.argmax(states[i][8][:2]))
            assert res[w][j, sid] == greedy[i] and res[w][j, 1 - sid] == 0
            mask = states[i][6] if sid == 0 else states[i][7]
            assert mask[int(sampled[w][j, sid])]                 # sampled actions are feasible
    assert max(server.batches) >= 2
