"""GPU, 2 ranks (NCCL): the EWMA proximal policy (prox_ewma) of a data-parallel PPOUpdater, on the SGNN's in-kernel peer
exchange and on the NCCL all-reduce path (k_apply) of both models.  Every rank applies the same reduced gradient, so
every rank holds the same parameters and the same theta_prox, without an exchange of its own; theta_prox is the fp32
replay of the update's parameter trajectory."""
import numpy as np
import pytest
import torch

from harness import spawn

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))
T, B = 96, 32


def _worker(rank, world):
    import torch.distributed as dist
    from drl_urban_planning_b200 import _lib, params as PL, synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    from harness import reproducible_states
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    spec = synth.COMMUNITIES["small"]
    states, actions = reproducible_states(79, T)
    rng = np.random.default_rng(79)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    outs = {}
    for model, mode, use_peers in MODES:
        flat = PL.MLP.default_init(79) if model == "mlp" else PL.default_init(79)
        up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, lr=3e-3, gamma=0.99, tau=0.95,
                        opt_num_epochs=2, mini_batch_size=B, model=model, clip_mode=_lib.CLIP_NEVER,
                        use_peers=use_peers, prox_ewma=0.7)
        assert up.world == world and up.fused_exchange == use_peers
        np.random.seed(5)
        up.update_params(states, actions, rewards, masks)
        p = torch.as_tensor(up.flat_params(), device=dev)
        q = torch.as_tensor(up.engine.get_prox_params(), device=dev)
        ps, qs = [torch.empty_like(p) for _ in range(world)], [torch.empty_like(q) for _ in range(world)]
        dist.all_gather(ps, p)
        dist.all_gather(qs, q)
        outs[(model, mode)] = ([x.cpu().numpy() for x in ps], [x.cpu().numpy() for x in qs])
    dist.destroy_process_group()
    return outs


def test_two_gpu_ranks_hold_the_same_prox_params():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)
    for model, mode, _ in MODES:
        ps, qs = got[0][(model, mode)]
        assert ps[0].tobytes() == ps[1].tobytes(), (model, mode)
        assert qs[0].tobytes() == qs[1].tobytes(), (model, mode)
        assert not np.array_equal(qs[0], ps[0]), (model, mode)         # the average lags the parameters
