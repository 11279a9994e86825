"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with the clipped value loss and the per-minibatch advantage
normalisation reproduces the single-GPU run.  Every rank normalises the whole epoch from the broadcast order and seeds its
graphs' values itself, so the exchanges carry nothing new: the SGNN through the NCCL all-reduce and through the in-kernel
peer exchange, the rl-mlp through the all-reduce.  Parameters and the value-clip statistics (slots 15 / 16) of every
minibatch of the last epoch are compared with one GPU."""
import numpy as np
import pytest
import torch

from harness import spawn

pytestmark = pytest.mark.gpu
OPTS = dict(value_clip=0.2, normalize_advantage=True)
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))


def _make_case(model):
    from drl_urban_planning_b200 import params as PL, synth
    T = 96
    states, actions = synth.make_states(78, "small", T)
    rng = np.random.default_rng(78)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    exps = np.ones(T, np.float32); exps[3::11] = 0.0
    flat = PL.MLP.default_init(78) if model == "mlp" else PL.default_init(78)
    return flat, states, actions, rewards, masks, exps


def _run(model, device, **kw):
    """(parameters, slots 15 / 16 of every minibatch row of the last epoch) of one update."""
    from drl_urban_planning_b200 import synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat, states, actions, rewards, masks, exps = _make_case(model)
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, gamma=0.99, tau=0.95, opt_num_epochs=2,
                    mini_batch_size=32, model=model, **OPTS, **kw)
    np.random.seed(5)
    up.update_params(states, actions, rewards, masks, exps)
    so, nb = up.engine.stat_offset, len(states) // 32
    return up, up.flat_params(), up._grad_ring[:nb, so + 15:so + 17].cpu().numpy()


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat, vclip = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        mine = torch.as_tensor(flat, device=dev)
        both = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(both, mine)
        outs[(model, mode)] = (flat, vclip, all(torch.equal(both[0], b) for b in both))
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_with_both_options_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)[0]
    for model, mode, _ in MODES:
        _, want, want_vclip = _run(model, torch.device("cuda", 0), process_group=None)
        flat, vclip, identical = got[(model, mode)]
        assert identical, (model, mode)
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
        assert want_vclip[:, 1].any()                                          # some clipped terms won
        assert np.allclose(vclip[:, 0], want_vclip[:, 0], rtol=1e-5), (model, mode)
        assert np.abs(vclip[:, 1] - want_vclip[:, 1]).max() <= 1, (model, mode)    # a graph on a tie may flip
