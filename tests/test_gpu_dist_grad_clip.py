"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with the global gradient-norm clip (max_grad_norm) reproduces the
single-GPU run.  The SGNN keeps the in-kernel peer exchange (every rank forms the norm from all ranks' contributions
in its own buffer) or takes the NCCL all-reduce + upb_apply; the rl-mlp takes the all-reduce.  Parameters and the
norm (slot 17) of every minibatch of the last epoch are compared with one GPU."""
import numpy as np
import pytest
import torch

from harness import spawn
from test_gpu_dist_value_clip import _make_case

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))
M = 0.05


def _run(model, device, **kw):
    from drl_urban_planning_b200 import _lib, synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat, states, actions, rewards, masks, exps = _make_case(model)
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, gamma=0.99, tau=0.95, opt_num_epochs=2,
                    mini_batch_size=32, model=model, clip_mode=_lib.CLIP_NEVER, max_grad_norm=M, **kw)
    np.random.seed(5)
    up.update_params(states, actions, rewards, masks, exps)
    so, nb = up.engine.stat_offset, len(states) // 32
    return up, up.flat_params(), up._grad_ring[:nb, so + 17].cpu().numpy()


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat, norms = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        assert up.engine.peer_timeouts() == 0 if use_peers else True
        mine = torch.as_tensor(flat, device=dev)
        both = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(both, mine)
        outs[(model, mode)] = (flat, norms, all(torch.equal(both[0], b) for b in both))
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_with_the_global_clip_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)[0]
    for model, mode, _ in MODES:
        _, want, want_norms = _run(model, torch.device("cuda", 0), process_group=None)
        flat, norms, identical = got[(model, mode)]
        assert identical, (model, mode)
        assert (want_norms > M).all()
        assert np.allclose(norms, want_norms, rtol=1e-5), (model, mode)
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
