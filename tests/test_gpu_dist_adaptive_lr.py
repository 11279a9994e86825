"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with the KL-adaptive lr (desired_kl).  Every rank decides on the same
globally reduced statistics -- inside the fused step after the in-kernel peer exchange (the SGNN), or in upb_apply after
the NCCL all-reduce -- so every rank ends with the same lr state, the same decisions and the same parameters, which match
one GPU."""
import numpy as np
import pytest
import torch

from harness import spawn
from test_gpu_dist_value_clip import _make_case

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))
DESIRED_KL = 2e-3


def _run(model, device, **kw):
    """(updater, flat, counters, final lr state, lr_changes) of one update."""
    from drl_urban_planning_b200 import _lib, synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat, states, actions, rewards, masks, exps = _make_case(model)
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, lr=3e-3, gamma=0.99, tau=0.95,
                    opt_num_epochs=3, mini_batch_size=32, model=model, clip_mode=_lib.CLIP_NEVER,
                    desired_kl=DESIRED_KL, lr_bounds=(1e-4, 1e-2), **kw)
    np.random.seed(5)
    out = up.update_params(states, actions, rewards, masks, exps)
    _, _, steps = up.engine.get_opt_state()
    return up, up.flat_params(), steps, np.asarray([out["lr"]], np.float64), out["lr_changes"]


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat, steps, lr, changes = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        assert up.engine.peer_timeouts() == 0 if use_peers else True
        same = True
        for mine in (torch.as_tensor(flat, device=dev), torch.as_tensor(steps, device=dev),
                     torch.as_tensor(lr, device=dev)):
            every = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(every, mine)
            same = same and all(torch.equal(every[0], x) for x in every)
        outs[(model, mode)] = (flat, steps, lr, changes, same)
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_adapts_the_same_lr_on_every_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)[0]
    for model, mode, _ in MODES:
        _, want, want_steps, want_lr, want_changes = _run(model, torch.device("cuda", 0), process_group=None)
        flat, steps, lr, changes, same = got[(model, mode)]
        assert same, (model, mode)                               # every rank holds the same bits
        assert steps.tolist() == want_steps.tolist(), (model, mode)
        assert lr.tolist() == want_lr.tolist() and changes == want_changes, (model, mode, lr, want_lr)
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
