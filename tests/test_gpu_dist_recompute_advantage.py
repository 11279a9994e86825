"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with recompute_advantage and value clipping.  Every rank sweeps the
whole buffer with the parameters it holds, which are the same bits on every rank, so every rank holds the same targets
without an exchange.  The SGNN runs the in-kernel peer exchange or the NCCL all-reduce + upb_apply; the rl-mlp the
all-reduce.  The advantages, returns and anchors of every epoch, the parameters, both moments and the counters are
identical on every rank and match one GPU."""
import numpy as np
import pytest
import torch

from harness import spawn
from test_gpu_dist_value_clip import _make_case

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))


def _run(model, device, **kw):
    """(flat, Adam m, v, counters, the recomputed targets of epochs 1 and 2 concatenated)."""
    from drl_urban_planning_b200 import _lib, synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat, states, actions, rewards, masks, exps = _make_case(model)
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, gamma=0.99, tau=0.95, opt_num_epochs=3,
                    mini_batch_size=32, model=model, clip_mode=_lib.CLIP_NEVER, value_clip=0.2,
                    recompute_advantage=True, **kw)
    targets = []
    recompute = up.recompute_targets

    def spy():
        recompute()
        targets.append(torch.cat([up.advantages, up.returns, up.old_values]))

    up.recompute_targets = spy
    np.random.seed(5)
    up.update_params(states, actions, rewards, masks, exps)
    m, v, steps = up.engine.get_opt_state()
    assert len(targets) == 2
    return up, up.flat_params(), m, v, steps, torch.cat(targets).cpu().numpy()


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat, m, v, steps, targets = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        assert up.engine.peer_timeouts() == 0 if use_peers else True
        floats = torch.as_tensor(np.concatenate([flat, m, v, targets]), device=dev)
        ints = torch.as_tensor(steps, device=dev)
        same = True
        for mine in (floats, ints):
            every = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(every, mine)
            same = same and all(torch.equal(every[0], x) for x in every)
        outs[(model, mode)] = (flat, steps, targets, same)
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_recomputes_the_same_targets_on_every_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)[0]
    for model, mode, _ in MODES:
        _, want, _, _, want_steps, want_targets = _run(model, torch.device("cuda", 0), process_group=None)
        flat, steps, targets, same = got[(model, mode)]
        assert same, (model, mode)                               # every rank holds the same bits
        assert steps.tolist() == want_steps.tolist(), (model, mode)
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
        assert np.abs(targets - want_targets).max() <= 1e-5 * max(np.abs(want_targets).max(), 1.0), (model, mode)
