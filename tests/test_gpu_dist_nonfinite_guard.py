"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with the non-finite guard (skip_nonfinite) on a rollout with one
poisoned sample, which falls into one rank's shard of its minibatch.  With the SGNN's in-kernel peer exchange every rank
holds every rank's contributions and forms the same norm; on the NCCL path every rank decides in upb_apply on the
all-reduced buffer.  All ranks skip the same steps (slot 19 of every minibatch row of the last epoch), stay
bit-identical to each other, and match one GPU within the bar of the other two-GPU tests (the two shards' sums are
added in another order than one GPU's)."""
import numpy as np
import pytest
import torch

from harness import spawn

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))
POISON = 40           # the first step of its episode: the backward GAE scan ends there, so it alone is infinite


def _make_case(model):
    """96 small graphs in episodes of 8, a few with exps = 0; the same on every rank."""
    from drl_urban_planning_b200 import params as PL, synth
    T = 96
    states, actions = synth.make_states(78, "small", T)
    rng = np.random.default_rng(78)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32)
    masks[7::8] = 0.0
    exps = np.ones(T, np.float32)
    exps[3::11] = 0.0
    flat = PL.MLP.default_init(78) if model == "mlp" else PL.default_init(78)
    return flat, states, actions, rewards, masks, exps


def _run(model, device, **kw):
    from drl_urban_planning_b200 import _lib, synth
    from drl_urban_planning_b200.ppo import NONFINITE_SLOT, PPOUpdater
    flat, states, actions, rewards, masks, exps = _make_case(model)
    assert exps[POISON] != 0 and masks[POISON - 1] == 0
    rewards[POISON] = np.inf
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, gamma=0.99, tau=0.95, opt_num_epochs=2,
                    mini_batch_size=32, model=model, clip_mode=_lib.CLIP_NEVER, skip_nonfinite=True, **kw)
    np.random.seed(5)
    out = up.update_params(states, actions, rewards, masks, exps)
    so, nb = up.engine.stat_offset, len(states) // 32
    return up, up.flat_params(), up._grad_ring[:nb, so + NONFINITE_SLOT].cpu().numpy(), out["nonfinite_skips"]


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat, marks, skips = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        assert up.engine.peer_timeouts() == 0 if use_peers else True
        mine = torch.as_tensor(np.concatenate([flat, marks, [skips]]).astype(np.float32), device=dev)
        both = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(both, mine)
        outs[(model, mode)] = (flat, marks, skips, all(torch.equal(both[0], b) for b in both))
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_skips_the_same_steps_as_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)[0]
    for model, mode, _ in MODES:
        _, want, want_marks, want_skips = _run(model, torch.device("cuda", 0), process_group=None)
        flat, marks, skips, identical = got[(model, mode)]
        assert identical, (model, mode)
        assert want_skips == skips == 2 and want_marks.sum() == 1
        assert np.array_equal(marks, want_marks), (model, mode)
        assert np.isfinite(flat).all()
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
