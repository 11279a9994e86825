"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with parameter groups and the shared encoder frozen.  The SGNN keeps
the in-kernel peer exchange (k_sgnn_pg: every rank masks the frozen columns of the rank-ordered sums and writes its own
per-tensor counts from the OR of the ranks' stage bits) or takes the NCCL all-reduce of the masked rows + upb_apply; the
rl-mlp takes the all-reduce.  On every rank the parameters, both moments, the per-segment counters, the per-tensor counts
and the gradient rows of the last epoch are identical; the encoder, its moments and its counts are untouched, its
gradient columns are 0, and the result matches one GPU."""
import numpy as np
import pytest
import torch

from harness import spawn
from test_gpu_dist_value_clip import _make_case

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))


def _run(model, device, **kw):
    """(initial flat, flat, Adam m, v, per-segment counters, per-tensor counts, gradient rows of the last epoch)."""
    from drl_urban_planning_b200 import _lib, params as PL, synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat, states, actions, rewards, masks, exps = _make_case(model)
    lay = PL.MLP if model == "mlp" else PL.SGNN
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, gamma=0.99, tau=0.95, opt_num_epochs=2,
                    mini_batch_size=32, model=model, clip_mode=_lib.CLIP_NEVER, param_groups=True, **kw)
    up.set_param_groups([dict(params=[n for n, s in lay.slots.items() if s.owner != "enc"], lr=4e-4,
                              weight_decay=1e-3)])
    np.random.seed(5)
    up.update_params(states, actions, rewards, masks, exps)
    m, v, steps = up.engine.get_opt_state()
    rows = up._grad_ring[:len(states) // 32].cpu().numpy()
    return up, flat, up.flat_params(), m, v, steps, up.engine.get_tensor_steps(), rows


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat0, flat, m, v, steps, ts, rows = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        assert up.engine.peer_timeouts() == 0 if use_peers else True
        floats = torch.as_tensor(np.concatenate([flat, m, v, rows.ravel()]), device=dev)
        ints = torch.as_tensor(np.concatenate([steps, ts]), device=dev)
        same = True
        for mine in (floats, ints):
            every = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(every, mine)
            same = same and all(torch.equal(every[0], x) for x in every)
        outs[(model, mode)] = (flat0, flat, m, v, steps, ts, rows, same)
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_with_a_frozen_encoder_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from drl_urban_planning_b200 import params as PL
    got = spawn(2, _worker)[0]
    for model, mode, _ in MODES:
        lay = PL.MLP if model == "mlp" else PL.SGNN
        enc, n_enc = lay.encoder_end, sum(1 for s in lay.slots.values() if s.owner == "enc")
        _, _, want, _, _, want_steps, want_ts, _ = _run(model, torch.device("cuda", 0), process_group=None)
        flat0, flat, m, v, steps, ts, rows, same = got[(model, mode)]
        assert same, (model, mode)                               # every rank holds the same bits
        assert np.array_equal(flat[:enc], flat0[:enc]), (model, mode)
        assert not m[:enc].any() and not v[:enc].any() and not rows[:, :enc].any(), (model, mode)
        assert not ts[:n_enc].any() and ts[n_enc:].all(), (model, mode)
        assert steps.tolist() == want_steps.tolist() and ts.tolist() == want_ts.tolist(), (model, mode)
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
