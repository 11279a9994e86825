"""GPU, 2 ranks (NCCL): a data-parallel PPOUpdater with adam_options, AdamW with AMSGrad through the context's
synthesised table.  The SGNN keeps the in-kernel peer exchange (k_sgnn_pg) or takes the NCCL all-reduce + upb_apply
(k_apply's table); the rl-mlp takes the all-reduce.  On every rank the parameters, both moments, max_exp_avg_sq, the
counters and the gradient rows of the last epoch are identical and match one GPU; ranks whose settings differ raise
before the first step."""
import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib
from harness import spawn
from test_gpu_dist_value_clip import _make_case

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))


def _updater(model, device, **kw):
    from drl_urban_planning_b200 import synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    flat = _make_case(model)[0]
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, device, gamma=0.99, tau=0.95, opt_num_epochs=2,
                    mini_batch_size=32, model=model, clip_mode=_lib.CLIP_NEVER, adam_options=True, **kw)
    up.set_hyperparameters(weight_decay=0.01, eps=1e-8, amsgrad=True, decoupled_weight_decay=True)
    return up


def _run(model, device, **kw):
    """(flat, Adam m, v, max_exp_avg_sq, counters, gradient rows of the last epoch)."""
    _, states, actions, rewards, masks, exps = _make_case(model)
    up = _updater(model, device, **kw)
    np.random.seed(5)
    up.update_params(states, actions, rewards, masks, exps)
    m, v, steps = up.engine.get_opt_state()
    rows = up._grad_ring[:len(states) // 32].cpu().numpy()
    return up, up.flat_params(), m, v, up.engine.get_amsgrad_state(), steps, rows


def _worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    outs = {}
    for model, mode, use_peers in MODES:
        up, flat, m, v, vmax, steps, rows = _run(model, dev, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        floats = torch.as_tensor(np.concatenate([flat, m, v, vmax, rows.ravel()]), device=dev)
        ints = torch.as_tensor(steps, device=dev)
        same = True
        for mine in (floats, ints):
            every = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(every, mine)
            same = same and all(torch.equal(every[0], x) for x in every)
        outs[(model, mode)] = (flat, m, v, vmax, steps, same)
    # a rank with another eps raises before the first step
    _, states, actions, rewards, masks, exps = _make_case("sgnn")
    up = _updater("sgnn", dev, use_peers=False)
    if rank == 1:
        up.set_hyperparameters(eps=1e-7)
    try:
        up.update_params(states, actions, rewards, masks, exps)
        outs["refused"] = False
    except _lib.UpbError as e:
        outs["refused"] = "eps" in str(e)
    dist.destroy_process_group()
    return outs


def test_two_gpu_adamw_amsgrad_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    got = spawn(2, _worker)
    for model, mode, _ in MODES:
        _, want, _, _, want_vmax, want_steps, _ = _run(model, torch.device("cuda", 0), process_group=None)
        flat, m, v, vmax, steps, same = got[0][(model, mode)]
        assert same, (model, mode)                               # every rank holds the same bits
        assert steps.tolist() == want_steps.tolist(), (model, mode)
        assert np.abs(flat - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0), (model, mode)
        assert vmax is not None and (vmax >= v).all(), (model, mode)
    assert got[0]["refused"] and got[1]["refused"]
