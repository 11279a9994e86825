"""GPU, 2 ranks (NCCL): data-parallel update_policy reproduces the single-GPU parameter trajectory (strong scaling:
the same global minibatches, each rank takes perm[...][rank::2]); the per-step exchange runs once as an NCCL all-reduce
of the gradient buffer and once inside the step kernel through peer memory (upb_peer_connect), with identical results."""
import numpy as np
import pytest
import torch

from harness import spawn

pytestmark = pytest.mark.gpu


def _make_case():
    from drl_urban_planning_b200 import params as PL, synth
    T = 96
    states, actions = synth.make_states(77, "small", T)
    rng = np.random.default_rng(77)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    return PL.default_init(77), states, actions, rewards, masks


def _run(updater, case, seed):
    flat, states, actions, rewards, masks = case
    np.random.seed(seed)
    updater.update_params(states, actions, rewards, masks)
    return updater.flat_params()


def _worker(rank, world):
    import torch.distributed as dist
    from drl_urban_planning_b200 import synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    case = _make_case()
    spec = synth.COMMUNITIES["small"]
    outs = {}
    for mode, use_peers in (("nccl", False), ("peers", True)):      # NCCL all-reduce per step / in-kernel peer exchange
        up = PPOUpdater(case[0], spec.max_num_nodes, spec.max_num_edges, torch.device("cuda", rank), gamma=0.99,
                        tau=0.95, opt_num_epochs=2, mini_batch_size=32, use_peers=use_peers)
        assert up.world == world and up.fused_exchange == use_peers
        outs[mode] = _run(up, case, seed=5)
        mine = torch.as_tensor(outs[mode], device=torch.device("cuda", rank))
        both = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(both, mine)
        outs[mode + "_ranks_identical"] = all(torch.equal(both[0], b) for b in both)
    outs["wide"] = _wide_grid_case(rank, world)
    dist.destroy_process_group()
    return outs


def _wide_grid_case(rank, world, steps=6):
    """Engine level, more graphs per rank than SMs (every CTA owns one 128-column slice: the single-pass shape of the
    fused tail), steps launched back to back without host synchronisation: peer exchange vs NCCL all-reduce."""
    import torch.distributed as dist
    from drl_urban_planning_b200 import params as PL, synth
    from drl_urban_planning_b200.engine import Engine
    from drl_urban_planning_b200.packing import pack_states
    dev = torch.device("cuda", rank)
    count = 200
    states, actions = synth.make_states(500 + rank, "small", count)
    blob = pack_states(states).to(dev)
    t = lambda x: torch.as_tensor(x, device=dev)
    adv, ret, exps = synth.make_ppo_targets(9 + rank, count)
    fixed = np.full((count, 1), -3.0, np.float32)
    res = {}
    for mode in ("nccl", "peers"):
        eng = Engine(dev, blob.n_cap, blob.e_cap)
        if mode == "peers":
            assert eng.connect_peers()
        params = t(PL.default_init(3)).clone()
        grad = eng.new_grad_buffer()
        args = (blob, params, t(actions), t(adv), t(ret), t(fixed), t(exps), 1.0 / (count * world), 1.0 / (count * world))
        for _ in range(steps):
            if mode == "peers" and eng.next_step_fused():
                eng.ppo_step(*args, out=grad)
            else:
                eng.ppo_grad(*args, out=grad)
                dist.all_reduce(grad)
                eng.apply(params, grad)
        torch.cuda.synchronize()
        res[mode] = params.cpu().numpy()
        res[mode + "_stats"] = grad[-28:-20].cpu().numpy()
    return res


def test_two_gpu_update_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from drl_urban_planning_b200 import synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    got = spawn(2, _worker)[0]
    case = _make_case()
    spec = synth.COMMUNITIES["small"]
    single = PPOUpdater(case[0], spec.max_num_nodes, spec.max_num_edges, torch.device("cuda", 0), gamma=0.99, tau=0.95,
                        opt_num_epochs=2, mini_batch_size=32, process_group=None)
    want = _run(single, case, seed=5)
    for mode in ("nccl", "peers"):
        assert got[mode + "_ranks_identical"]
        assert np.abs(got[mode] - want).max() <= 2e-6 * max(np.abs(want).max(), 1.0)
    # the two exchanges differ only in rounding (the attention chain runs before / after the cross-rank sum)
    assert np.abs(got["nccl"] - got["peers"]).max() <= 2e-6 * max(np.abs(want).max(), 1.0)
    wide = got["wide"]
    assert np.abs(wide["nccl"] - wide["peers"]).max() <= 2e-6 * max(np.abs(wide["nccl"]).max(), 1.0)
    assert np.allclose(wide["nccl_stats"], wide["peers_stats"], rtol=1e-5, atol=1e-6)
