"""GPU, 2 ranks (NCCL): the gradient-noise measurement of a data-parallel PPOUpdater (grad_noise_every), on the SGNN's
in-kernel peer exchange and on the NCCL all-reduce path of both models.  Each rank measures its own shard; one
all-reduce of (U, V, D) per update makes every rank report the same estimate, which equals the combination of the two
shards' measurements taken one process at a time."""
import numpy as np
import pytest
import torch

from harness import spawn

pytestmark = pytest.mark.gpu
MODES = (("sgnn", "nccl", False), ("sgnn", "peers", True), ("mlp", "nccl", False))
T, B = 96, 32


def _make_case(model):
    from drl_urban_planning_b200 import params as PL
    from harness import reproducible_states
    states, actions = reproducible_states(78, T)
    rng = np.random.default_rng(78)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[7::8] = 0.0
    exps = np.ones(T, np.float32); exps[3::11] = 0.0
    flat = PL.MLP.default_init(78) if model == "mlp" else PL.default_init(78)
    return flat, states, actions, rewards, masks, exps


def _worker(rank, world):
    import torch.distributed as dist
    from drl_urban_planning_b200 import _lib, synth
    from drl_urban_planning_b200.ppo import PPOUpdater
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    spec = synth.COMMUNITIES["small"]
    outs = {}
    for model, mode, use_peers in MODES:
        flat, states, actions, rewards, masks, exps = _make_case(model)
        # one epoch, and a period above its 3 steps: only step 0 is measured, at the parameters every rank starts from
        up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, lr=3e-3, gamma=0.99, tau=0.95,
                        opt_num_epochs=1, mini_batch_size=B, model=model, clip_mode=_lib.CLIP_NEVER,
                        use_peers=use_peers, grad_noise_every=8)
        assert up.world == world and up.fused_exchange == use_peers
        np.random.seed(5)
        out = up.update_params(states, actions, rewards, masks, exps)
        got = torch.tensor([out[k] for k in ("grad_noise_scale", "grad_noise_g2", "grad_noise_trace",
                                             "grad_noise_samples")], dtype=torch.float64, device=dev)
        every = [torch.empty_like(got) for _ in range(world)]
        dist.all_gather(every, got)
        # this rank's shard of minibatch 0, measured again by this process alone at the starting parameters
        np.random.seed(5)
        perm = np.arange(T)
        np.random.shuffle(perm)
        shard = perm[:B][rank::world]
        ids = np.random.default_rng([0, 0, 0, rank]).permutation(shard).astype(np.int32)
        n_ind = int((exps[perm[:B]] != 0).sum())
        _, noise = up.engine.ppo_grad_noise(up.blob, torch.as_tensor(flat, device=dev), up.actions, up.advantages,
                                            up.returns, up.fixed_log_probs, up.exps, 1.0 / B, 1.0 / n_ind,
                                            ids=torch.as_tensor(ids, device=dev))
        rows = [torch.empty_like(noise) for _ in range(world)]
        dist.all_gather(rows, noise)
        outs[(model, mode)] = ([x.cpu().numpy() for x in every], [r.cpu().numpy() for r in rows])
    dist.destroy_process_group()
    return outs


def test_two_gpu_update_reports_the_combined_estimate_on_every_rank():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from drl_urban_planning_b200.engine import grad_noise_estimate, grad_noise_terms
    got = spawn(2, _worker)
    for model, mode, _ in MODES:
        reports, rows = got[0][(model, mode)]
        assert all(r.tobytes() == reports[0].tobytes() for r in reports), (model, mode)       # every rank the same
        assert got[1][(model, mode)][0][0].tobytes() == reports[0].tobytes()
        assert [r[3] for r in rows] == [B / 2, B / 2]
        U, V, D = np.add(grad_noise_terms(rows[0]), grad_noise_terms(rows[1]))
        want = grad_noise_estimate(U, V, D, B, 1)
        assert np.allclose(reports[0], [want[k] for k in ("grad_noise_scale", "grad_noise_g2", "grad_noise_trace",
                                                          "grad_noise_samples")], rtol=1e-12, atol=0), (model, mode)
