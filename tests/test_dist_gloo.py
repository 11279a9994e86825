"""CPU, world_size 2 (gloo): the data-parallel decomposition of one global minibatch -- each rank takes
perm[...][rank::world], uses the GLOBAL 1/B and 1/|ind|, and a sum all-reduce of the flat [gradient | statistics]
buffer reproduces the single-process batch gradient and losses.  The per-rank gradient here comes from the numpy
oracle (the CUDA engine needs a GPU); the sharding / reduction host logic is what is under test."""
import numpy as np
import torch
import torch.distributed as dist

from drl_urban_planning_b200 import _lib, params as PL, synth
from harness import spawn


def _shard_buffer(flat, states, actions, adv, ret, fixed, exps, ids, B, n_ind):
    """What upb_ppo_grad returns for the graphs `ids` of a global minibatch of B graphs (oracle stand-in)."""
    from oracle import sgnn_numpy as ON
    buf = np.zeros(_lib.UPB_GRAD_STRIDE, np.float64)
    if len(ids) == 0:
        return buf
    sub = [states[i] for i in ids]
    r = ON.ppo_minibatch(flat, sub, actions[ids], adv[ids], ret[ids], fixed[ids], exps[ids])
    # ppo_minibatch normalises by the shard's own sizes; rescale the three loss terms to the global ones
    b, ni = len(ids), max(int((exps[ids] != 0).sum()), 1)
    P = ON._p64(flat)
    g = np.zeros(PL.NUM_PARAMS)
    for j, i in enumerate(ids):
        gph = ON.unpad(states[i]); sid = int(np.argmax(gph.stage[:2]))
        fw = ON.forward(P, gph, action=int(actions[i, sid]), keep=True)
        g_v = 2 * 0.5 * (fw["value"] - float(ret[i, 0])) / B
        g_lp = g_en = 0.0
        if exps[i] != 0:
            ratio = np.exp(fw["log_prob"] - float(fixed[i, 0])); A = float(adv[i, 0])
            s1, s2 = ratio * A, np.clip(ratio, 0.8, 1.2) * A
            if 0.8 <= ratio <= 1.2 or s1 < s2:
                g_lp = -A * ratio / n_ind
            g_en = -0.01 / n_ind
        G = ON.backward(P, gph, fw, g_v, g_lp, g_en)
        for s in PL.SLOTS.values():
            g[s.offset:s.offset + s.size] += G[s.name].reshape(-1)
    buf[:PL.NUM_PARAMS] = g
    st = buf[_lib.UPB_STAT_OFFSET:]
    st[0] = r["value_loss"] * b; st[1] = r["surr_loss"] * ni; st[2] = r["entropy_loss"] * ni
    st[3] = b; st[4] = int((exps[ids] != 0).sum())
    return buf


def _worker(rank, world):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B = 10
    states, actions = synth.make_states(3, "tiny", B)
    adv, ret, exps = synth.make_ppo_targets(3, B)
    exps[2] = 0
    fixed = np.full((B, 1), -2.5, np.float32)
    flat = PL.default_init(3)
    perm = np.random.default_rng(0).permutation(B)
    n_ind = int((exps != 0).sum())
    ids = perm[rank::world]                                   # PPOUpdater.update_policy sharding rule
    buf = torch.tensor(_shard_buffer(flat, states, actions, adv, ret, fixed, exps, ids, B, n_ind))
    dist.all_reduce(buf, op=dist.ReduceOp.SUM)                # PPOUpdater.allreduce
    dist.destroy_process_group()
    return buf.numpy()


def test_two_rank_shards_sum_to_batch_gradient():
    from oracle import sgnn_numpy as ON
    got = spawn(2, _worker, timeout=300)[0]
    B = 10
    states, actions = synth.make_states(3, "tiny", B)
    adv, ret, exps = synth.make_ppo_targets(3, B)
    exps[2] = 0
    fixed = np.full((B, 1), -2.5, np.float32)
    ref = ON.ppo_minibatch(PL.default_init(3), states, actions, adv, ret, fixed, exps)
    g = got[:PL.NUM_PARAMS]
    assert np.abs(g - ref["grad"]).max() <= 1e-9 * max(np.abs(ref["grad"]).max(), 1)
    st = got[_lib.UPB_STAT_OFFSET:]
    assert st[3] == B and st[4] == int((exps != 0).sum())
    assert np.isclose(st[0] / st[3], ref["value_loss"]) and np.isclose(st[1] / st[4], ref["surr_loss"])
    assert np.isclose(st[2] / st[4], ref["entropy_loss"])


def _order_worker(rank, world):
    """Host logic of PPOUpdater's sharding with DIFFERENT np.random seeds per rank (the usual torchrun setup)."""
    import types
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from drl_urban_planning_b200.ppo import PPOUpdater
    T = 37
    info = np.stack([np.arange(T) + 5, np.arange(T) * 3, np.arange(T) % 7, np.arange(T) % 2], 1).astype(np.int32)
    duck = types.SimpleNamespace(world=world, rank=rank, pg=None, device=torch.device("cpu"), batch_stage=False,
                                 _stage=info[:, 3].astype(np.int64), exps_host=np.ones(T, np.float32),
                                 actions=torch.zeros(T, 2))
    PPOUpdater._check_same_buffer(duck, info.astype(np.int64))            # identical buffers: passes
    np.random.seed(100 + rank)                                            # per-rank seeds
    order = np.arange(T)
    orders = []
    for _ in range(3):
        order = PPOUpdater._epoch_order(duck, order)
        orders.append(order.copy())
    bad = info.astype(np.int64).copy()
    if rank == 1:
        bad[3, 0] += 1                                                    # rank 1 holds a different buffer
    try:
        PPOUpdater._check_same_buffer(duck, bad)
        mismatch_detected = False
    except _lib.UpbError:
        mismatch_detected = True
    duck.batch_stage = True
    staged = PPOUpdater._epoch_order(duck, np.arange(T))
    dist.destroy_process_group()
    return np.stack(orders), mismatch_detected, staged


def test_rank0_order_is_broadcast_and_buffers_are_checked():
    res = spawn(2, _order_worker, timeout=300)
    assert np.array_equal(res[0][0], res[1][0])                 # every rank walks rank 0's permutations
    # rank 0's stream: composed permutations (urban_planning_agent.py:306-312)
    np.random.seed(100)
    order = np.arange(37)
    for k in range(3):
        perm = np.arange(37); np.random.shuffle(perm)
        order = order[perm]
        assert np.array_equal(res[0][0][k], order)
        B = 8
        for i in range(37 // B):                                # the two shards partition each global minibatch
            mb = order[i * B:(i + 1) * B]
            assert sorted(np.concatenate([mb[0::2], mb[1::2]]).tolist()) == sorted(mb.tolist())
    assert res[0][1] and res[1][1]                              # both ranks see the mismatch
    st = res[0][2] % 2                                          # stage = index % 2: land use first, road second
    assert np.array_equal(res[0][2], res[1][2]) and (np.diff(st) >= 0).all()
