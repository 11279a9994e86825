"""CPU: the host packer (reference 9-array states -> unpadded blob) against a numpy re-derivation, plus the
layout-contract errors and ragged / edge cases."""
import numpy as np
import pytest

from blobview import decode
from drl_urban_planning_b200 import _lib, synth
from drl_urban_planning_b200.packing import pack_states


def host_bytes(blob):
    h = blob.host
    return h.numpy() if hasattr(h, "numpy") else h


def check_blob(states, blob, unbalanced=()):
    """Re-derives every section of the blob from the states.  `unbalanced`: indices of graphs left out of the pull
    schedule's balance check (a hub row heavier than the whole bound; see tests/test_caps.py)."""
    d = decode(host_bytes(blob)[:blob.nbytes])
    assert d["header"]["count"] == len(states)
    for i, st in enumerate(states):
        numerical, nf, ei, cur, nm, em, lum, rm, stage = st
        g = d["desc"][i]
        n, e = int(nm.sum()), int(em.sum())
        assert (g["n"], g["e"]) == (n, e)
        assert g["stage"] == int(np.argmax(stage[:2]))
        x = d["x"][g["x_row"]:g["x_row"] + n]
        assert np.array_equal(x[:, :23], nf[:n]) and not x[:, 23].any()
        assert np.array_equal(d["num"][i], numerical) and np.array_equal(d["cur"][i][:23], cur)
        rp = d["rowptr"][g["rp_off"]:g["rp_off"] + n + 1].astype(np.int64)
        adj = d["adj"][g["adj_off"]:g["adj_off"] + 2 * e]
        deg = np.bincount(ei[:e, 0], minlength=n) + np.bincount(ei[:e, 1], minlength=n)
        assert rp[0] == 0 and np.array_equal(np.diff(rp), deg)
        sched = d["order"][g["ord_off"]:g["ord_off"] + g["ord_rounds"] * 128].astype(np.int64).reshape(-1, 16, 8)
        listed = sched[sched != 0xFFFF]
        assert sorted(listed.tolist()) == list(range(n))            # every node exactly once
        load, heaviest = np.zeros(16), 0
        for r in range(sched.shape[0]):
            for w in range(16):
                grp = sched[r, w][sched[r, w] != 0xFFFF]
                if grp.size:
                    cost = (deg[grp].max() + 1) // 2 + 2
                    load[w] += cost
                    heaviest = max(heaviest, cost)
        if n >= 256 and i not in unbalanced:     # warps are balanced; a hub row's group can only run alone on its warp
            assert load.max() <= max(1.25 * load.mean() + 4, heaviest), load
        # the symmetrised adjacency holds every undirected edge exactly twice (once per endpoint)
        got = sorted((min(i_, int(a & 0xffff)), max(i_, int(a & 0xffff)))
                     for i_ in range(n) for a in adj[rp[i_]:rp[i_ + 1]])
        want = sorted((min(int(u), int(v)), max(int(u), int(v))) for u, v in ei[:e] for _ in range(2))
        assert got == want
        k = int(g["k"])
        cuv = d["cuv"][g["cand_off"]:g["cand_off"] + k]
        cidx = d["cidx"][g["cand_off"]:g["cand_off"] + k]
        if g["stage"] == 0:
            idx = np.flatnonzero(lum)
            assert np.array_equal(cidx, idx)
            assert np.array_equal(cuv & 0xffff, ei[idx, 0]) and np.array_equal(cuv >> 16, ei[idx, 1])
            # every directed entry of a candidate edge carries slot+1 in its upper half
            tagged = {}
            for i_ in range(n):
                for a in adj[rp[i_]:rp[i_ + 1]]:
                    if (a >> 16) & 0x7fff:
                        tagged.setdefault(int((a >> 16) & 0x7fff) - 1, []).append((i_, int(a & 0xffff)))
            assert sorted(tagged) == list(range(k))
            for s, ends in tagged.items():
                u, v = int(ei[idx[s], 0]), int(ei[idx[s], 1])
                assert sorted(ends) == sorted([(u, v), (v, u)])
        else:
            idx = np.flatnonzero(rm)
            assert np.array_equal(cidx, idx) and np.array_equal(cuv, idx)
            assert not ((adj >> 16) & 0x7fff).any()
        # bit 31: the row's node is the edge's FIRST endpoint -> exactly the directed entries (u -> v) of the edge list
        first = sorted((i_, int(a & 0xffff)) for i_ in range(n) for a in adj[rp[i_]:rp[i_ + 1]] if a >> 31)
        assert first == sorted((int(u), int(v)) for u, v in ei[:e])
    info = blob.info
    assert np.array_equal(info[:, 0], [int(s[4].sum()) for s in states])


@pytest.mark.parametrize("community,count", [("tiny", 40), ("small", 24), ("hlg", 6), ("hlg_concept", 3)])
def test_pack_matches_numpy(community, count):
    states, _ = synth.make_states(5, community, count)
    for threads in (1, 4):
        check_blob(states, pack_states(states, threads=threads, pinned=False))


def test_pack_edge_cases():
    spec = synth.COMMUNITIES["tiny"]
    rng = np.random.default_rng(0)
    s_one_node, _ = synth.make_state(rng, spec, n=1, stage=1, e=0)          # single node, no edges
    s_full, _ = synth.make_state(rng, spec, n=spec.max_num_nodes, stage=0)   # node cap reached
    s_no_cand, _ = synth.make_state(rng, spec, n=10, stage=0)
    s_no_cand[6][:] = False                                                  # empty action mask
    s_all_cand, _ = synth.make_state(rng, spec, n=12, stage=0)
    s_all_cand[6][:int(s_all_cand[5].sum())] = True                          # every real edge is a candidate
    states = [s_one_node, s_full, s_no_cand, s_all_cand]
    blob = pack_states(states, pinned=False)
    check_blob(states, blob)
    assert blob.info[0].tolist()[:2] == [1, 0] and blob.info[2][2] == 0


def test_pack_boundary_shapes():
    """The graphs of tests/test_gpu_shapes.py: exact n / 2e / k at the kernels' shape limits, a hub row, isolated
    nodes, odd-degree rows and the caps; the pull schedule covers every node once (check_blob) in each of them."""
    import shape_cases as SC
    states, _, _ = SC.boundary_batch()
    blob = pack_states(states, pinned=False)
    check_blob(states, blob)
    info = blob.info
    for (label, n, e, k, stage, hub, isolated), st, row in zip(SC.BOUNDARY, states, info):
        assert row[:4].tolist() == [n, e, k, stage], label
        deg = SC.degrees(st)
        assert (deg == 0).sum() == isolated, label
        if hub:
            assert deg.max() == n - 1, label
        ei = st[2]                       # the reference's edge list: u < v, sorted, distinct, pad value N - 1
        assert (ei[:e, 0] < ei[:e, 1]).all() and (ei[e:] == SC.SPEC.max_num_nodes - 1).all(), label
        key = ei[:e, 0] * SC.SPEC.max_num_nodes + ei[:e, 1]
        assert (np.diff(key) > 0).all(), label
    assert any((SC.degrees(st) % 2 == 1).any() for st in states)
    big = [SC.is_big(*r[:3]) for r in info]
    assert any(big) and not all(big)


def test_pack_accepts_torch_and_lists():
    import torch
    states, _ = synth.make_states(1, "tiny", 3)
    as_torch = [[torch.tensor(x) for x in s] for s in states]
    a = pack_states(states, pinned=False)
    b = pack_states(as_torch, n_cap=a.n_cap, e_cap=a.e_cap, pinned=False)
    assert np.array_equal(host_bytes(a)[:a.nbytes], host_bytes(b)[:b.nbytes])


@pytest.mark.parametrize("breaker,msg", [
    (lambda s: s[4].__setitem__(0, False), "prefix"),
    (lambda s: s[2].__setitem__((0, 0), 47), "padded node"),
    (lambda s: s[6].__setitem__(159, True), "padded edge"),
    (lambda s: s[8].__setitem__(slice(None), [0, 0, 1]), "one-hot"),
])
def test_pack_rejects_contract_violations(breaker, msg):
    rng = np.random.default_rng(1)
    st, _ = synth.make_state(rng, synth.COMMUNITIES["tiny"], n=20, stage=0)
    breaker(st)
    with pytest.raises(_lib.UpbError, match=msg):
        pack_states([st], pinned=False)


def test_fill_in_place_path_validates_edges():
    """With a caller-provided buffer the packer skips the measuring pass; the edge endpoints are then checked while the
    CSR is built (one read of the edge list), including negative indices, and nothing is written out of bounds."""
    import torch
    states, _ = synth.make_states(3, "tiny", 20)
    ref = pack_states(states, pinned=False)
    out = torch.empty(ref.nbytes + 4096, dtype=torch.uint8)
    same = pack_states(states, ref.n_cap, ref.e_cap, out_host=out)
    assert same.nbytes == ref.nbytes and np.array_equal(host_bytes(same)[:ref.nbytes], host_bytes(ref)[:ref.nbytes])
    for bad_value in (-1, 47, 2 ** 40):
        broken = [list(s) for s in states]
        broken[13][2] = broken[13][2].copy()
        broken[13][2][0, 1] = bad_value
        with pytest.raises(_lib.UpbError, match="state 13.*padded node"):
            pack_states(broken, ref.n_cap, ref.e_cap, out_host=out)


def test_pack_from_concurrent_threads_and_after_fork():
    """The worker pool is shared by all callers of a process and must be rebuilt in a forked child (the reference forks
    its rollout workers, khrylib/rl/agents/agent.py:83-89)."""
    import os, threading
    states, _ = synth.make_states(7, "small", 64)
    ref = pack_states(states, threads=1, pinned=False)
    want = host_bytes(ref)[:ref.nbytes].tobytes()
    errors = []

    def job():
        try:
            for _ in range(10):
                b = pack_states(states, threads=4, pinned=False)
                assert host_bytes(b)[:b.nbytes].tobytes() == want
        except Exception as ex:      # pragma: no cover
            errors.append(ex)

    ts = [threading.Thread(target=job) for _ in range(3)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errors
    pid = os.fork()
    if pid == 0:
        ok = 1
        try:
            b = pack_states(states, threads=4, pinned=False)
            ok = 0 if host_bytes(b)[:b.nbytes].tobytes() == want else 2
        finally:
            os._exit(ok)
    _, status = os.waitpid(pid, 0)
    assert os.WEXITSTATUS(status) == 0


def test_chunked_plan_fill_equals_one_shot_and_ranges_cover_the_blob():
    """upb_pack_plan_create / _fill (chunked packing for the overlapped upload of PackedGraphs.pack_and_upload): the blob
    is byte-identical to upb_pack_fill's and the byte ranges reported per chunk tile it exactly once."""
    import ctypes as C
    from drl_urban_planning_b200.packing import _pointer_table
    states, _ = synth.make_states(5, "small", 57)
    ref = pack_states(states, pinned=False)
    refb = np.asarray(ref.host)[:ref.nbytes] if not hasattr(ref.host, "numpy") else ref.host.numpy()[:ref.nbytes]
    L = _lib.lib()
    ptrs, keep = _pointer_table(states, ref.n_cap, ref.e_cap)
    plan, nb = C.c_void_p(), C.c_uint64()
    _lib.check(L.upb_pack_plan_create(len(states), ptrs.ctypes.data, ref.n_cap, ref.e_cap, 2, C.byref(plan), C.byref(nb)))
    assert nb.value == ref.nbytes
    raw = np.zeros(nb.value + 16, np.uint8)
    off = (-raw.ctypes.data) % 16
    host = raw[off:off + nb.value]
    covered = np.zeros(nb.value, np.int32)
    ranges = np.zeros((9, 2), np.uint64)
    for first in range(0, len(states), 10):
        cnt = min(10, len(states) - first)
        _lib.check(L.upb_pack_plan_fill(plan, ptrs.ctypes.data, first, cnt, 2, host.ctypes.data, nb.value,
                                        ranges.ctypes.data))
        for o, ln in ranges:
            covered[int(o):int(o) + int(ln)] += 1
    assert L.upb_pack_plan_fill(plan, ptrs.ctypes.data, 50, 10, 2, host.ctypes.data, nb.value, ranges.ctypes.data) != 0
    L.upb_pack_plan_destroy(plan)
    assert np.array_equal(host, refb)
    assert (covered == 1).all()
