"""CPU: the packer on graphs above the hlg caps (tests/cap_cases.py) -- the concept configs' 1500 / 4000 caps and the
blob format's 16-bit limits -- against check_blob's numpy re-derivation, the decoded fields that carry bit 15, and the
refusals at the limits: caps above 65535 / 32767, and action masks past the candidate limits (land use k <= e <= e_cap,
road k <= n <= n_cap; the caps are the only candidate limit)."""
import ctypes as C

import numpy as np
import pytest

import cap_cases as CC
from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.packing import _pointer_table, pack_states
from blobview import decode
from test_packing import check_blob, host_bytes


@pytest.fixture(scope="module")
def abi():
    states, actions, labels = CC.abi_batch()
    return states, labels, pack_states(states, pinned=False)


def graph_fields(blob, i):
    d = decode(host_bytes(blob)[:blob.nbytes])
    g = d["desc"][i]
    n, e, k = int(g["n"]), int(g["e"]), int(g["k"])
    return dict(n=n, e=e, k=k,
                rp=d["rowptr"][g["rp_off"]:g["rp_off"] + n + 1],
                adj=d["adj"][g["adj_off"]:g["adj_off"] + 2 * e],
                cuv=d["cuv"][g["cand_off"]:g["cand_off"] + k],
                order=d["order"][g["ord_off"]:g["ord_off"] + g["ord_rounds"] * 128])


def test_concept_caps_pack_exactly():
    states, _, labels = CC.concept_batch()
    blob = pack_states(states, pinned=False)
    assert (blob.n_cap, blob.e_cap) == (1500, 4000)
    for threads in (1, 4):
        check_blob(states, pack_states(states, threads=threads, pinned=False))
    info = blob.info
    for label, n, e, k, stage, hub, iso in CC.CONCEPT_CASES:
        assert info[labels.index(label)][:4].tolist() == [n, e, k, stage], label
    hub = states[labels.index("c_hub")]
    deg = np.bincount(hub[2][:4000].ravel(), minlength=1500)
    assert deg.max() == 1499


def test_abi_limits_pack_exactly(abi):
    """Every ABI-limit case re-derived from its state; the hub of degree 32767 is left out of the balance check only:
    its row alone costs 16,386 of the schedule's load units, more than the 1.25 x mean bound, and the round count is
    capped, so its warp must also take other groups."""
    states, labels, blob = abi
    assert (blob.n_cap, blob.e_cap) == (65535, 32767)
    check_blob(states, blob, unbalanced={labels.index(x) for x in CC.UNBALANCED})
    info = blob.info
    for label, n, e, k, stage, hub, iso in CC.ABI_CASES:
        assert info[labels.index(label)][:4].tolist() == [n, e, k, stage], label


def test_fields_with_bit_15_set(abi):
    states, labels, blob = abi
    # node ids: 65534 in the upper half (max_lu: v of a candidate edge) and lower half (max_road) of cand_uv, and an id
    # with bit 15 set as a land-use candidate's first endpoint (the reversed edge of max_lu)
    lu = graph_fields(blob, labels.index("max_lu"))
    assert lu["k"] == CC.MAX_LU_K and CC.TOP in (lu["cuv"] >> 16).tolist()
    assert CC.TOP - 1 in (lu["cuv"] & 0xFFFF).tolist()
    rd = graph_fields(blob, labels.index("max_road"))
    assert rd["k"] == CC.MAX_ROAD_K and np.array_equal(rd["cuv"], np.arange(CC.MAX_N))
    first = graph_fields(blob, labels.index("n32769_road"))
    assert 32768 in (first["adj"] & 0xFFFF).tolist()
    # slot + 1 runs to the top of the 15-bit field without touching bit 31's first-endpoint flag
    tags = (lu["adj"] >> 16) & 0x7FFF
    assert tags.max() == 32767 and np.array_equal(np.bincount(tags, minlength=32768)[1:], np.full(32767, 2))
    assert int((lu["adj"] >> 31).sum()) == lu["e"]
    # row pointers: 32768 and above
    for label, last in (("rp_e16383", 32766), ("rp_e16384", 32768), ("rp_e16385", 32770), ("hub32767", 65534),
                        ("max_lu", 65534)):
        f = graph_fields(blob, labels.index(label))
        assert int(f["rp"][-1]) == last == 2 * f["e"], label
        assert (np.diff(f["rp"].astype(np.int64)) >= 0).all(), label
    hub = graph_fields(blob, labels.index("hub32767"))
    assert np.diff(hub["rp"].astype(np.int64)).max() == 32767
    # the pull schedule: node 65534 listed, every real node exactly once, never a real node written as 0xFFFF
    for label in ("max_lu", "max_road"):
        f = graph_fields(blob, labels.index(label))
        listed = f["order"][f["order"] != 0xFFFF]
        assert CC.TOP in listed.tolist() and listed.size == CC.MAX_N, label
        assert int((f["order"] == 0xFFFF).sum()) == f["order"].size - CC.MAX_N, label


def test_chunked_plan_matches_one_shot_at_the_limits(abi):
    """upb_pack_plan_create / _fill (the overlapped upload's path) on the ABI batch, one state per chunk."""
    states, labels, blob = abi
    L = _lib.lib()
    ptrs, keep = _pointer_table(states, blob.n_cap, blob.e_cap)
    plan, nb = C.c_void_p(), C.c_uint64()
    _lib.check(L.upb_pack_plan_create(len(states), ptrs.ctypes.data, blob.n_cap, blob.e_cap, 2, C.byref(plan),
                                      C.byref(nb)))
    try:
        assert nb.value == blob.nbytes
        raw = np.zeros(nb.value + 16, np.uint8)
        off = (-raw.ctypes.data) % 16
        host = raw[off:off + nb.value]
        ranges = np.zeros((9, 2), np.uint64)
        for first in range(len(states)):
            _lib.check(L.upb_pack_plan_fill(plan, ptrs.ctypes.data, first, 1, 2, host.ctypes.data, nb.value,
                                            ranges.ctypes.data))
    finally:
        L.upb_pack_plan_destroy(plan)
    assert np.array_equal(host, host_bytes(blob)[:blob.nbytes])


def call_measure(states, n_cap, e_cap):
    """upb_pack_measure straight through the C ABI (pack_states checks the arrays' padded widths first)."""
    ptrs, keep = _pointer_table(states, *states_caps(states))
    nb = C.c_uint64()
    return _lib.lib().upb_pack_measure(len(states), ptrs.ctypes.data, n_cap, e_cap, 1, C.byref(nb))


def states_caps(states):
    return states[0][1].shape[0], states[0][2].shape[0]


@pytest.mark.parametrize("n_cap,e_cap,ok", [(65535, 32767, True), (65536, 32767, False), (65535, 32768, False),
                                            (0, 10, False), (65535, -1, False)])
def test_packer_caps_refused_past_the_format(n_cap, e_cap, ok):
    """The caps are checked before any state is read, so one small state stands for any."""
    st, _ = CC.abi_case("n32768_lu")
    rc = call_measure([st], n_cap, e_cap)
    if ok:
        assert rc == 0, _lib.lib().upb_last_error()
    else:
        assert rc == -1 and b"caps must satisfy" in _lib.lib().upb_last_error()      # UPB_ERR_ARG


def test_candidate_limits_at_and_past_the_caps():
    """At the limit: a land-use state with 32767 candidates (every edge at e = e_cap) and a road state with 65535 (every
    node at n = n_cap) are packed.  The candidate limit is the caps themselves, so there is no separate count check to
    go past: one more candidate is either a mask on a padded node or edge (refused with UPB_ERR_FORMAT by the action-
    mask checks) or needs caps past the format (refused with UPB_ERR_ARG by the cap check)."""
    lu, _ = CC.abi_case("max_lu")
    rd, _ = CC.abi_case("max_road")
    blob = pack_states([lu, rd], pinned=False)
    assert blob.info[:, 2].tolist() == [CC.MAX_LU_K, CC.MAX_ROAD_K]
    # road: one node fewer -> the 65535th candidate lies on a padded node
    short = [a.copy() for a in rd]
    short[4][CC.TOP] = False
    short[2][short[2] == CC.TOP] = 0                        # keep every real edge on a real node
    with pytest.raises(_lib.UpbError, match="road_mask marks a padded node"):
        pack_states([short], pinned=False)
    # land use: an edge fewer -> the 32767th candidate lies on a padded edge
    fewer = [a.copy() for a in lu]
    fewer[5][CC.MAX_E - 1] = False
    with pytest.raises(_lib.UpbError, match="land_use_mask marks a padded edge"):
        pack_states([fewer], pinned=False)
    # 32768 land-use candidates need e_cap = 32768: refused as a cap
    wide = [a.copy() for a in lu]
    wide[2] = np.concatenate([wide[2], wide[2][-1:]])
    for j in (5, 6):
        wide[j] = np.concatenate([wide[j], [True]])
    wide[2][-1] = [0, 1]
    assert int(wide[6].sum()) == 32768
    with pytest.raises(_lib.UpbError, match="caps must satisfy"):
        pack_states([wide], pinned=False)
