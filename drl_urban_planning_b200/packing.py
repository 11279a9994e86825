"""Host packing of rollout states: reference 9-array layout -> one unpadded blob (csrc/blob.h).

Replaces `tensorfy` (urban_planning/agents/urban_planning_agent.py:16-20) and `SGNNStateEncoder.batch_data`
(urban_planning/models/state_encoder.py:163-177): instead of 9 x B small tensors and nine padded stacks the
update path consumes ONE contiguous buffer per set of states (one H2D copy, ~3.4x fewer bytes than the padded
layout at HLG sizes).  The C packer validates the layout contract and raises on violations.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import _lib

_DTYPES = (np.float32, np.float32, np.int64, np.float32, np.bool_, np.bool_, np.bool_, np.bool_, np.float32)


def _as_numpy(a, want):
    if not isinstance(a, np.ndarray):
        if hasattr(a, "detach"):           # torch tensor (the reference hands tensorfy'd states to the modules)
            a = a.detach().cpu().numpy()
        else:
            a = np.asarray(a)
    if a.dtype != want or not a.flags.c_contiguous:
        a = np.ascontiguousarray(a, dtype=want)
    return a


try:                                   # C helper (csrc/pyptr.c); the pure-Python loop below is the fallback
    from . import _upb_pyptr as _pyptr
except ImportError:                    # pragma: no cover
    _pyptr = None


def _pointer_table(states: Sequence[Sequence], n_cap: int, e_cap: int):
    """Raw pointers of the 9 arrays of every state.  The packer reads n_cap / e_cap elements through them, so the
    element counts are checked here (ValueError) -- a state padded to other widths would be an out-of-bounds read."""
    n = len(states)
    ptrs = np.empty(9 * n, dtype=np.uint64)
    keep = []
    if _pyptr is not None and _pyptr.pointer_table(states, ptrs, int(n_cap), int(e_cap)) < 0:
        return ptrs, keep              # every array was already a C-contiguous buffer of the right item type
    want = (52, n_cap * 23, e_cap * 2, 23, n_cap, e_cap, e_cap, n_cap, 3)
    k = 0
    for i, st in enumerate(states):
        if len(st) != 9:
            raise ValueError("a state must hold 9 arrays (observation_extractor.py:207-228)")
        for j in range(9):
            a = st[j]
            if not (type(a) is np.ndarray and a.dtype == _DTYPES[j] and a.flags.c_contiguous):
                a = _as_numpy(a, _DTYPES[j])
                keep.append(a)
            if (a.size < 2) if j == 8 else (a.size != want[j]):
                raise ValueError(f"state {i}, array {j}: {a.size} elements, expected {want[j]} for the padded widths "
                                 f"n_cap={n_cap}, e_cap={e_cap}")
            ptrs[k] = a.__array_interface__["data"][0]
            k += 1
    return ptrs, keep


def torch_int64():
    import torch
    return torch.int64


def infer_caps(states: Sequence[Sequence]):
    st = states[0]
    return int(np.shape(st[1])[0]), int(np.shape(st[2])[0])


class PackedGraphs:
    """A packed blob in host memory (pinned when torch+CUDA are available) and, after `.to(device)`, on a GPU."""

    def __init__(self, host, nbytes: int, count: int, n_cap: int, e_cap: int):
        self.host = host              # torch uint8 tensor (pinned) or numpy uint8 array
        self.nbytes = nbytes
        self.count = count
        self.n_cap, self.e_cap = n_cap, e_cap
        self.dev = None
        self._info = None

    @property
    def cand_len(self) -> int:
        """Length of the blob's candidate section (the sum of every graph's k, each padded to 4): the size of the
        per-candidate arrays indexed by candidate position (Engine.forward(cand_log_probs=True))."""
        h = self.host.numpy() if hasattr(self.host, "numpy") else self.host
        off = np.frombuffer(h[:128].tobytes(), dtype=np.uint64)          # BlobHeader (csrc/blob.h), 8-byte words
        return int(off[10] - off[9]) // 4                                 # off_cand_idx - off_cand_uv, uint32 entries

    def host_ptr(self) -> int:
        return self.host.data_ptr() if hasattr(self.host, "data_ptr") else self.host.ctypes.data

    @property
    def info(self) -> np.ndarray:
        """(count, 4) int32: n, e, k (action candidates), stage per graph."""
        if self._info is None:
            out = np.zeros((self.count, 4), dtype=np.int32)
            cnt = C.c_int()
            _lib.check(_lib.lib().upb_blob_info(self.host_ptr(), self.nbytes, C.byref(cnt), out.ctypes.data),
                       "upb_blob_info")
            self._info = out
        return self._info

    def to(self, device, non_blocking: bool = True, out=None):
        """Upload with a single H2D copy.  `out` may be a preallocated device uint8 tensor to reuse."""
        import torch
        if not hasattr(self.host, "data_ptr"):
            self.host = torch.from_numpy(self.host)
        if out is None or out.numel() < self.nbytes:
            out = torch.empty(self.nbytes, dtype=torch.uint8, device=device)
        out[:self.nbytes].copy_(self.host[:self.nbytes], non_blocking=non_blocking)
        self.dev = out
        return self

    def dev_ptr(self) -> int:
        if self.dev is None:
            raise RuntimeError("PackedGraphs.to(device) has not been called")
        return self.dev.data_ptr()

    def algorithmic_bytes(self) -> int:
        """SURVEY.md section 8(d): B_alg(n, e) = 1208 n + 42 e + 1300 summed over the graphs (unpadded, fp32)."""
        i = self.info.astype(np.int64)
        return int((1208 * i[:, 0] + 42 * i[:, 1] + 1300).sum())


def pack_states(states: Sequence[Sequence], n_cap: Optional[int] = None, e_cap: Optional[int] = None,
                threads: int = 0, pinned: Optional[bool] = None, out_host=None) -> PackedGraphs:
    """Pack `states` (list of 9-array lists/tuples, numpy or CPU torch) into one blob."""
    if len(states) == 0:
        raise ValueError("pack_states needs at least one state")
    if n_cap is None or e_cap is None:
        n_cap, e_cap = infer_caps(states)
    L = _lib.lib()
    ptrs, keep = _pointer_table(states, n_cap, e_cap)
    if out_host is not None:
        # reuse the caller's (pinned) buffer: fill straight away, the blob header tells how many bytes were used;
        # only a too-small buffer costs the extra measuring pass below
        cap = int(out_host.numel())
        rc = L.upb_pack_fill(len(states), ptrs.ctypes.data, n_cap, e_cap, threads, out_host.data_ptr(), cap)
        if rc == 0:
            nb = int(out_host[16:24].view(torch_int64()).item())          # BlobHeader.total_bytes
            return PackedGraphs(out_host, nb, len(states), n_cap, e_cap)
        if rc != -4:                                                       # anything but UPB_ERR_CAPACITY
            _lib.check(rc, "upb_pack_fill")
    nbytes = C.c_uint64()
    _lib.check(L.upb_pack_measure(len(states), ptrs.ctypes.data, n_cap, e_cap, threads, C.byref(nbytes)),
               "upb_pack_measure")
    nb = int(nbytes.value)
    host = out_host
    if host is None or host.numel() < nb:
        try:
            import torch
            use_pin = torch.cuda.is_available() if pinned is None else pinned
            host = torch.empty(nb, dtype=torch.uint8, pin_memory=bool(use_pin))
        except ImportError:     # pragma: no cover
            host = np.empty(nb, dtype=np.uint8)
    blob = PackedGraphs(host, nb, len(states), n_cap, e_cap)
    _lib.check(L.upb_pack_fill(len(states), ptrs.ctypes.data, n_cap, e_cap, threads, blob.host_ptr(), nb),
               "upb_pack_fill")
    del keep
    return blob


def pack_and_upload(states: Sequence[Sequence], n_cap: int, e_cap: int, device, threads: int = 0, chunk: int = 2048,
                    host=None, dev=None) -> PackedGraphs:
    """Pack a large buffer of states and upload it, overlapped: the blob is filled chunk by chunk (`chunk` states at a
    time, all packer threads on one chunk) and the byte ranges of every finished chunk are copied to the device with
    asynchronous copies from the pinned buffer while the next chunk is being packed.  `host` / `dev` are reusable pinned /
    device uint8 tensors (grown when too small).  Result: the same blob as pack_states(...).to(device)."""
    import torch
    if len(states) == 0:
        raise ValueError("pack_and_upload needs at least one state")
    L = _lib.lib()
    ptrs, keep = _pointer_table(states, n_cap, e_cap)
    plan, nbytes = C.c_void_p(), C.c_uint64()
    _lib.check(L.upb_pack_plan_create(len(states), ptrs.ctypes.data, n_cap, e_cap, threads, C.byref(plan),
                                      C.byref(nbytes)), "upb_pack_plan_create")
    try:
        nb = int(nbytes.value)
        if host is None or host.numel() < nb:
            host = torch.empty(nb, dtype=torch.uint8, pin_memory=True)
        if dev is None or dev.numel() < nb:
            dev = torch.empty(nb, dtype=torch.uint8, device=device)
        ranges = np.zeros((9, 2), np.uint64)
        for first in range(0, len(states), chunk):
            cnt = min(chunk, len(states) - first)
            _lib.check(L.upb_pack_plan_fill(plan, ptrs.ctypes.data, first, cnt, threads, host.data_ptr(), nb,
                                            ranges.ctypes.data), "upb_pack_plan_fill")
            for off, ln in ranges:
                off, ln = int(off), int(ln)
                if ln:
                    dev[off:off + ln].copy_(host[off:off + ln], non_blocking=True)
    finally:
        L.upb_pack_plan_destroy(plan)
    del keep
    blob = PackedGraphs(host, nb, len(states), n_cap, e_cap)
    blob.dev = dev
    return blob
