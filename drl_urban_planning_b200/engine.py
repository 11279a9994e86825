"""Thin Python face of the C ABI: one `Engine` per (process, device).

PyTorch is only the container for device memory and the source of the current CUDA stream; every computation
of the update path happens inside libupb200.so.  Reference call sites mirrored by the methods are cited in
include/upb200.h.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from .packing import PackedGraphs


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _f32(t: torch.Tensor, device) -> torch.Tensor:
    if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return t


def _cpulist(text: str):
    out = []
    for part in text.strip().split(","):
        if not part:
            continue
        a, _, b = part.partition("-")
        out += list(range(int(a), int(b or a) + 1))
    return out


def bind_host_to_gpu_node(device=None):
    """Restrict this process (and the threads it creates later: the packer's workers, the pinned-buffer first touch) to
    the CPUs of the NUMA node the GPU hangs off.  Host glue for the end-to-end path: the packer reads rollout states
    and writes the pinned staging blob, the copy engine reads it; all three want the same node.  Returns
    (node, cpus, nodes_total) or None when the topology cannot be read (then nothing is changed).  Call it before the
    big host allocations; one process per GPU."""
    import glob
    import os
    try:
        idx = torch.cuda.current_device() if device is None else torch.device(device).index or 0
        pr = torch.cuda.get_device_properties(idx)
        bdf = "%04x:%02x:%02x.0" % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read().strip())
        nodes = len(glob.glob("/sys/devices/system/node/node[0-9]*"))
        if node < 0 or nodes < 2:
            return None
        cpus = set(_cpulist(open(f"/sys/devices/system/node/node{node}/cpulist").read()))
        allowed = cpus & set(os.sched_getaffinity(0))
        if len(allowed) < 2:
            return None
        os.sched_setaffinity(0, allowed)
        return node, sorted(allowed), nodes
    except (OSError, ValueError, AttributeError, RuntimeError):
        return None


class Engine:
    def __init__(self, device, n_cap: int, e_cap: int, lr: float = 4e-4, betas=(0.9, 0.999), eps: float = 1e-5,
                 clip_epsilon: float = 0.2, value_pred_coef: float = 0.5, entropy_coef: float = 0.01,
                 clip_mode: int = _lib.CLIP_REFERENCE, grid_limit: int = 0, max_graphs: int = 1 << 20,
                 model: str = "sgnn"):
        if model not in ("sgnn", "mlp"):
            raise ValueError("model must be 'sgnn' (rl-sgnn) or 'mlp' (rl-mlp ablation)")
        # model = "mlp": the reference's rl-mlp ablation (create_mlp_model); every call below then runs the k_mlp kernels
        # on that model's flat layout.  Both models have the fused single-launch step (ppo_step); the in-kernel peer
        # exchange exists for the SGNN only, so a multi-GPU rl-mlp step is upb_mlp_ppo_grad + all-reduce + upb_mlp_apply.
        self.model = model
        self._p = "upb_mlp_" if model == "mlp" else "upb_"
        self.num_params = _lib.UPB_MLP_NUM_PARAMS if model == "mlp" else _lib.UPB_NUM_PARAMS
        self.grad_stride = _lib.UPB_MLP_GRAD_STRIDE if model == "mlp" else _lib.UPB_GRAD_STRIDE
        self.stat_offset = _lib.UPB_MLP_STAT_OFFSET if model == "mlp" else _lib.UPB_STAT_OFFSET
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.UpbError("the update path runs on a CUDA device only (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        cfg = _lib.Config(self.device.index, n_cap, e_cap, max_graphs, lr, betas[0], betas[1], eps,
                          clip_epsilon, value_pred_coef, entropy_coef, clip_mode, grid_limit)
        self.cfg = cfg
        self._ctx = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().upb_create(C.byref(cfg), C.byref(self._ctx)), "upb_create")
        self.n_cap, self.e_cap = n_cap, e_cap
        self.peers, self.peers_ok = 1, False          # multi-GPU fused step: see connect_peers

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            _lib.lib().upb_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _check_blob(self, blob: PackedGraphs):
        if blob.n_cap > self.n_cap or blob.e_cap > self.e_cap:
            raise _lib.UpbError(f"blob caps ({blob.n_cap},{blob.e_cap}) exceed the engine's ({self.n_cap},{self.e_cap})")

    # ------------------------------------------------------------------ no-grad passes
    def forward(self, blob: PackedGraphs, params: torch.Tensor, actions: Optional[torch.Tensor] = None,
                ids: Optional[torch.Tensor] = None, want_greedy: bool = False):
        """value, log_prob, entropy (and greedy action index) per graph of the blob, each shaped (count,).
        Outputs are indexed by blob position; entries not listed in `ids` are left untouched (zero)."""
        self._check_blob(blob)
        n = blob.count
        dev = self.device
        value = torch.zeros(n, dtype=torch.float32, device=dev)
        logp = torch.zeros(n, dtype=torch.float32, device=dev)
        ent = torch.zeros(n, dtype=torch.float32, device=dev)
        greedy = torch.zeros(n, dtype=torch.int32, device=dev) if want_greedy else None
        if actions is not None:
            actions = _f32(actions, dev)
            assert actions.numel() == 2 * n, "actions must be (count, 2) like the reference's"
        cnt = n if ids is None else int(ids.numel())
        assert params.numel() == self.num_params, "flat parameter vector of the wrong model"
        _lib.check(getattr(_lib.lib(), self._p + "forward")(self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(),
                                                           _ptr(actions), value.data_ptr(), logp.data_ptr(),
                                                           ent.data_ptr(), _ptr(greedy), self._stream()),
                   self._p + "forward")
        return (value, logp, ent, greedy) if want_greedy else (value, logp, ent)

    # ------------------------------------------------------------------ training step pieces
    def new_grad_buffer(self) -> torch.Tensor:
        return torch.zeros(self.grad_stride, dtype=torch.float32, device=self.device)

    def ppo_grad(self, blob: PackedGraphs, params: torch.Tensor, actions: torch.Tensor, advantages: torch.Tensor,
                 returns: torch.Tensor, fixed_log_probs: torch.Tensor, exps: torch.Tensor, inv_batch: float,
                 inv_ind: float, ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None
                 ) -> torch.Tensor:
        """Gradient of the PPO loss of the graphs `ids` (all if None) w.r.t. the flat parameters, plus the loss
        statistics, in one flat buffer (see upb200.h).  Per-sample arrays are indexed by blob position."""
        self._check_blob(blob)
        dev = self.device
        if out is None:
            out = self.new_grad_buffer()
        cnt = blob.count if ids is None else int(ids.numel())
        _lib.check(getattr(_lib.lib(), self._p + "ppo_grad")(
            self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(), _f32(actions, dev).data_ptr(),
            _f32(advantages, dev).data_ptr(), _f32(returns, dev).data_ptr(), _f32(fixed_log_probs, dev).data_ptr(),
            _f32(exps, dev).data_ptr(), float(inv_batch), float(inv_ind), out.data_ptr(), self._stream()),
            self._p + "ppo_grad")
        return out

    def ppo_step(self, blob: PackedGraphs, params: torch.Tensor, actions: torch.Tensor, advantages: torch.Tensor,
                 returns: torch.Tensor, fixed_log_probs: torch.Tensor, exps: torch.Tensor, inv_batch: float,
                 inv_ind: float, ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None
                 ) -> torch.Tensor:
        """Single-GPU optimiser step in one launch (gradient + reduction + Adam, upb_ppo_step / upb_mlp_ppo_step);
        falls back to ppo_grad + apply inside the library on steps that clip.  Returns the gradient / statistics
        buffer."""
        self._check_blob(blob)
        dev = self.device
        if out is None:
            out = self.new_grad_buffer()
        cnt = blob.count if ids is None else int(ids.numel())
        _lib.check(getattr(_lib.lib(), self._p + "ppo_step")(
            self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(), _f32(actions, dev).data_ptr(),
            _f32(advantages, dev).data_ptr(), _f32(returns, dev).data_ptr(), _f32(fixed_log_probs, dev).data_ptr(),
            _f32(exps, dev).data_ptr(), float(inv_batch), float(inv_ind), out.data_ptr(), self._stream()),
            self._p + "ppo_step")
        return out

    def select_action(self, blob: PackedGraphs, params: torch.Tensor, uniforms: Optional[torch.Tensor] = None,
                      ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Action index per graph of the blob (int32, indexed by blob position): greedy arg-max when `uniforms` is
        None (policy.py:72-79 `mean_action`), else drawn by inverse CDF from one uniform per graph (policy.py:81-83)."""
        self._check_blob(blob)
        out = torch.zeros(blob.count, dtype=torch.int32, device=self.device)
        cnt = blob.count if ids is None else int(ids.numel())
        u = None
        if uniforms is not None:
            u = _f32(uniforms, self.device).reshape(-1)
            if u.numel() != blob.count:
                raise ValueError("uniforms must hold one value per graph of the blob")
        _lib.check(getattr(_lib.lib(), self._p + "select_action")(
            self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(), None if u is None else u.data_ptr(),
            out.data_ptr(), self._stream()), self._p + "select_action")
        return out

    # ---- multi-GPU fused step (include/upb200.h: upb_peer_*) -----------------------------------------------------
    def peer_export(self) -> bytes:
        buf = C.create_string_buffer(_lib.UPB_PEER_HANDLE_BYTES)
        _lib.check(_lib.lib().upb_peer_export(self._ctx, buf), "upb_peer_export")
        return buf.raw

    def peer_connect(self, world: int, rank: int, handles: bytes) -> None:
        assert len(handles) == world * _lib.UPB_PEER_HANDLE_BYTES
        _lib.check(_lib.lib().upb_peer_connect(self._ctx, int(world), int(rank), C.c_char_p(handles)), "upb_peer_connect")
        self.peers = world

    def peer_timeouts(self) -> int:
        """CTAs that ever gave up waiting for a peer inside a fused step (sticky; non-zero = ranks out of sync)."""
        n = C.c_int64()
        _lib.check(_lib.lib().upb_peer_timeouts(self._ctx, C.byref(n)), "upb_peer_timeouts")
        return int(n.value)

    def next_step_fused(self) -> bool:
        """True if the next ppo_step runs as one launch (it does not clip)."""
        return bool(getattr(_lib.lib(), self._p + "next_step_fused")(self._ctx))

    def connect_peers(self, process_group=None) -> bool:
        """Exchange the ranks' IPC handles over `process_group` (NCCL) and map the peers' exchange buffers.  Collective;
        returns True on every rank or False on every rank (then the NCCL all-reduce path stays in use)."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(process_group), dist.get_rank(process_group)
        if self.model != "sgnn":
            return False
        if world < 2 or getattr(self, "peers", 1) > 1:
            return getattr(self, "peers", 1) > 1
        ok = torch.ones(1, dtype=torch.int32, device=self.device)
        try:
            mine = torch.frombuffer(bytearray(self.peer_export()), dtype=torch.uint8).to(self.device)
        except _lib.UpbError:
            mine = torch.zeros(_lib.UPB_PEER_HANDLE_BYTES, dtype=torch.uint8, device=self.device)
            ok.zero_()
        everyone = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(everyone, mine, group=process_group)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=process_group)
        if int(ok.item()) == 1:
            try:
                self.peer_connect(world, rank, b"".join(bytes(t.cpu().numpy().tobytes()) for t in everyone))
            except _lib.UpbError:
                ok.zero_()
        # a rank that failed to map a peer must not leave the others waiting for it inside a kernel
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=process_group)
        self.peers_ok = int(ok.item()) == 1
        return self.peers_ok

    def apply(self, params: torch.Tensor, grad: torch.Tensor) -> None:
        _lib.check(getattr(_lib.lib(), self._p + "apply")(self._ctx, params.data_ptr(), grad.data_ptr(), self._stream()),
                   self._p + "apply")

    def read_losses(self, grad: torch.Tensor) -> Tuple[float, float, float, float]:
        out = (C.c_float * 4)()
        _lib.check(getattr(_lib.lib(), self._p + "read_losses")(self._ctx, grad.data_ptr(), out, self._stream()),
                   self._p + "read_losses")
        return tuple(float(x) for x in out)

    def gae(self, rewards: torch.Tensor, masks: torch.Tensor, values: torch.Tensor, gamma: float, tau: float):
        dev = self.device
        r, m, v = _f32(rewards.reshape(-1), dev), _f32(masks.reshape(-1), dev), _f32(values.reshape(-1), dev)
        T = r.numel()
        adv = torch.empty(T, dtype=torch.float32, device=dev)
        ret = torch.empty(T, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().upb_gae(self._ctx, r.data_ptr(), m.data_ptr(), v.data_ptr(), T, float(gamma),
                                      float(tau), adv.data_ptr(), ret.data_ptr(), self._stream()), "upb_gae")
        return adv, ret

    # ------------------------------------------------------------------ optimiser state
    def get_opt_state(self):
        m = np.zeros(self.num_params, np.float32)
        v = np.zeros(self.num_params, np.float32)
        steps = np.zeros(4, np.int64)
        _lib.check(getattr(_lib.lib(), self._p + "get_opt_state")(self._ctx, m.ctypes.data, v.ctypes.data,
                                                                 steps.ctypes.data), self._p + "get_opt_state")
        return m, v, steps

    def set_opt_state(self, m: np.ndarray, v: np.ndarray, steps: np.ndarray, rearm_first_step_clip: bool = False
                      ) -> None:
        m = np.ascontiguousarray(m, np.float32)
        v = np.ascontiguousarray(v, np.float32)
        steps = np.ascontiguousarray(steps, np.int64)
        assert m.size == self.num_params and v.size == self.num_params
        _lib.check(getattr(_lib.lib(), self._p + "set_opt_state")(self._ctx, m.ctypes.data, v.ctypes.data,
                                                                 steps.ctypes.data), self._p + "set_opt_state")
        if rearm_first_step_clip:
            _lib.check(getattr(_lib.lib(), self._p + "rearm_clip")(self._ctx), self._p + "rearm_clip")

    def profile(self, enable: bool) -> None:
        _lib.check(_lib.lib().upb_profile_enable(self._ctx, int(enable)), "upb_profile_enable")

    def profile_read(self):
        """(summed ms of the bracketed fused-kernel launches, number of launches) since the last read."""
        ms, n = C.c_double(), C.c_int()
        _lib.check(_lib.lib().upb_profile_read(self._ctx, C.byref(ms), C.byref(n)), "upb_profile_read")
        return float(ms.value), int(n.value)

    @property
    def grid(self) -> int:
        return int(_lib.lib().upb_grid_size(self._ctx))

    @staticmethod
    def graph_cost(info: np.ndarray) -> np.ndarray:
        """Estimated cycles of one graph in the fused training kernel from (n, e, k, stage) rows
        (least-squares fit of the per-CTA busy cycles, tools/balance_check.py: pulls ~ 17 / edge, node phases ~ 80 /
        node, policy head ~ 134 / candidate, and ~ 41 k cycles per graph that do not depend on its size)."""
        i = np.asarray(info, dtype=np.int64)
        return 17 * i[:, 1] + 80 * i[:, 0] + 134 * i[:, 2] + 41500

    def balance_ids(self, ids: np.ndarray, cost: np.ndarray) -> np.ndarray:
        """Order graph ids for the kernel's static schedule (ids[i] -> CTA i % grid, round i // grid).
        Longest-processing-time-first: graphs in descending cost go to the least loaded CTA; CTAs are then numbered by
        how many graphs they hold (round r must cover CTAs 0..len_r-1), so e.g. with 256 graphs on 132 SMs the 8
        largest graphs run alone and the other 248 are paired long + short."""
        import heapq
        ids = np.asarray(ids)
        g = self.grid
        if len(ids) <= g:
            return ids[np.argsort(-np.asarray(cost)[ids], kind="stable")]
        c = np.asarray(cost, dtype=np.float64)[ids]
        order = np.argsort(-c, kind="stable")
        m = len(ids)
        if m <= 2 * g and c[order[0]] < c[order[g - 1]] + c[order[-1]]:
            # closed form of the loop below for one partial second round (the usual 256 graphs on 132 CTAs): no single
            # graph outweighs a pair, so LPT pairs the (g - j)-th largest with the (g + j)-th largest; pairs first
            srt = ids[order]
            npair = m - g
            return np.concatenate([srt[g - npair:g], srt[:g - npair], srt[m - 1:g - 1:-1] if npair else srt[:0]])
        bins = [[] for _ in range(g)]
        heap = [(0.0, b) for b in range(g)]
        for k in order:
            load, b = heapq.heappop(heap)
            bins[b].append(int(ids[k]))
            heapq.heappush(heap, (load + float(c[k]), b))
        bins.sort(key=lambda x: -len(x))
        out = []
        for r in range(len(bins[0])):
            row = [b[r] for b in bins if len(b) > r]
            out.extend(row)
        return np.asarray(out, dtype=ids.dtype)

    def set_stamp_buffer(self, buf: Optional[torch.Tensor]) -> None:
        """int64[64] device tensor receiving clock64() phase stamps (debug), or None."""
        _lib.check(_lib.lib().upb_set_stamp_buffer(self._ctx, _ptr(buf)), "upb_set_stamp_buffer")

    @property
    def launches(self) -> int:
        return int(_lib.lib().upb_launch_count(self._ctx))
