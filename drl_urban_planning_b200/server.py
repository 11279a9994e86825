"""Batched GPU policy inference for the forked rollout workers (SURVEY.md section 8(f)-2).

The reference samples trajectories in `num_threads` forked processes, each calling
`policy_net.select_action(tensorfy([state]), use_mean_action)` with B = 1 on the CPU
(urban_planning/agents/urban_planning_agent.py:49-91, khrylib/rl/agents/agent.py:75-100).  This module keeps the
geometry environment in those CPU workers and moves only the policy call: every worker writes its state into its own
shared-memory slab and posts its id; a server thread in the parent process (the owner of the CUDA context) collects
the requests that are pending, packs them into one blob and runs ONE `upb_select_action` launch for the batch, then
hands every worker its action index.

    server = InferenceServer.for_engine(engine, params, n_cap, e_cap, num_workers)   # parent, before forking
    server.start()
    ... fork workers; in worker w:   policy = server.client(w)
                                      action = policy.select_action([state], mean_action)      # (1, 2) float32 tensor
    server.stop()

`client(w).select_action` has the call signature of `UrbanPlanningPolicy.select_action` for a single state (numpy or
torch arrays), so `sample_worker` runs unchanged with `self.policy_net = server.client(pid)`.  Greedy actions are
bit-identical to the reference's `probs.argmax`; sampled actions are drawn by inverse CDF from a uniform the WORKER
draws from its own numpy generator (seeded per worker like `seed_worker`, agent.py:67-70), so rollouts are reproducible
per worker seed but not bit-equal to torch's `Categorical.sample` stream.

No CUDA call is ever made in a worker (fork-safe): workers touch only the shared slabs, a multiprocessing queue and
their own semaphore.  The batching core is independent of CUDA (`infer_fn`), which is how the CPU tests drive it.
"""
from __future__ import annotations

import multiprocessing as mp
import threading
import time
from typing import Callable, List, Optional, Sequence

import numpy as np

_DTYPES = (np.float32, np.float32, np.int64, np.float32, np.bool_, np.bool_, np.bool_, np.bool_, np.float32)
_BELOW_ONE = np.nextafter(np.float32(1), np.float32(0))     # the largest float32 uniform, 1 - 2^-24


def _shapes(n_cap: int, e_cap: int):
    return ((52,), (n_cap, 23), (e_cap, 2), (23,), (n_cap,), (e_cap,), (e_cap,), (n_cap,), (3,))


class _Slab:
    """One worker's shared-memory state (the 9 arrays of the reference layout, observation_extractor.py:207-228), a
    request header and the reply."""

    def __init__(self, ctx, n_cap: int, e_cap: int):
        self.shapes = _shapes(n_cap, e_cap)
        self.bufs = [ctx.RawArray("b", int(np.prod(s)) * np.dtype(d).itemsize) for s, d in zip(self.shapes, _DTYPES)]
        self.head = ctx.RawArray("d", 4)          # [0] mean_action flag, [1] uniform, [2] reply action index, [3] error flag
        self.done = ctx.Semaphore(0)

    def arrays(self) -> List[np.ndarray]:
        return [np.frombuffer(b, dtype=d).reshape(s) for b, s, d in zip(self.bufs, self.shapes, _DTYPES)]


class InferenceClient:
    """The worker-side stand-in for `policy_net` (select_action only)."""

    def __init__(self, slab: _Slab, wid: int, requests, dtype=None):
        self._slab, self._wid, self._req = slab, wid, requests
        self._views = None
        self._rng = None
        self.dtype = dtype

    def seed(self, seed: int) -> None:
        self._rng = np.random.default_rng(seed)

    def select_action(self, x, mean_action=False):
        """x: a list holding ONE state (9 arrays, numpy or CPU torch).  Returns a (1, 2) float32 torch tensor with the
        chosen land-use edge index in column 0 or road node index in column 1 (policy.py:67-85)."""
        import torch
        if len(x) != 1:
            raise ValueError("the rollout workers call select_action with one state at a time (agent.py:75-100)")
        if self._views is None:
            self._views = self._slab.arrays()
        if self._rng is None:
            self._rng = np.random.default_rng(np.random.randint(1 << 31))      # after seed_worker's np.random.seed
        st = x[0]
        for dst, src in zip(self._views, st):
            a = src.detach().cpu().numpy() if hasattr(src, "detach") else np.asarray(src)
            if a.size != dst.size:
                raise ValueError(f"state array of {a.size} elements does not match the server's padded widths {dst.shape}")
            np.copyto(dst, a.reshape(dst.shape), casting="unsafe")
        stage = self._views[8]
        h = self._slab.head
        h[0] = 1.0 if mean_action else 0.0
        h[1] = float(self._rng.random())
        self._req.put(self._wid)
        self._slab.done.acquire()
        if h[3] != 0.0:
            raise RuntimeError("inference server failed while serving this request (see the parent's log)")
        out = torch.zeros(1, 2, dtype=torch.float32)
        out[0, int(np.argmax(stage[:2]))] = float(h[2])
        return out


class InferenceServer:
    """Collects the workers' pending requests and serves them in batches through `infer_fn`.

    infer_fn(states, uniforms) -> int array: `states` is a list of 9-array states (numpy views of the slabs),
    `uniforms` a float32 array with one value per state, NaN meaning "greedy"; returns the action index per state.
    """

    def __init__(self, infer_fn: Callable[[Sequence, np.ndarray], np.ndarray], n_cap: int, e_cap: int,
                 num_workers: int, max_wait_s: float = 2e-4, ctx=None):
        self._ctx = ctx or mp.get_context("fork")
        self._infer = infer_fn
        self.n_cap, self.e_cap, self.num_workers = n_cap, e_cap, num_workers
        self._slabs = [_Slab(self._ctx, n_cap, e_cap) for _ in range(num_workers)]
        self._requests = self._ctx.Queue()
        self._views = [s.arrays() for s in self._slabs]
        self._thread: Optional[threading.Thread] = None
        self._stop = False
        self.max_wait_s = max_wait_s
        self.batches: List[int] = []              # served batch sizes (diagnostics)
        self.error: Optional[BaseException] = None

    # ---- construction from the CUDA engine
    @classmethod
    def for_engine(cls, engine, params, n_cap: int, e_cap: int, num_workers: int, **kw):
        """`params` is the flat device parameter tensor (e.g. PPOUpdater.params): it is read at every batch, so the server
        always serves the current weights."""
        import torch
        from .packing import pack_states
        host_buf = {}

        def infer(states, uniforms):
            blob = pack_states(states, n_cap, e_cap, threads=1, out_host=host_buf.get("h"))
            host_buf["h"] = blob.host if hasattr(blob.host, "data_ptr") else None
            blob.to(engine.device, out=host_buf.get("d"))
            host_buf["d"] = blob.dev
            greedy = np.isnan(uniforms)
            out = np.zeros(len(states), np.int64)
            if greedy.any():
                ids = torch.as_tensor(np.flatnonzero(greedy).astype(np.int32), device=engine.device)
                out[greedy] = engine.select_action(blob, params, ids=ids).cpu().numpy()[greedy]
            if (~greedy).any():
                ids = torch.as_tensor(np.flatnonzero(~greedy).astype(np.int32), device=engine.device)
                u = torch.as_tensor(np.nan_to_num(uniforms, nan=0.0).astype(np.float32), device=engine.device)
                out[~greedy] = engine.select_action(blob, params, uniforms=u, ids=ids).cpu().numpy()[~greedy]
            return out
        return cls(infer, n_cap, e_cap, num_workers, **kw)

    # ---- lifecycle
    def client(self, wid: int) -> InferenceClient:
        return InferenceClient(self._slabs[wid], wid, self._requests)

    def start(self) -> "InferenceServer":
        self._stop = False
        self._thread = threading.Thread(target=self._loop, name="upb-inference-server", daemon=True)
        self._thread.start()
        return self

    def stop(self) -> None:
        self._stop = True
        self._requests.put(-1)
        if self._thread is not None:
            self._thread.join(timeout=10)
            self._thread = None

    def __enter__(self):
        return self.start()

    def __exit__(self, *exc):
        self.stop()

    # ---- the batching loop
    def _loop(self) -> None:
        import queue as _q
        while not self._stop:
            first = self._requests.get()
            if first < 0:
                break
            wids = [first]
            deadline = time.perf_counter() + self.max_wait_s
            # take everything that is already pending, then wait a moment for stragglers (workers run in lock step
            # through similar environments, so their requests arrive in bursts)
            while len(wids) < self.num_workers:
                try:
                    w = self._requests.get_nowait()
                except _q.Empty:
                    if time.perf_counter() >= deadline:
                        break
                    time.sleep(2e-5)
                    continue
                if w < 0:
                    self._stop = True
                    break
                wids.append(w)
            self._serve(wids)

    def _serve(self, wids: List[int]) -> None:
        states = [self._views[w] for w in wids]
        uniforms = np.array([np.nan if self._slabs[w].head[0] != 0.0 else self._slabs[w].head[1] for w in wids],
                            np.float32)
        # the workers draw in float64: every draw in [1 - 2^-25, 1) rounds to exactly 1.0f, outside the [0, 1) that
        # select_action takes; keep it below 1 (NaN, the greedy flag, passes through np.minimum)
        uniforms = np.minimum(uniforms, _BELOW_ONE)
        try:
            actions = np.asarray(self._infer(states, uniforms)).reshape(-1)
            err = 0.0
        except BaseException as e:       # never leave a worker blocked
            self.error = e
            actions = np.zeros(len(wids))
            err = 1.0
        self.batches.append(len(wids))
        for w, a in zip(wids, actions):
            h = self._slabs[w].head
            h[2] = float(a)
            h[3] = err
            self._slabs[w].done.release()
