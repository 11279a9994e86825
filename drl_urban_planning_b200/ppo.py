"""PPO update of one training iteration on the H100 path.

Mirrors `UrbanPlanningAgent.update_params` / `update_policy` (reference
urban_planning/agents/urban_planning_agent.py:248-361) with the same observable behaviour -- values pass, GAE,
fixed log-probs, `num_optim_epoch` x floor(T/B) minibatch steps on np.random.shuffle permutations, four loss
scalars per minibatch -- but a different data path:

  * the rollout states are packed ONCE per iteration into an unpadded blob and uploaded with one copy
    (the reference re-tensorfies every state for each of the 2 + epochs sweeps);
  * a minibatch is an int32 index list into the resident blob, so a step moves ~1 KB H2D;
  * one encoder pass yields value, log-prob and entropy (the reference runs the encoder twice per step);
  * loss scalars stay on the device and are read back once per epoch (the reference syncs 4x per step).

Data parallel: every rank holds the whole buffer and takes `order[i*B:(i+1)*B][rank::world]` of each global
minibatch, where `order` is RANK 0's permutation broadcast once per epoch (the ranks' np.random streams need not
agree) and `load_states` checks that all ranks hold the same buffer; 1/B and 1/|ind| are global, so the summed shard
gradients equal the single-GPU batch gradient (SURVEY.md section 8(e)).  The per-rank 58 KB column sums are exchanged inside the step kernel through peer memory (NVLink, no NCCL call,
one launch per step); steps that clip gradients, and process groups without peer access, all-reduce one 55 KB
gradient+statistics buffer with NCCL instead.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .engine import Engine
from .packing import PackedGraphs, pack_and_upload, pack_states, infer_caps


class PPOUpdater:
    def __init__(self, flat_params, n_cap: int, e_cap: int, device, lr: float = 4e-4, eps: float = 1e-5,
                 clip_epsilon: float = 0.2, value_pred_coef: float = 0.5, entropy_coef: float = 0.01,
                 gamma: float = 1.0, tau: float = 0.0, opt_num_epochs: int = 4, mini_batch_size: int = 256,
                 clip_mode: int = _lib.CLIP_REFERENCE, process_group="auto", pack_threads: int = 0,
                 use_peers: bool = True, batch_stage: bool = False, model: str = "sgnn"):
        self.device = torch.device(device)
        self.engine = Engine(self.device, n_cap, e_cap, lr=lr, eps=eps, clip_epsilon=clip_epsilon,
                             value_pred_coef=value_pred_coef, entropy_coef=entropy_coef, clip_mode=clip_mode,
                             model=model)
        self.device = self.engine.device
        if isinstance(flat_params, torch.Tensor):
            self.params = flat_params.detach().to(self.device, torch.float32).contiguous().clone()
        else:
            self.params = torch.as_tensor(np.asarray(flat_params, np.float32), device=self.device).clone()
        assert self.params.numel() == self.engine.num_params
        self.gamma, self.tau = gamma, tau
        self.opt_num_epochs, self.mini_batch_size = opt_num_epochs, mini_batch_size
        self.value_pred_coef, self.entropy_coef = value_pred_coef, entropy_coef
        self.pack_threads = pack_threads
        self.batch_stage = bool(batch_stage)            # agent_specs.batch_stage (urban_planning_agent.py:314-319)
        # process_group: "auto" = the default group if torch.distributed is initialised, None = single process,
        # or an explicit group
        self.world, self.rank = 1, 0
        dist_up = torch.distributed.is_available() and torch.distributed.is_initialized()
        if process_group == "auto":
            process_group = None
            use_dist = dist_up
        else:
            use_dist = process_group is not None
            if not use_dist and dist_up and torch.distributed.get_world_size() > 1:
                import warnings
                warnings.warn("PPOUpdater(process_group=None) runs single-process although torch.distributed is "
                              "initialised with world_size > 1: every rank will update independently and the ranks "
                              "diverge.  Pass process_group='auto' (or a group) for data-parallel updates.",
                              RuntimeWarning, stacklevel=2)
        self.pg = process_group
        if use_dist:
            import torch.distributed as dist
            self.world = dist.get_world_size(process_group)
            self.rank = dist.get_rank(process_group)
        self.grad = self.engine.new_grad_buffer()
        # ranks on one node exchange gradients inside the step kernel (peer memory over NVLink) when the process group
        # is NCCL and the peers' buffers can be mapped; otherwise one NCCL all-reduce per step
        self.fused_exchange = False
        if use_dist and use_peers and self.world > 1:
            import torch.distributed as dist
            if dist.get_backend(process_group) == "nccl":
                self.fused_exchange = self.engine.connect_peers(process_group)
        self.blob: Optional[PackedGraphs] = None
        self._dev_blob_buf = None
        self.loss_iter = 0

    # ------------------------------------------------------------------ buffer
    def load_states(self, states: Sequence, actions, exps=None):
        """Pack + upload the iteration's rollout states (list of reference 9-array states) and their actions."""
        nvtx = torch.cuda.nvtx
        nvtx.range_push("upb.pack_and_upload")
        # chunked: the H2D copies of a packed chunk run while the next chunk is being packed
        self.blob = pack_and_upload(states, self.engine.n_cap, self.engine.e_cap, self.device, threads=self.pack_threads,
                                    host=getattr(self, "_host_blob_buf", None), dev=self._dev_blob_buf)
        self._host_blob_buf = self.blob.host
        nvtx.range_pop()
        self._dev_blob_buf = self.blob.dev
        T = self.blob.count
        self.actions = torch.as_tensor(np.ascontiguousarray(actions, np.float32)).reshape(T, 2).to(self.device)
        e = np.ones(T, np.float32) if exps is None else np.ascontiguousarray(exps, np.float32).reshape(T)
        self.exps_host = e
        self.exps = torch.as_tensor(e).to(self.device)
        info = self.blob.info.astype(np.int64)
        self._cost = Engine.graph_cost(info)
        self._stage = info[:, 3].copy()
        self._check_same_buffer(info)
        return self.blob

    def _check_same_buffer(self, info: np.ndarray) -> None:
        """Data-parallel ranks must hold the SAME rollout buffer (the shards are index ranges into it)."""
        if self.world <= 1:
            return
        import zlib
        import torch.distributed as dist
        sig = [int(info.shape[0]), zlib.crc32(np.ascontiguousarray(info).tobytes()),
               zlib.crc32(np.ascontiguousarray(self.exps_host).tobytes()),
               zlib.crc32(self.actions.cpu().numpy().tobytes())]
        on = self.device if dist.get_backend(self.pg) == "nccl" else torch.device("cpu")
        lo = torch.tensor(sig, dtype=torch.int64, device=on)
        hi = lo.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=self.pg)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=self.pg)
        if not torch.equal(lo, hi):
            raise _lib.UpbError("data-parallel ranks hold different rollout buffers (count / graph sizes / exps / "
                                "actions differ): every rank must load the same states")

    def _epoch_order(self, order: np.ndarray) -> np.ndarray:
        """Next epoch's sample order, composed like the reference: it re-permutes the ALREADY permuted lists every
        epoch (urban_planning_agent.py:306-312 reassigns `states = index_select_list(states, perm_np)`), so epoch k
        walks perm_1 o ... o perm_k; then the optional stage grouping (:314-319).  Every rank draws from np.random
        (keeps the streams aligned when they are seeded alike) but rank 0's order is the one used."""
        T = order.shape[0]
        perm = np.arange(T)
        np.random.shuffle(perm)                                                        # :306-307
        order = order[perm]
        if self.batch_stage:                                                           # get_perm_batch_stage :273-279
            st = self._stage[order]
            order = np.concatenate([order[st == 0], order[st != 0]])
        if self.world > 1:
            import torch.distributed as dist
            on = self.device if dist.get_backend(self.pg) == "nccl" else torch.device("cpu")
            t = torch.as_tensor(order.astype(np.int64), device=on)
            dist.broadcast(t, src=dist.get_global_rank(self.pg, 0) if self.pg is not None else 0, group=self.pg)
            order = t.cpu().numpy()
        return order

    # ------------------------------------------------------------------ pieces of update_params
    def forward_all(self):
        """value, log_prob, entropy of every state in the buffer (reference :256-264 and :283-292, one pass)."""
        return self.engine.forward(self.blob, self.params, self.actions)

    def allreduce(self, buf: torch.Tensor):
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.pg)

    def minibatch_step(self, ids: torch.Tensor, global_batch: int, global_ind: int):
        """One optimiser step on the graphs `ids` (this rank's shard of a global minibatch of `global_batch`
        graphs, `global_ind` of which have exps != 0): urban_planning_agent.py:322-337."""
        args = (self.blob, self.params, self.actions, self.advantages, self.returns, self.fixed_log_probs, self.exps,
                1.0 / max(global_batch, 1), 1.0 / max(global_ind, 1))
        if self.world == 1 or (self.fused_exchange and self.engine.next_step_fused()):
            # one launch: gradient, reduction (over the SGNN ranks too, through peer memory), Adam.  rl-mlp ranks never
            # have fused_exchange (Engine.connect_peers) and keep the NCCL path below
            self.engine.ppo_step(*args, ids=ids, out=self.grad)
        else:
            self.engine.ppo_grad(*args, ids=ids, out=self.grad)
            self.allreduce(self.grad)
            self.engine.apply(self.params, self.grad)

    # ------------------------------------------------------------------ the reference's update_params
    def update_params(self, states: Sequence, actions, rewards, masks, exps=None,
                      log_fn: Optional[Callable[[str, float, int], None]] = None, iteration: int = 0):
        """Full update of one iteration.  Returns dict of mean losses per epoch (the reference's 'total_*')."""
        self.load_states(states, actions, exps)
        T = self.blob.count
        dev = self.device
        # one no-grad sweep yields both pre-pass results of the reference: values (:256-264) and the fixed
        # log-probs (:283-292); neither depends on the other
        values, self.fixed_log_probs, _ = self.forward_all()
        rewards_t = torch.as_tensor(np.ascontiguousarray(rewards, np.float32)).reshape(T).to(dev)
        masks_t = torch.as_tensor(np.ascontiguousarray(masks, np.float32)).reshape(T).to(dev)
        self.advantages, self.returns = self.engine.gae(rewards_t, masks_t, values, self.gamma, self.tau)  # :267
        return self.update_policy(iteration, log_fn)

    def update_policy(self, iteration: int = 0, log_fn=None):
        T, B = self.blob.count, self.mini_batch_size
        nb = int(math.floor(T / B))
        # one gradient / statistics row per minibatch of the epoch: the step kernels write their loss statistics
        # straight into their own row (no per-step device copy), read back once per epoch
        ring = getattr(self, "_grad_ring", None)
        if ring is None or ring.shape[0] < max(nb, 1):
            ring = torch.zeros(max(nb, 1), self.engine.grad_stride, dtype=torch.float32, device=self.device)
            self._grad_ring = ring
        totals = np.zeros(4)

        def prepare(order):
            """Host side of one epoch: the sample order, this rank's shard of every minibatch in the order of the
            kernel's static CTA schedule (long + short graph per CTA), one upload."""
            order = self._epoch_order(order)
            shards = [self.engine.balance_ids(order[i * B:(i + 1) * B][self.rank::self.world], self._cost)
                      for i in range(nb)]
            width = max((len(x) for x in shards), default=0)
            ids_host = np.zeros((max(nb, 1), max(width, 1)), np.int32)
            for i, x in enumerate(shards):
                ids_host[i, :len(x)] = x
            n_ind = [int((self.exps_host[order[i * B:(i + 1) * B]] != 0).sum()) for i in range(nb)]
            return order, [len(x) for x in shards], torch.as_tensor(ids_host).to(self.device, non_blocking=True), n_ind

        cur = prepare(np.arange(T))
        for epoch in range(self.opt_num_epochs):
            torch.cuda.nvtx.range_push(f"upb.epoch{epoch}")
            order, lens, ids_dev, n_inds = cur
            for i in range(nb):
                self.grad = ring[i]
                self.minibatch_step(ids_dev[i, :lens[i]], min((i + 1) * B, T) - i * B, n_inds[i])
            # the next epoch's host work overlaps this epoch's kernels (one process; with several ranks the order is
            # broadcast on the stream, which would wait for them)
            if epoch + 1 < self.opt_num_epochs and self.world == 1:
                cur = prepare(order)
            so = self.engine.stat_offset
            stats_all = ring[:nb, so:so + 16]
            st = stats_all.cpu().numpy().astype(np.float64)                            # one sync per epoch
            nB, nI = np.maximum(st[:, 3], 1), np.maximum(st[:, 4], 1)
            vl, sl_, el = st[:, 0] / nB, st[:, 1] / nI, st[:, 2] / nI
            loss = sl_ + self.value_pred_coef * vl + self.entropy_coef * el
            if self.fused_exchange and self.engine.peer_timeouts():
                raise _lib.UpbError("multi-GPU step: a peer rank never published its gradient sums (timed out inside "
                                    "the step kernel); that step's Adam update was skipped on this rank -- the ranks "
                                    "are out of sync, restore the last checkpoint")
            if nb and st[:, 7].any():
                raise FloatingPointError("non-finite value / log-prob / entropy in the PPO update")
            if log_fn is not None:
                for i in range(nb):
                    log_fn("loss/loss", float(loss[i]), self.loss_iter + i)
                    log_fn("loss/value_loss", float(vl[i]), self.loss_iter + i)
                    log_fn("loss/surr_loss", float(sl_[i]), self.loss_iter + i)
                    log_fn("loss/entropy_loss", float(el[i]), self.loss_iter + i)
                ge = iteration * self.opt_num_epochs + epoch
                log_fn("loss/epoch_loss", float(loss.sum()), ge)
                log_fn("loss/epoch_value_loss", float(vl.sum()), ge)
                log_fn("loss/epoch_surr_loss", float(sl_.sum()), ge)
                log_fn("loss/epoch_entropy_loss", float(el.sum()), ge)
            self.loss_iter += nb
            totals += [loss.sum(), vl.sum(), sl_.sum(), el.sum()]
            torch.cuda.nvtx.range_pop()
            if epoch + 1 < self.opt_num_epochs and self.world > 1:
                cur = prepare(order)
        totals /= max(self.opt_num_epochs, 1)
        if log_fn is not None:
            log_fn("loss/total_loss", float(totals[0]), iteration)
            log_fn("loss/total_value_loss", float(totals[1]), iteration)
            log_fn("loss/total_surr_loss", float(totals[2]), iteration)
            log_fn("loss/total_entropy_loss", float(totals[3]), iteration)
        return dict(total_loss=totals[0], total_value_loss=totals[1], total_surr_loss=totals[2],
                    total_entropy_loss=totals[3])

    def flat_params(self) -> np.ndarray:
        return self.params.detach().cpu().numpy()
