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
from .diagnostics import NAMES as DIAG_NAMES, grad_clip_coef, ppo_diagnostics
from .engine import (LR_BOUNDS, Engine, adapt_kl_coef, adapt_lr, check_adam, check_adam_options, check_adaptive_lr,
                     check_clip_epsilon, check_grad_noise_every, check_kl_penalty,
                     check_dual_clip, check_huber_delta, check_loss_coef, check_lr, check_max_grad_norm, check_prox_ewma,
                     check_recompute_advantage, check_skip_nonfinite, check_value_clip, check_value_norm,
                     check_weight_decay, grad_noise_estimate, grad_noise_terms)
from .packing import PackedGraphs, pack_and_upload, pack_states, infer_caps

KL_STOP_SLOT, KL_SKIP_SLOT = 13, 14       # statistics slots of the KL stop (include/upb200.h: upb_set_target_kl)
VCLIP_LOSS_SLOT, VCLIP_COUNT_SLOT = 15, 16  # sum max(a, b) and #graphs with b > a (include/upb200.h: upb_set_value_clip)
GCLIP_NORM_SLOT = 17                         # the pre-clip global norm a step used (include/upb200.h: upb_set_max_grad_norm)
KLPEN_SLOT = 18                              # sum of the exact per-graph KL (include/upb200.h: upb_set_kl_penalty)
NONFINITE_COUNT_SLOT, NONFINITE_SLOT = 7, 19  # #non-finite per-graph results; 1 on a step the guard skipped
                                             # (include/upb200.h: upb_set_nonfinite_guard)
DUAL_COUNT_SLOT = 20                         # #graphs whose dual-clip bound was active (include/upb200.h: upb_set_dual_clip)
HUBER_COUNT_SLOT = 21                        # #graphs in Huber's linear branch (include/upb200.h: upb_set_huber_delta)
LR_DECISION_SLOT = 22                        # the KL-adaptive lr's decision +1 / -1 / 0 (include/upb200.h:
                                             # upb_set_adaptive_lr)
PROX_WEIGHT_SLOT, PROX_KL_SLOT = 23, 24      # sum w and the behaviour-to-proximal KL estimate (include/upb200.h:
                                             # upb_set_prox_ewma)


def unguarded_nonfinite(st: np.ndarray, skip_nonfinite: bool) -> bool:
    """True when a statistics row counts a non-finite per-graph result (slot 7, a NaN there included) that nothing
    kept away from the log: always while the guard is off; with it on, a counted row the guard did not skip (slot 19
    clear).  That is a row that stopped on the KL criterion first, whose losses are logged and are not finite, or a
    fault of the library."""
    bad = st[:, NONFINITE_COUNT_SLOT] != 0
    if skip_nonfinite:
        bad = bad & (st[:, NONFINITE_SLOT] == 0)
    return bool(bad.any())


class UpdateLog:
    """Host bookkeeping of one PPO update from the statistics rows its epochs leave in the gradient ring: the reference's
    per-minibatch and per-epoch loss tags (urban_planning_agent.py:338-345), the iteration's totals, the diagnostics
    means and, with the KL stop on, where the update stopped.

    With the stop on, a row with slot 13 set is the step that stopped: its losses are logged (as Stable-Baselines3 records
    that step) but it changed no parameter.  Rows with slot 14 set are steps skipped after it and log nothing.  Either
    marker ends the update after its epoch; totals and diagnostics means are over the epochs and rows that ran.

    With value clipping on, the value loss (and so the loss) is the clipped one the step optimised, slot 15, and the
    diagnostics gain value_clip_fraction, the share of the minibatch's graphs whose clipped branch won (slot 16).

    With the Huber value loss on (huber), the value loss is likewise slot 15, and the diagnostics gain huber_fraction, the
    share of the minibatch's graphs whose value term is in Huber's linear branch (slot 21 / B).  With dual clip on
    (dual_clip), they gain dual_clip_fraction, the share of the graphs with exps != 0 whose dual bound was active (slot 20
    / |ind|).

    With the global clip on (max_grad_norm), the diagnostics gain grad_norm, the pre-clip global norm a step used
    (slot 17), and grad_clip_fraction, 1 where that step's coefficient was below 1.  Both cover only the steps that
    applied Adam (not the step that stopped on the KL criterion); their totals are means over those steps.

    With the KL penalty on (kl_coef, the coefficient beta this update used), loss/kl_loss is the mean exact KL of a
    minibatch (slot 18 / |ind|, unscaled, like entropy_loss), the loss includes beta times it, and the epoch / iteration
    tags and totals follow the other losses'; diag/kl_coef logs beta once per iteration.  kl_rows holds slot 18's and
    slot 4's sums over the rows of the last epoch that ran, the measurement the adaptive coefficient uses.

    With the KL-adaptive lr on, epoch() takes the lr every row's step applied (rebuilt from slot 22) and logs it as
    diag/lr on the rows it logs.

    With the non-finite guard on (skip_nonfinite), a row with slot 19 set is a step that changed nothing because its
    statistics or its gradient were not finite.  Its sums are not finite either, so it is left out of everything above
    (the per-minibatch tags, whose step axis then counts the rows that are logged, the epoch sums, the totals, the
    diagnostics, kl_rows), like a slot-14 row, and counted: finish() returns nonfinite_skips and logs
    diag/nonfinite_skips.  An update in which such rows are all there is (no step applied) raises FloatingPointError in
    finish(): nothing was learned, and the parameters or the whole buffer are themselves bad.

    With the gradient-noise measurement on (grad_noise_batch, the update's mini_batch_size), grad_noise() adds each
    epoch's measurements whose step applied Adam (slots 13, 14 and 19 clear) and whose four values are finite, and
    finish() returns and logs, once at `iteration`, diag/grad_noise_scale, _g2, _trace and _samples from the sums
    noise_terms (engine.grad_noise_estimate), which the caller may first add across ranks."""

    def __init__(self, opt_num_epochs: int, value_pred_coef: float, entropy_coef: float, iteration: int = 0,
                 loss_iter: int = 0, log_fn=None, kl_stop: bool = False, value_clip: bool = False,
                 max_grad_norm: Optional[float] = None, kl_coef: Optional[float] = None,
                 skip_nonfinite: bool = False, dual_clip: bool = False, huber: bool = False,
                 grad_noise_batch: Optional[int] = None, prox: bool = False):
        self.skip_nonfinite, self.nonfinite_skips = bool(skip_nonfinite), 0
        self.grad_noise_batch = grad_noise_batch
        self.noise_terms, self.noise_samples = np.zeros(3), 0     # (U, V, D) sums and the counted measurements
        self.opt_num_epochs, self.value_pred_coef, self.entropy_coef = opt_num_epochs, value_pred_coef, entropy_coef
        self.kl_coef = kl_coef
        self.kl_total, self.kl_rows = 0.0, (0.0, 0.0)
        self.iteration, self.loss_iter, self.log_fn, self.kl_stop_on = iteration, loss_iter, log_fn, kl_stop
        self.value_clip, self.dual_clip, self.huber, self.prox = value_clip, dual_clip, huber, prox
        self.diag_names = (DIAG_NAMES + (("value_clip_fraction",) if value_clip else ())
                           + (("dual_clip_fraction",) if dual_clip else ()) + (("huber_fraction",) if huber else ())
                           + (("prox_weight", "prox_kl") if prox else ()))
        self.totals = np.zeros(4)
        self.diag_sums, self.diag_count = dict.fromkeys(self.diag_names, 0.0), 0
        self.max_grad_norm = max_grad_norm
        self.gclip_names = ("grad_norm", "grad_clip_fraction") if max_grad_norm is not None else ()
        self.gclip_sums, self.gclip_count = dict.fromkeys(self.gclip_names, 0.0), 0
        self.epochs, self.steps = 0, 0            # epochs that ran, minibatch rows logged
        self.kl_stop = None                       # (epoch, minibatch) of the step that stopped

    def epoch(self, epoch: int, st: np.ndarray, diag: Optional[dict] = None, lr: Optional[np.ndarray] = None) -> bool:
        """Logs one epoch's rows st (minibatches, >= 25 with prox, >= 22 with dual_clip or huber, >= 20 with skip_nonfinite, >= 19 with
        the KL penalty, >= 18 with max_grad_norm, else >= 15) and
        their diagnostics (ppo_diagnostics, or None); returns True
        when the update ends with this epoch."""
        ended = False
        if self.kl_stop_on and st.shape[0]:
            marked = np.flatnonzero((st[:, KL_STOP_SLOT] != 0) | (st[:, KL_SKIP_SLOT] != 0))
            if marked.size:
                ended = True
                first = int(marked[0])
                n = first + 1 if st[first, KL_STOP_SLOT] != 0 else first
                if n > first:
                    self.kl_stop = (epoch, first)
                st = st[:n]
                if diag is not None:
                    diag = {name: v[:n] for name, v in diag.items()}
                if lr is not None:
                    lr = lr[:n]
        if self.skip_nonfinite and st.shape[0]:
            ran = st[:, NONFINITE_SLOT] == 0
            self.nonfinite_skips += int((~ran).sum())
            st = st[ran]
            if diag is not None:
                diag = {name: v[ran] for name, v in diag.items()}
            if lr is not None:
                lr = lr[ran]
        nb = st.shape[0]
        nB, nI = np.maximum(st[:, 3], 1), np.maximum(st[:, 4], 1)
        vl = st[:, VCLIP_LOSS_SLOT if self.value_clip or self.huber else 0] / nB
        sl_, el = st[:, 1] / nI, st[:, 2] / nI
        if diag is not None and self.value_clip:
            diag = dict(diag, value_clip_fraction=st[:, VCLIP_COUNT_SLOT] / nB)
        if diag is not None and self.dual_clip:
            diag = dict(diag, dual_clip_fraction=st[:, DUAL_COUNT_SLOT] / nI)
        if diag is not None and self.huber:
            diag = dict(diag, huber_fraction=st[:, HUBER_COUNT_SLOT] / nB)
        if diag is not None and self.prox:
            diag = dict(diag, prox_weight=st[:, PROX_WEIGHT_SLOT] / nI, prox_kl=st[:, PROX_KL_SLOT] / nI)
        loss = sl_ + self.value_pred_coef * vl + self.entropy_coef * el
        kl = None
        if self.kl_coef is not None:
            kl = st[:, KLPEN_SLOT] / nI
            loss = loss + self.kl_coef * kl
            self.kl_rows = (float(st[:, KLPEN_SLOT].sum()), float(st[:, 4].sum()))
        gclip = None
        if diag is not None and self.gclip_names:
            applied = np.flatnonzero(st[:, KL_STOP_SLOT] == 0) if self.kl_stop_on else np.arange(nb)
            norm = st[applied, GCLIP_NORM_SLOT]
            gclip = (applied, dict(grad_norm=norm,
                                   grad_clip_fraction=(grad_clip_coef(norm, self.max_grad_norm) < 1).astype(np.float64)))
        log_fn = self.log_fn
        if log_fn is not None:
            for i in range(nb):
                log_fn("loss/loss", float(loss[i]), self.loss_iter + i)
                log_fn("loss/value_loss", float(vl[i]), self.loss_iter + i)
                log_fn("loss/surr_loss", float(sl_[i]), self.loss_iter + i)
                log_fn("loss/entropy_loss", float(el[i]), self.loss_iter + i)
                if kl is not None:
                    log_fn("loss/kl_loss", float(kl[i]), self.loss_iter + i)
                if diag is not None:
                    for name in self.diag_names:
                        log_fn("diag/" + name, float(diag[name][i]), self.loss_iter + i)
                if lr is not None:
                    log_fn("diag/lr", float(lr[i]), self.loss_iter + i)
            if gclip is not None:
                for k, i in enumerate(gclip[0]):
                    for name in self.gclip_names:
                        log_fn("diag/" + name, float(gclip[1][name][k]), self.loss_iter + int(i))
            ge = self.iteration * self.opt_num_epochs + epoch
            log_fn("loss/epoch_loss", float(loss.sum()), ge)
            log_fn("loss/epoch_value_loss", float(vl.sum()), ge)
            log_fn("loss/epoch_surr_loss", float(sl_.sum()), ge)
            log_fn("loss/epoch_entropy_loss", float(el.sum()), ge)
            if kl is not None:
                log_fn("loss/epoch_kl_loss", float(kl.sum()), ge)
        self.loss_iter += nb
        self.totals += [loss.sum(), vl.sum(), sl_.sum(), el.sum()]
        if kl is not None:
            self.kl_total += float(kl.sum())
        if diag is not None:
            for name in self.diag_names:
                self.diag_sums[name] += float(diag[name].sum())
            self.diag_count += nb
        if gclip is not None:
            for name in self.gclip_names:
                self.gclip_sums[name] += float(gclip[1][name].sum())
            self.gclip_count += gclip[0].size
        self.epochs += 1
        self.steps += nb
        return ended

    def grad_noise(self, st: np.ndarray, measured: Sequence[int], noise: np.ndarray) -> None:
        """Adds one epoch's gradient-noise measurements: noise[j] ({A, S, Q, N}) was taken before the step of row
        st[measured[j]], and counts when that step applied Adam and the four values are finite."""
        for j, i in enumerate(measured):
            row = st[i]
            if row[KL_STOP_SLOT] != 0 or row[KL_SKIP_SLOT] != 0 or row[NONFINITE_SLOT] != 0:
                continue
            if not np.isfinite(noise[j]).all():
                continue
            self.noise_terms += grad_noise_terms(noise[j])
            self.noise_samples += 1

    def finish(self, diagnostics: bool) -> dict:
        """Logs the iteration's totals; the dict update_params returns."""
        if self.nonfinite_skips and self.steps - (self.kl_stop is not None) == 0:
            raise FloatingPointError(f"every optimiser step of the PPO update was skipped as non-finite "
                                     f"({self.nonfinite_skips} steps): the parameters or the rollout buffer are bad")
        totals = self.totals / max(self.epochs, 1)
        log_fn, iteration = self.log_fn, self.iteration
        if log_fn is not None:
            log_fn("loss/total_loss", float(totals[0]), iteration)
            log_fn("loss/total_value_loss", float(totals[1]), iteration)
            log_fn("loss/total_surr_loss", float(totals[2]), iteration)
            log_fn("loss/total_entropy_loss", float(totals[3]), iteration)
        out = dict(total_loss=totals[0], total_value_loss=totals[1], total_surr_loss=totals[2],
                   total_entropy_loss=totals[3])
        if self.kl_coef is not None:
            out["total_kl_loss"] = self.kl_total / max(self.epochs, 1)
            out["kl_coef"] = self.kl_coef
            if log_fn is not None:
                log_fn("loss/total_kl_loss", float(out["total_kl_loss"]), iteration)
                log_fn("diag/kl_coef", float(self.kl_coef), iteration)
        if diagnostics:
            # means over every minibatch step of the iteration
            for name in self.diag_names:
                out["total_" + name] = self.diag_sums[name] / self.diag_count if self.diag_count else float("nan")
                if log_fn is not None:
                    log_fn("diag/total_" + name, float(out["total_" + name]), iteration)
            for name in self.gclip_names:          # means over the steps that applied Adam
                out["total_" + name] = self.gclip_sums[name] / self.gclip_count if self.gclip_count else float("nan")
                if log_fn is not None:
                    log_fn("diag/total_" + name, float(out["total_" + name]), iteration)
        if self.skip_nonfinite:
            out["nonfinite_skips"] = self.nonfinite_skips
            if log_fn is not None:
                log_fn("diag/nonfinite_skips", float(self.nonfinite_skips), iteration)
        if self.grad_noise_batch is not None:
            est = grad_noise_estimate(*self.noise_terms, self.grad_noise_batch, self.noise_samples)
            out.update(est)
            if log_fn is not None:
                for name, v in est.items():
                    log_fn("diag/" + name, float(v), iteration)
        if self.kl_stop_on:
            out["steps_applied"] = self.steps - (self.kl_stop is not None)
            out["kl_stop"] = self.kl_stop
            if log_fn is not None:
                log_fn("diag/steps_applied", float(out["steps_applied"]), iteration)
        return out


class PPOUpdater:
    def __init__(self, flat_params, n_cap: int, e_cap: int, device, lr: float = 4e-4, eps: float = 1e-5,
                 clip_epsilon: float = 0.2, value_pred_coef: float = 0.5, entropy_coef: float = 0.01,
                 gamma: float = 1.0, tau: float = 0.0, opt_num_epochs: int = 4, mini_batch_size: int = 256,
                 clip_mode: int = _lib.CLIP_REFERENCE, process_group="auto", pack_threads: int = 0,
                 use_peers: bool = True, batch_stage: bool = False, model: str = "sgnn",
                 weight_decay: float = 0.0, diagnostics: bool = False, target_kl: Optional[float] = None,
                 value_clip: Optional[float] = None, normalize_advantage: bool = False,
                 max_grad_norm: Optional[float] = None, kl_coef: Optional[float] = None,
                 kl_target: Optional[float] = None, skip_nonfinite: bool = False, value_norm: bool = False,
                 value_norm_beta: float = 0.99999, param_groups: bool = False, recompute_advantage: bool = False,
                 adam_options: bool = False, dual_clip: Optional[float] = None, huber_delta: Optional[float] = None,
                 desired_kl: Optional[float] = None, lr_bounds=LR_BOUNDS, grad_noise_every: Optional[int] = None,
                 prox_ewma: Optional[float] = None):
        # prox_ewma: PPO-EWMA's proximal policy, the clip's anchor an exponential moving average of the weights with
        # weight prox_ewma per optimiser step (upb_set_prox_ewma).  Its parameters start from the live ones at the top of
        # the first update (and after a checkpoint without them); the behaviour policy stays in the importance weight.
        # None = off
        self.prox_ewma = check_prox_ewma(prox_ewma)
        self._prox_ready = False
        # grad_noise_every: measure the gradient noise scale before minibatch step i of every epoch when
        # i % grad_noise_every == 0, from one extra gradient launch of this rank's shard in a seeded random order
        # (Engine.ppo_grad_noise); update_params returns and logs the update's estimate.  Training is unchanged.  None = off
        self.grad_noise_every = check_grad_noise_every(grad_noise_every)
        # diagnostics: also report approx. KL, clip fraction, explained variance and the pre-clip gradient norms of
        # every minibatch (diag/* tags, total_* entries); costs one extra launch per epoch, none per step
        self.diagnostics = bool(diagnostics)
        # target_kl: Stable-Baselines3's early stop, decided inside the step kernels (upb_set_target_kl): the update ends
        # before the first step whose approximate KL exceeds 1.5 * target_kl; no later epoch is launched
        self.target_kl = target_kl
        # value_clip: the clipped value loss (upb_set_value_clip) against the values of the update's pre-pass;
        # normalize_advantage: each minibatch's advantages normalised on the device at the top of every epoch
        # (upb_normalize_advantages).  Both off by default
        self.value_clip = check_value_clip(value_clip) or None
        self.normalize_advantage = bool(normalize_advantage)
        # dual_clip: dual-clip PPO, a negative advantage's surrogate bounded below by dual_clip * A (upb_set_dual_clip);
        # huber_delta: the Huber value loss with threshold huber_delta (upb_set_huber_delta).  Both off by default
        self.dual_clip = check_dual_clip(dual_clip) or None
        self.huber_delta = check_huber_delta(huber_delta) or None
        # desired_kl: RSL-RL's adaptive lr schedule, decided by every minibatch step inside the step kernels on the
        # approximate KL at the parameters it starts from (upb_set_adaptive_lr): lr / 1.5 above 2 desired_kl, lr * 1.5
        # below desired_kl / 2, within lr_bounds; the adapted lr carries into the next update.  None = off
        desired_kl, lr_min, lr_max = check_adaptive_lr(desired_kl, lr_bounds)
        self.desired_kl, self.lr_bounds = desired_kl or None, (lr_min, lr_max)
        # max_grad_norm: clip_grad_norm_(parameters(), max_grad_norm) on every step inside the step kernels
        # (upb_set_max_grad_norm); needs clip_mode=CLIP_NEVER.  None = off
        self.max_grad_norm = check_max_grad_norm(max_grad_norm, clip_mode) or None
        # kl_coef: the KL penalty beta * KL(pi_old || pi) on the exact categorical KL against the update's pre-pass
        # (upb_set_kl_penalty); kl_target: adapt beta after every update by the PPO paper's rule (adapt_kl_coef) on the
        # mean KL the last epoch's steps measured.  None = off / a fixed beta
        kl_coef, kl_target = check_kl_penalty(kl_coef, kl_target)
        self.kl_coef_init = kl_coef or None
        self.kl_coef = self.kl_coef_init
        self.kl_target = kl_target or None
        # skip_nonfinite: a step whose statistics or reduced gradient are not finite changes nothing, decided inside the
        # step kernels (upb_set_nonfinite_guard); the update goes on, counts such steps (nonfinite_skips) and raises
        # only when no step was applied.  False: a non-finite minibatch raises FloatingPointError after its epoch
        self.skip_nonfinite = check_skip_nonfinite(skip_nonfinite)
        # value_norm: the value head predicts values normalised by running return statistics (MAPPO's ValueNorm, EMA
        # weight value_norm_beta) and its last layer is rescaled to preserve its outputs when they move (PopArt); GAE
        # runs on the denormalised values, the value loss on normalised returns (upb_set_value_norm).  False = off
        self.value_norm, self.value_norm_beta = check_value_norm(value_norm, value_norm_beta)
        # recompute_advantage: every epoch after the first trains on advantages, returns and value-clip anchors from a
        # value-only sweep of the whole buffer at the parameters the previous epoch left (recompute_targets), as Tianshou's
        # recompute_advantage.  False = all from the update's pre-pass
        self.recompute_advantage = check_recompute_advantage(recompute_advantage)
        check_clip_epsilon(clip_epsilon)
        self.device = torch.device(device)
        self.engine = Engine(self.device, n_cap, e_cap, lr=lr, eps=eps, clip_epsilon=clip_epsilon,
                             value_pred_coef=value_pred_coef, entropy_coef=entropy_coef, clip_mode=clip_mode,
                             model=model, weight_decay=weight_decay, diagnostics=self.diagnostics,
                             target_kl=target_kl, value_clip=self.value_clip, max_grad_norm=self.max_grad_norm,
                             kl_coef=self.kl_coef, skip_nonfinite=self.skip_nonfinite, value_norm=self.value_norm,
                             value_norm_beta=self.value_norm_beta, dual_clip=self.dual_clip,
                             huber_delta=self.huber_delta, desired_kl=self.desired_kl, lr_bounds=self.lr_bounds,
                             grad_noise_every=self.grad_noise_every, prox_ewma=self.prox_ewma)
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
        self.old_values = None            # the pre-pass values, kept for the clipped value loss (normalised with
                                          # value_norm)
        self.old_cand_log_probs = None    # the pre-pass candidate log-probs, kept for the KL penalty
        # param_groups: torch.optim.Adam's param_groups and frozen tensors (set_param_groups, upb_set_param_groups); it
        # starts as one group of every tensor at lr and weight_decay.  False: every tensor is trained with lr and
        # weight_decay (set_hyperparameters), as before
        self.param_groups = bool(param_groups)
        # adam_options: betas, eps, amsgrad and decoupled_weight_decay (torch.optim.AdamW) follow set_hyperparameters or,
        # with param_groups, each group's keys (upb_set_adam, upb_set_param_groups_adam).  False: Adam with the
        # construction's betas and eps, coupled weight decay, as before
        self.adam_options = check_adam_options(adam_options)
        if self.param_groups:
            self.set_param_groups([dict(params=list(self.engine.layout.slots), lr=self.engine.lr,
                                        weight_decay=self.engine.weight_decay)])

    # the values set_hyperparameters changes, in the order of the cross-rank signature (_check_same_buffer)
    HYPERPARAMETERS = ("lr", "clip_epsilon", "value_pred_coef", "entropy_coef", "weight_decay", "gamma", "tau",
                       "opt_num_epochs", "mini_batch_size")

    # the Adam settings set_hyperparameters changes with adam_options on, after HYPERPARAMETERS in the signature
    ADAM_OPTIONS = ("betas", "eps", "amsgrad", "decoupled_weight_decay")

    def hyperparameters(self) -> dict:
        """The Python values the next update trains with (the ones last passed to the engine for its settings); with
        adam_options on, also the Adam settings (ADAM_OPTIONS)."""
        e = self.engine
        out = dict(lr=e.lr, clip_epsilon=e.clip_epsilon, value_pred_coef=self.value_pred_coef,
                   entropy_coef=self.entropy_coef, weight_decay=e.weight_decay, gamma=self.gamma, tau=self.tau,
                   opt_num_epochs=self.opt_num_epochs, mini_batch_size=self.mini_batch_size)
        if getattr(self, "adam_options", False):
            b1, b2, eps, ams, dec = e.adam
            out.update(betas=(b1, b2), eps=eps, amsgrad=ams, decoupled_weight_decay=dec)
        return out

    def set_hyperparameters(self, lr=None, clip_epsilon=None, value_pred_coef=None, entropy_coef=None,
                            weight_decay=None, gamma=None, tau=None, opt_num_epochs=None, mini_batch_size=None,
                            betas=None, eps=None, amsgrad=None, decoupled_weight_decay=None) -> None:
        """Change the training hyperparameters from the next update on, as a reference user does between iterations (an
        lr scheduler on the optimizer, agent.entropy_coef = ..., urban_planning_agent.py:248-361 reads them at every
        update).  None keeps a value.  Every value is validated first (ValueError, as torch.optim.Adam raises for lr and
        weight_decay), and nothing changes if one is invalid.  A value equal to the current one issues no call; lr and
        the loss coefficients are kept as the Python values passed, the library rounds the coefficients to fp32."""
        if getattr(self, "param_groups", False) and (lr is not None or weight_decay is not None):
            raise ValueError("parameter groups are on: each tensor's lr and weight_decay come from set_param_groups")
        adam_given = dict(betas=betas, eps=eps, amsgrad=amsgrad, decoupled_weight_decay=decoupled_weight_decay)
        if any(v is not None for v in adam_given.values()):
            if not getattr(self, "adam_options", False):
                raise ValueError("betas, eps, amsgrad and decoupled_weight_decay need the updater built with "
                                 "adam_options=True")
            if self.param_groups:
                raise ValueError("parameter groups are on: each tensor's Adam settings come from set_param_groups")

        def count(name, v):
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < 1:
                raise ValueError(f"Invalid {name} value: {v!r} (a positive integer)")
            return int(v)

        def finite(name, v):
            f = float(v)
            if not math.isfinite(f):
                raise ValueError(f"Invalid {name} value: {v}")
            return f

        checks = dict(lr=check_lr, clip_epsilon=check_clip_epsilon,
                      value_pred_coef=lambda v: check_loss_coef("value_pred_coef", v),
                      entropy_coef=lambda v: check_loss_coef("entropy_coef", v), weight_decay=check_weight_decay,
                      gamma=lambda v: finite("gamma", v), tau=lambda v: finite("tau", v),
                      opt_num_epochs=lambda v: count("opt_num_epochs", v),
                      mini_batch_size=lambda v: count("mini_batch_size", v))
        given = dict(lr=lr, clip_epsilon=clip_epsilon, value_pred_coef=value_pred_coef, entropy_coef=entropy_coef,
                     weight_decay=weight_decay, gamma=gamma, tau=tau, opt_num_epochs=opt_num_epochs,
                     mini_batch_size=mini_batch_size)
        cur = self.hyperparameters()
        new = dict(cur, **{k: checks[k](v) for k, v in given.items() if v is not None})
        eng = self.engine
        adam = None
        if any(v is not None for v in adam_given.values()):
            b1, b2, e, ams, dec = eng.adam
            a = dict(dict(betas=(b1, b2), eps=e, amsgrad=ams, decoupled_weight_decay=dec),
                     **{k: v for k, v in adam_given.items() if v is not None})
            adam = check_adam(a["betas"], a["eps"], a["amsgrad"], a["decoupled_weight_decay"])
        if new["lr"] != cur["lr"]:
            eng.set_lr(new["lr"])
        if new["clip_epsilon"] != cur["clip_epsilon"]:
            eng.set_clip_epsilon(new["clip_epsilon"])
        if (new["value_pred_coef"], new["entropy_coef"]) != (cur["value_pred_coef"], cur["entropy_coef"]):
            eng.set_loss_coefs(new["value_pred_coef"], new["entropy_coef"])
        if new["weight_decay"] != cur["weight_decay"]:
            eng.set_weight_decay(new["weight_decay"])
        if adam is not None and adam != eng.adam:
            eng.set_adam(adam[:2], *adam[2:])
        self.value_pred_coef, self.entropy_coef = new["value_pred_coef"], new["entropy_coef"]
        self.gamma, self.tau = new["gamma"], new["tau"]
        self.opt_num_epochs, self.mini_batch_size = new["opt_num_epochs"], new["mini_batch_size"]

    def set_param_groups(self, groups) -> None:
        """The parameter groups of the next updates: a list of {"params": [slot names], "lr", "weight_decay"} (slot
        names of params.SGNN / params.MLP; weight_decay defaults to 0), as torch.optim.Adam's param_groups.  A tensor in
        no group is frozen: no Adam step, a zero gradient column, its moments and count kept.  With adam_options on, a
        group may also carry "betas", "eps", "amsgrad" and "decoupled_weight_decay" (defaults: the updater's betas and
        eps, False, False).  A tensor in two groups, an unknown name, an invalid lr, weight decay or Adam setting or no
        trained tensor raises ValueError and changes nothing.  A table equal to the current one issues no call.  Needs the
        updater built with param_groups=True."""
        if not self.param_groups:
            raise ValueError("parameter groups are off: construct the updater with param_groups=True")
        options = getattr(self, "adam_options", False)
        names = list(self.engine.layout.slots)
        lr, wd, trained = [0.0] * len(names), [0.0] * len(names), [False] * len(names)
        default = (*self.engine.betas, self.engine.eps, False, False) if options else None
        adam = [default] * len(names)
        for g in groups:
            g_lr, g_wd = check_lr(g["lr"]), check_weight_decay(g.get("weight_decay", 0.0))
            g_adam = default
            if options:
                g_adam = check_adam(g.get("betas", default[:2]), g.get("eps", default[2]), g.get("amsgrad", False),
                                    g.get("decoupled_weight_decay", False))
            for name in g["params"]:
                if name not in names:
                    raise ValueError(f"parameter groups: unknown tensor {name!r}")
                k = names.index(name)
                if trained[k]:
                    raise ValueError(f"parameter groups: tensor {name!r} is in more than one group")
                lr[k], wd[k], trained[k], adam[k] = g_lr, g_wd, True, g_adam
        table = (tuple(lr), tuple(wd), tuple(trained))
        # each group's first tensor (None: a group without one) and its lr: the adaptive lr reports per group
        self._lr_groups = [(names.index(g["params"][0]) if g["params"] else None, check_lr(g["lr"])) for g in groups]
        if not options:
            if table != self.engine.param_groups:
                self.engine.set_param_groups(*table)
        elif table != self.engine.param_groups or tuple(adam) != self.engine.param_group_adam:
            self.engine.set_param_groups(*table, adam=tuple(adam))

    def _param_group_signature(self) -> dict:
        """The per-tensor table as signature entries of _check_same_buffer."""
        lr, wd, trained = self.engine.param_groups
        adam = getattr(self.engine, "param_group_adam", None)
        out = {}
        for k, name in enumerate(self.engine.layout.slots):
            out[f"lr[{name}]"], out[f"weight_decay[{name}]"] = lr[k], wd[k]
            out[f"trained[{name}]"] = float(trained[k])
            if adam is not None:
                for key, v in zip(("beta1", "beta2", "eps", "amsgrad", "decoupled_weight_decay"), adam[k]):
                    out[f"{key}[{name}]"] = float(v)
        return out

    def set_kl_coef(self, beta: float) -> None:
        """The KL penalty's coefficient for the next updates (the penalty must have been configured with kl_coef)."""
        if self.kl_coef is None:
            raise ValueError("the KL penalty is off: construct the updater with kl_coef")
        b = float(beta)
        if not math.isfinite(b) or b <= 0.0:
            raise ValueError(f"Invalid kl_coef value: {beta}")
        self.engine.set_kl_coef(b)
        self.kl_coef = b

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
        hyper = self.hyperparameters()
        if "betas" in hyper:        # adam_options: one float per signature entry
            hyper["beta1"], hyper["beta2"] = hyper.pop("betas")
        if getattr(self, "param_groups", False):
            hyper.update(self._param_group_signature())
        hyper["recompute_advantage"] = float(getattr(self, "recompute_advantage", False))
        hyper["dual_clip"] = float(getattr(self, "dual_clip", None) or 0.0)
        hyper["huber_delta"] = float(getattr(self, "huber_delta", None) or 0.0)
        if getattr(self, "desired_kl", None) is not None:
            hyper["desired_kl"] = float(self.desired_kl)
            hyper["lr_min"], hyper["lr_max"] = self.lr_bounds
        hyper["grad_noise_every"] = float(getattr(self, "grad_noise_every", None) or 0)
        prox = getattr(self, "prox_ewma", None)
        hyper["prox_ewma"] = -1.0 if prox is None else float(prox)
        self._check_same_buffer(info, hyper)
        return self.blob

    def _check_same_buffer(self, info: np.ndarray, hyper: Optional[dict] = None) -> None:
        """Data-parallel ranks must hold the SAME rollout buffer (the shards are index ranges into it) and train with the
        same hyperparameters `hyper` (name -> value; their steps are one step, so a rank that anneals differently, e.g. a
        ReduceLROnPlateau fed per-rank rewards, would make the ranks' parameters drift apart)."""
        if self.world <= 1:
            return
        import zlib
        import torch.distributed as dist
        sig = [int(info.shape[0]), zlib.crc32(np.ascontiguousarray(info).tobytes()),
               zlib.crc32(np.ascontiguousarray(self.exps_host).tobytes()),
               zlib.crc32(self.actions.cpu().numpy().tobytes())]
        names = list((hyper or {}).keys())
        # the float64 bit patterns: equal exactly when the Python floats are
        sig += [int(np.float64(hyper[k]).view(np.int64)) for k in names]
        on = self.device if dist.get_backend(self.pg) == "nccl" else torch.device("cpu")
        lo = torch.tensor(sig, dtype=torch.int64, device=on)
        hi = lo.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=self.pg)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=self.pg)
        differ = (lo != hi).cpu().numpy()
        if differ[:4].any():
            raise _lib.UpbError("data-parallel ranks hold different rollout buffers (count / graph sizes / exps / "
                                "actions differ): every rank must load the same states")
        if differ[4:].any():
            bad = ", ".join(k for k, d in zip(names, differ[4:]) if d)
            raise _lib.UpbError(f"data-parallel ranks train with different hyperparameters ({bad} differ): every rank "
                                "must set the same values before an update (a scheduler fed per-rank metrics must be "
                                "fed the same value on every rank)")

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
    def forward_all(self, cand_log_probs: bool = False):
        """value, log_prob, entropy (and the candidates' log-probs) of every state in the buffer (reference :256-264
        and :283-292, one pass)."""
        return self.engine.forward(self.blob, self.params, self.actions, cand_log_probs=cand_log_probs)

    def allreduce(self, buf: torch.Tensor):
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.pg)

    def _step_inputs(self, global_batch: int, global_ind: int):
        """The training calls' positional arguments for a minibatch of `global_batch` graphs, `global_ind` of which have
        exps != 0, and the reference data its options need (old values, old candidate log-probs; None while off)."""
        adv = self.norm_advantages if self.normalize_advantage else self.advantages
        args = (self.blob, self.params, self.actions, adv, self.returns, self.fixed_log_probs, self.exps,
                1.0 / max(global_batch, 1), 1.0 / max(global_ind, 1))
        ov = self.old_values if self.value_clip is not None else None
        oc = self.old_cand_log_probs if self.kl_coef is not None else None
        return args, ov, oc

    def minibatch_step(self, ids: torch.Tensor, global_batch: int, global_ind: int):
        """One optimiser step on the graphs `ids` (this rank's shard of a global minibatch of `global_batch`
        graphs, `global_ind` of which have exps != 0): urban_planning_agent.py:322-337."""
        args, ov, oc = self._step_inputs(global_batch, global_ind)
        if self.world == 1 or (self.fused_exchange and self.engine.next_step_fused()):
            # one launch: gradient, reduction (over the SGNN ranks too, through peer memory), Adam.  rl-mlp ranks never
            # have fused_exchange (Engine.connect_peers) and keep the NCCL path below
            self.engine.ppo_step(*args, ids=ids, out=self.grad, old_values=ov, old_cand_log_probs=oc)
        else:
            self.engine.ppo_grad(*args, ids=ids, out=self.grad, old_values=ov, old_cand_log_probs=oc)
            self.allreduce(self.grad)
            self.engine.apply(self.params, self.grad)

    def measure_grad_noise(self, ids: torch.Tensor, global_batch: int, global_ind: int, noise_out: torch.Tensor):
        """The gradient-noise measurement of the minibatch whose step minibatch_step(ids', global_batch, global_ind) runs
        next: Engine.ppo_grad_noise of this rank's shard `ids` (in a random order) with that step's inputs, into a
        scratch gradient buffer (never the step's ring row) and noise_out.  Rank-local; queued on the stream."""
        args, ov, oc = self._step_inputs(global_batch, global_ind)
        if getattr(self, "_noise_grad", None) is None:
            self._noise_grad = self.engine.new_grad_buffer()
        self.engine.ppo_grad_noise(*args, ids=ids, out=self._noise_grad, noise_out=noise_out, old_values=ov,
                                   old_cand_log_probs=oc)

    def _read_epoch_with_norms(self, ring: torch.Tensor, nb: int, stats: torch.Tensor, then=None):
        """The epoch's statistics rows and the squared gradient norms of its ring rows (one launch), both copied into
        pinned host memory and read after one synchronisation.  then: as for _wait_for_rows."""
        norms = self.engine.grad_norms(ring[:nb])
        hs, hn = self._pinned_rows(nb, stats.shape[1])
        hs.copy_(stats, non_blocking=True)
        hn.copy_(norms, non_blocking=True)
        self._wait_for_rows(then)
        return hs.numpy().astype(np.float64), hn.numpy().astype(np.float64)

    def _read_epoch_then(self, nb: int, stats: torch.Tensor, then) -> np.ndarray:
        """The epoch's statistics rows, copied into pinned host memory and read once the copy is done; `then` is queued
        behind the copy (_wait_for_rows)."""
        hs, _ = self._pinned_rows(nb, stats.shape[1])
        hs.copy_(stats, non_blocking=True)
        self._wait_for_rows(then)
        return hs.numpy().astype(np.float64)

    def _pinned_rows(self, nb: int, width: int):
        host = getattr(self, "_diag_host", None)
        if host is None or host[0].shape[0] < nb:
            host = tuple(torch.empty(nb, w, dtype=torch.float32, pin_memory=True) for w in (width, 3))
            self._diag_host = host
        return host[0][:nb], host[1][:nb]

    def _wait_for_rows(self, then=None) -> None:
        """Waits for the copies queued so far.  then (None: nothing) is called after an event is recorded behind them:
        the work it queues runs on the device while the host waits for the copies and reads them."""
        stream = torch.cuda.current_stream(self.device)
        if then is None:
            stream.synchronize()
            return
        if getattr(self, "_rows_copied", None) is None:
            self._rows_copied = torch.cuda.Event()
        self._rows_copied.record(stream)
        then()
        self._rows_copied.synchronize()

    def recompute_targets(self) -> None:
        """recompute_advantage: the advantages, returns and (with value_clip) value-clip anchors of the next epoch from
        one value-only sweep of the whole buffer at the current parameters (Engine.values) and one launch of
        Engine.gae_targets with the update's gamma and tau.  With value_norm, the values are denormalised and the returns
        normalised with the statistics of this update, which do not move.  Queued on the stream; no synchronisation.
        Every rank of a data-parallel update holds the same buffer and parameters, so every rank gets the same targets
        without an exchange."""
        head = self.engine.values(self.blob, self.params)
        adv, ret, anchor = self.engine.gae_targets(self._rewards_t, self._masks_t, head, self.gamma, self.tau)
        self.advantages, self.returns = adv, ret
        if self.value_clip is not None:
            self.old_values = anchor

    # ------------------------------------------------------------------ the reference's update_params
    def update_params(self, states: Sequence, actions, rewards, masks, exps=None,
                      log_fn: Optional[Callable[[str, float, int], None]] = None, iteration: int = 0):
        """Full update of one iteration.  Returns dict of mean losses per epoch (the reference's 'total_*')."""
        self.load_states(states, actions, exps)
        T = self.blob.count
        dev = self.device
        # one no-grad sweep yields both pre-pass results of the reference: values (:256-264) and the fixed
        # log-probs (:283-292); neither depends on the other.  With the KL penalty on, the same sweep also yields every
        # candidate's log-prob, the reference distribution of the penalty
        if self.kl_coef is not None:
            values, self.fixed_log_probs, _, self.old_cand_log_probs = self.forward_all(cand_log_probs=True)
        else:
            values, self.fixed_log_probs, _ = self.forward_all()
        if self.value_norm:
            values = self.engine.denormalize_values(values)        # the head's outputs are in normalised units
        self.old_values = values
        rewards_t = torch.as_tensor(np.ascontiguousarray(rewards, np.float32)).reshape(T).to(dev)
        masks_t = torch.as_tensor(np.ascontiguousarray(masks, np.float32)).reshape(T).to(dev)
        self._rewards_t, self._masks_t = rewards_t, masks_t          # recompute_targets' inputs
        self.advantages, self.returns = self.engine.gae(rewards_t, masks_t, values, self.gamma, self.tau)  # :267
        vn_host = None
        if self.value_norm:
            # the statistics move once per update, from every return (exps == 0 graphs included: the value loss covers
            # them); the head is rescaled in place, and the steps train on normalised returns and old values
            self.returns, self.old_values, mean_std = self.engine.value_norm_update(self.returns, self.params, values)
            # read after the first epoch's synchronisation, which this copy precedes in stream order
            vn_host = getattr(self, "_vn_host", None)
            if vn_host is None:
                vn_host = self._vn_host = torch.empty(2, dtype=torch.float64, pin_memory=True)
                self._vn_done = torch.cuda.Event()
            vn_host.copy_(mean_std, non_blocking=True)
            self._vn_done.record(torch.cuda.current_stream(dev))
        out = self.update_policy(iteration, log_fn)
        if vn_host is not None:
            self._vn_done.synchronize()            # complete already after an epoch's read; waits only when nothing ran
            mean, std = (float(x) for x in vn_host.numpy())
            out["value_norm_mean"], out["value_norm_std"] = mean, std
            if log_fn is not None:
                log_fn("diag/value_norm_mean", mean, iteration)
                log_fn("diag/value_norm_std", std, iteration)
        return out

    def update_policy(self, iteration: int = 0, log_fn=None):
        T, B = self.blob.count, self.mini_batch_size
        nb = int(math.floor(T / B))
        # one gradient / statistics row per minibatch of the epoch: the step kernels write their loss statistics
        # straight into their own row (no per-step device copy), read back once per epoch
        ring = getattr(self, "_grad_ring", None)
        if ring is None or ring.shape[0] < max(nb, 1):
            ring = torch.zeros(max(nb, 1), self.engine.grad_stride, dtype=torch.float32, device=self.device)
            self._grad_ring = ring
        book = UpdateLog(self.opt_num_epochs, self.value_pred_coef, self.entropy_coef, iteration, self.loss_iter, log_fn,
                         kl_stop=self.target_kl is not None, value_clip=self.value_clip is not None,
                         max_grad_norm=self.max_grad_norm, kl_coef=self.kl_coef, skip_nonfinite=self.skip_nonfinite,
                         dual_clip=self.dual_clip is not None, huber=self.huber_delta is not None,
                         grad_noise_batch=B if getattr(self, "grad_noise_every", None) is not None else None,
                         prox=getattr(self, "prox_ewma", None) is not None)
        if getattr(self, "prox_ewma", None) is not None and not self._prox_ready:
            # the proximal parameters start from the live ones (queued on the stream; every rank holds the same)
            self.engine.init_prox_params(self.params)
            self._prox_ready = True
        # grad_noise_every: the measured steps of every epoch, their {A, S, Q, N} rows on the device and a pinned copy
        k_noise = getattr(self, "grad_noise_every", None)
        measured = list(range(0, nb, k_noise)) if k_noise is not None else []
        if measured:
            noise_dev = torch.zeros(len(measured), 4, dtype=torch.float64, device=self.device)
            noise_host = getattr(self, "_noise_host", None)
            if noise_host is None or noise_host.shape[0] < len(measured):
                noise_host = self._noise_host = torch.zeros(len(measured), 4, dtype=torch.float64, pin_memory=True)
        if self.normalize_advantage:
            # minibatches outside floor(T / B) * B keep the raw advantages (they are never stepped on)
            self.norm_advantages = self.advantages.clone()

        def prepare(order, epoch):
            """Host side of one epoch: the sample order, this rank's shard of every minibatch in the order of the
            kernel's static CTA schedule (long + short graph per CTA), one upload.  With grad_noise_every, the measured
            minibatches' shards follow in a random order (rows nb, nb + 1, ...), each from its own generator seeded by
            (iteration, epoch, minibatch, rank) so that np.random, whose stream the epochs' permutations draw, is not
            touched: under the static schedule a CTA's graphs are then a random subset of the shard."""
            order = self._epoch_order(order)
            raw = [order[i * B:(i + 1) * B][self.rank::self.world] for i in range(nb)]
            shards = [self.engine.balance_ids(x, self._cost) for x in raw]
            shards += [np.random.default_rng([iteration % 2**32, epoch, i, self.rank]).permutation(raw[i])
                       for i in measured]
            width = max((len(x) for x in shards), default=0)
            ids_host = np.zeros((max(nb, 1) + len(measured), max(width, 1)), np.int32)
            for i, x in enumerate(shards):
                ids_host[i, :len(x)] = x
            n_ind = [int((self.exps_host[order[i * B:(i + 1) * B]] != 0).sum()) for i in range(nb)]
            # the global order, for the advantage normalisation of every minibatch (the same on every rank)
            order_dev = (torch.as_tensor(order[:nb * B].astype(np.int32)).to(self.device, non_blocking=True)
                         if self.normalize_advantage else None)
            return (order, [len(x) for x in shards], torch.as_tensor(ids_host).to(self.device, non_blocking=True), n_ind,
                    order_dev)

        cur = prepare(np.arange(T), 0)
        if self.target_kl is not None:
            self.engine.reset_kl_stop()            # a new update trains again
        adaptive = getattr(self, "desired_kl", None) is not None
        if adaptive:
            # the lrs the update starts from, as the engine last set or rebuilt them, and a pinned copy of the device
            # state queued before every epoch's read (the last one is the update's final state)
            lrs, trained, lr_host = self._lr_start()
            lr_changes = dict(up=0, down=0)
        for epoch in range(self.opt_num_epochs):
            torch.cuda.nvtx.range_push(f"upb.epoch{epoch}")
            order, lens, ids_dev, n_inds, order_dev = cur
            if order_dev is not None and nb:
                # in stream order after the previous epoch's steps
                self.engine.normalize_advantages(self.advantages, self.exps, order_dev, B, out=self.norm_advantages)
            for i in range(nb):
                self.grad = ring[i]
                if k_noise is not None and i % k_noise == 0:
                    # at the parameters step i starts from; its own row of the upload, the shard in a random order
                    self.measure_grad_noise(ids_dev[nb + i // k_noise, :lens[i]], min((i + 1) * B, T) - i * B,
                                            n_inds[i], noise_dev[i // k_noise])
                self.minibatch_step(ids_dev[i, :lens[i]], min((i + 1) * B, T) - i * B, n_inds[i])
            # the next epoch's host work overlaps this epoch's kernels (one process; with several ranks the order is
            # broadcast on the stream, which would wait for them)
            if epoch + 1 < self.opt_num_epochs and self.world == 1:
                cur = prepare(order, epoch + 1)
            so = self.engine.stat_offset
            stats_all = ring[:nb, so:so + (25 if book.prox else (23 if adaptive else 22))]
                                                    # [0, 22): the sums, the KL stop's markers, the value-clip sums,
                                                    # the global clip's norm, the KL penalty's sum, the guard's marker,
                                                    # the dual-clip and Huber counts; [22] the adaptive lr's decision;
                                                    # [23, 25) the proximal policy's sums
            if adaptive:
                self.engine.read_lr_state_async(lr_host)
            if measured:
                # read with the statistics rows, after the same synchronisation
                noise_host[:len(measured)].copy_(noise_dev, non_blocking=True)
            # recompute_advantage: the next epoch's targets, queued behind the copy of this epoch's rows so that the
            # host's read and logging overlap the sweep.  None after the last epoch; an update that stops on the KL
            # criterion leaves its last sweep unused
            sweep = (self.recompute_targets if self.recompute_advantage and nb and epoch + 1 < self.opt_num_epochs
                     else None)
            diag = None
            if self.diagnostics and nb:
                st, sq = self._read_epoch_with_norms(ring, nb, stats_all, then=sweep)   # one sync per epoch
                with np.errstate(invalid="ignore", over="ignore"):       # a skipped row's sums are not finite
                    diag = ppo_diagnostics(st, sq)
            elif sweep is not None:
                st = self._read_epoch_then(nb, stats_all, sweep)                       # one sync per epoch
            else:
                st = stats_all.cpu().numpy().astype(np.float64)                        # one sync per epoch
            if self.fused_exchange and self.engine.peer_timeouts():
                raise _lib.UpbError("multi-GPU step: a peer rank never published its gradient sums (timed out inside "
                                    "the step kernel); that step's Adam update was skipped on this rank -- the ranks "
                                    "are out of sync, restore the last checkpoint")
            if nb and unguarded_nonfinite(st, self.skip_nonfinite):
                raise FloatingPointError("non-finite value / log-prob / entropy in the PPO update")
            row_lr = None
            if adaptive:
                # every row's step applied the lr its decision gave (0 on a row that applied nothing)
                row_lr = np.empty(st.shape[0])
                for i, dec in enumerate(st[:, LR_DECISION_SLOT]):
                    dec = int(dec)
                    lrs = [adapt_lr(x, dec, *self.lr_bounds) if t else x for x, t in zip(lrs, trained)]
                    row_lr[i] = self._group_lrs(lrs)[0]
                    lr_changes["up" if dec > 0 else "down"] += dec != 0
            if measured:
                book.grad_noise(st, measured, noise_host[:len(measured)].numpy())
            ended = book.epoch(epoch, st, diag, row_lr)
            self.loss_iter = book.loss_iter
            torch.cuda.nvtx.range_pop()
            if ended:                                # the KL stop: every rank reads the same rows and ends here
                break
            if epoch + 1 < self.opt_num_epochs and self.world > 1:
                cur = prepare(order, epoch + 1)
        if k_noise is not None and self.world > 1:
            # U, V and D add across ranks: one all-reduce per update, after which every rank reports the same estimate
            import torch.distributed as dist
            on = self.device if dist.get_backend(self.pg) == "nccl" else torch.device("cpu")
            terms = torch.as_tensor(book.noise_terms, dtype=torch.float64, device=on)
            dist.all_reduce(terms, op=dist.ReduceOp.SUM, group=self.pg)
            book.noise_terms = terms.cpu().numpy()
        out = book.finish(self.diagnostics)
        if adaptive:
            final = lr_host.numpy().tolist()
            if final != lrs:
                raise _lib.UpbError(f"the adaptive lr state on the device ({final}) differs from the one its steps' "
                                    f"decisions give ({lrs})")
            self._lr_end(final)
            out["lr"] = self._group_lrs(final) if self.engine.param_groups is not None else final[0]
            out["lr_changes"] = lr_changes
        if self.kl_coef is not None:
            if self.kl_target is not None:
                # every rank read the same (all-reduced) rows, so every rank takes the same decision
                nxt = adapt_kl_coef(self.kl_coef, *book.kl_rows, self.kl_target)
                if nxt != self.kl_coef:
                    self.set_kl_coef(nxt)
            out["kl_coef_next"] = self.kl_coef
        return out

    def _lr_start(self):
        """The adaptive lr's starting lrs (one, or one per tensor with parameter groups), each tensor's trained flag and
        the pinned buffer of the device state's copies."""
        eng = self.engine
        if eng.param_groups is not None:
            lrs, trained = list(eng.param_groups[0]), list(eng.param_groups[2])
        else:
            lrs, trained = [eng.lr], [True]
        host = getattr(self, "_lr_host", None)
        if host is None or host.numel() != len(lrs):
            host = self._lr_host = torch.zeros(len(lrs), dtype=torch.float64, pin_memory=True)
        return lrs, trained, host

    def _group_lrs(self, lrs) -> list:
        """Per-tensor lrs (one entry without parameter groups) as one lr per group of the last set_param_groups: its first
        tensor's (every tensor of a group takes the same decisions from the same lr), or the group's own lr when it holds
        no tensor.  Without parameter groups, [lr]."""
        if self.engine.param_groups is None:
            return [lrs[0]]
        return [lrs[k] if k is not None else lr for k, lr in self._lr_groups]

    def _lr_end(self, final) -> None:
        """The engine's Python lrs become the adapted ones the device holds, without a call: the next update starts from
        them unless set_hyperparameters / set_param_groups passes other values."""
        eng = self.engine
        if eng.param_groups is not None:
            eng.param_groups = (tuple(final),) + tuple(eng.param_groups[1:])
        else:
            eng.lr = final[0]

    def flat_params(self) -> np.ndarray:
        return self.params.detach().cpu().numpy()
