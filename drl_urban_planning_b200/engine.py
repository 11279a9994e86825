"""Thin Python face of the C ABI: one `Engine` per (process, device).

PyTorch is only the container for device memory and the source of the current CUDA stream; every computation
of the update path happens inside libupb200.so.  Reference call sites mirrored by the methods are cited in
include/upb200.h.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib, params as PL
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


def check_weight_decay(weight_decay) -> float:
    """The value as a float; ValueError for a negative or non-finite one, as torch.optim.Adam raises."""
    wd = float(weight_decay)
    if not math.isfinite(wd) or wd < 0.0:
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
    return wd


def check_target_kl(target_kl) -> float:
    """The KL-stop target as a float, None meaning 0 (off); ValueError for a negative or non-finite one."""
    kl = 0.0 if target_kl is None else float(target_kl)
    if not math.isfinite(kl) or kl < 0.0:
        raise ValueError(f"Invalid target_kl value: {target_kl}")
    return kl


def check_value_clip(value_clip) -> float:
    """The value-loss clip range as a float, None meaning 0 (off); ValueError for zero, a negative or a non-finite one."""
    if value_clip is None:
        return 0.0
    c = float(value_clip)
    if not math.isfinite(c) or c <= 0.0:
        raise ValueError(f"Invalid value_clip value: {value_clip}")
    return c


F32_MAX = float(np.finfo(np.float32).max)


def check_dual_clip(dual_clip) -> float:
    """The dual-clip bound c as a float, None meaning 0 (off); ValueError for a bool, a NaN, an infinite value and one
    not above 1, also once rounded to fp32 (as Tianshou asserts dual_clip > 1; the kernels keep fp32(c))."""
    if dual_clip is None:
        return 0.0
    if isinstance(dual_clip, (bool, np.bool_)):
        raise ValueError(f"Invalid dual_clip value: {dual_clip!r}")
    c = float(dual_clip)
    if not (math.isfinite(c) and 1.0 < c <= F32_MAX and np.float32(c) > 1.0):
        raise ValueError(f"Invalid dual_clip value: {dual_clip} (finite and > 1)")
    return c


def check_prox_ewma(prox_ewma) -> Optional[float]:
    """The EWMA proximal policy's weight beta as a float, None meaning off; ValueError for a bool, a value that is not
    finite, one outside [0, 1), and one that rounds to 1.0 in fp32 (the kernels keep fp32(beta))."""
    if prox_ewma is None:
        return None
    if isinstance(prox_ewma, (bool, np.bool_)):
        raise ValueError(f"Invalid prox_ewma value: {prox_ewma!r}")
    b = float(prox_ewma)
    if not (math.isfinite(b) and 0.0 <= b < 1.0 and float(np.float32(b)) < 1.0):
        raise ValueError(f"Invalid prox_ewma value: {prox_ewma} (finite, >= 0 and < 1, also in fp32)")
    return b


def prox_ewma_age(beta: float, batch: int = 1) -> float:
    """The EWMA proximal policy's mean age: beta / (1 - beta) optimiser steps, times `batch` graphs per step."""
    return batch * beta / (1.0 - beta)


def prox_ewma_for_batch(beta: float, batch: int, new_batch: int) -> float:
    """The weight that keeps the proximal policy's mean age in graphs, B beta / (1 - beta), when the global minibatch
    changes from `batch` to `new_batch` graphs per optimiser step."""
    age = prox_ewma_age(beta, batch) / new_batch
    return age / (1.0 + age)


def check_huber_delta(huber_delta) -> float:
    """The Huber value loss threshold delta as a float, None meaning 0 (off); ValueError for a bool, a NaN, an infinite
    value and one not above 0, also once rounded to fp32."""
    if huber_delta is None:
        return 0.0
    if isinstance(huber_delta, (bool, np.bool_)):
        raise ValueError(f"Invalid huber_delta value: {huber_delta!r}")
    d = float(huber_delta)
    if not (math.isfinite(d) and 0.0 < d <= F32_MAX and np.float32(d) > 0.0):
        raise ValueError(f"Invalid huber_delta value: {huber_delta} (finite and > 0)")
    return d


LR_BOUNDS = (1e-5, 1e-2)          # RSL-RL's bounds of the adaptive schedule


def check_adaptive_lr(desired_kl, lr_bounds=LR_BOUNDS) -> Tuple[float, float, float]:
    """The KL-adaptive lr's (desired_kl, lr_min, lr_max) as floats, desired_kl None meaning 0 (off); ValueError for a
    desired_kl that is a bool, not finite, not above 0 or whose fp32 thresholds fp32(desired_kl / 2) and
    fp32(2 desired_kl) are 0 or infinite, and for lr_bounds that are not a pair of finite values with 0 < lo <= hi.  The
    bounds are checked whether or not the option is on; None stands for LR_BOUNDS."""
    if lr_bounds is None:
        lr_bounds = LR_BOUNDS
    try:
        lo, hi = lr_bounds
    except (TypeError, ValueError):
        raise ValueError(f"Invalid lr_bounds value: {lr_bounds!r} (a pair (lr_min, lr_max))") from None
    if any(isinstance(b, (bool, np.bool_)) or not isinstance(b, (int, float, np.integer, np.floating)) for b in (lo, hi)):
        raise ValueError(f"Invalid lr_bounds value: {lr_bounds!r}")
    lo, hi = float(lo), float(hi)
    if not (math.isfinite(lo) and math.isfinite(hi) and 0.0 < lo <= hi):
        raise ValueError(f"Invalid lr_bounds value: {lr_bounds!r} (finite, 0 < lr_min <= lr_max)")
    if desired_kl is None:
        return 0.0, lo, hi
    if isinstance(desired_kl, (bool, np.bool_)) or not isinstance(desired_kl, (int, float, np.integer, np.floating)):
        raise ValueError(f"Invalid desired_kl value: {desired_kl!r}")
    d = float(desired_kl)
    with np.errstate(over="ignore"):
        up, down = np.float32(d / 2.0), np.float32(2.0 * d)
    if not (math.isfinite(d) and d > 0.0 and up > 0.0 and math.isfinite(down)):
        raise ValueError(f"Invalid desired_kl value: {desired_kl!r} (finite, > 0, with fp32 thresholds above 0 and "
                         "finite)")
    return d, lo, hi


def adapt_lr(lr: float, decision: int, lr_min: float, lr_max: float) -> float:
    """The KL-adaptive lr after a step's decision (statistics slot 22: +1 up, -1 down, 0 none) in float64, as the
    kernels form it (include/upb200.h: upb_set_adaptive_lr): max(lr_min, lr / 1.5), min(lr_max, lr * 1.5) or lr."""
    if decision < 0:
        return max(lr_min, lr / 1.5)
    if decision > 0:
        return min(lr_max, lr * 1.5)
    return lr


def check_max_grad_norm(max_grad_norm, clip_mode) -> float:
    """The global gradient-norm clip as a float, None meaning 0 (off); ValueError for zero, a negative or a non-finite
    one, and for any value with a clip_mode other than CLIP_NEVER (the reference's two-group clip would apply too)."""
    if max_grad_norm is None:
        return 0.0
    m = float(max_grad_norm)
    if not math.isfinite(m) or m <= 0.0:
        raise ValueError(f"Invalid max_grad_norm value: {max_grad_norm}")
    if clip_mode != _lib.CLIP_NEVER:
        raise ValueError("max_grad_norm replaces the reference's two-group gradient clip: pass clip_mode=CLIP_NEVER "
                         f"(got clip_mode={clip_mode})")
    return m


def check_kl_penalty(kl_coef, kl_target=None):
    """The KL penalty's initial coefficient and target as floats, None meaning 0 (off; kl_target off: a fixed
    coefficient); ValueError for zero, a negative or a non-finite value, and for a kl_target without a kl_coef."""
    def positive(name, v):
        if v is None:
            return 0.0
        f = float(v)
        if not math.isfinite(f) or f <= 0.0:
            raise ValueError(f"Invalid {name} value: {v}")
        return f
    beta, target = positive("kl_coef", kl_coef), positive("kl_target", kl_target)
    if target != 0.0 and beta == 0.0:
        raise ValueError("kl_target adapts the KL penalty's coefficient: it needs a kl_coef")
    return beta, target


def adapt_kl_coef(beta: float, kl_sum: float, n_ind: float, kl_target: float) -> float:
    """The PPO paper's adaptive rule (Schulman et al. 2017, section 4), in float64, on the mean KL d = kl_sum / n_ind
    (statistics slots 18 and 4 summed over the rows of an update's last epoch): halve beta when d is below
    kl_target / 1.5, double it above 1.5 * kl_target, keep it otherwise, for a NaN d and when n_ind is 0."""
    if not n_ind > 0:
        return beta
    d = float(kl_sum) / float(n_ind)
    if d < kl_target / 1.5:
        return beta / 2.0
    if d > kl_target * 1.5:
        return beta * 2.0
    return beta


def check_skip_nonfinite(skip_nonfinite) -> bool:
    """The non-finite guard's switch as a bool; ValueError for anything but a bool or 0 / 1 (a float or a string here is
    a misplaced argument, not a choice)."""
    if isinstance(skip_nonfinite, (bool, np.bool_)) or (isinstance(skip_nonfinite, (int, np.integer))
                                                        and skip_nonfinite in (0, 1)):
        return bool(skip_nonfinite)
    raise ValueError(f"Invalid skip_nonfinite value: {skip_nonfinite!r}")


def check_recompute_advantage(recompute_advantage) -> bool:
    """The switch of the per-epoch advantage recomputation as a bool; ValueError for anything but a bool or 0 / 1."""
    if isinstance(recompute_advantage, (bool, np.bool_)) or (isinstance(recompute_advantage, (int, np.integer))
                                                              and recompute_advantage in (0, 1)):
        return bool(recompute_advantage)
    raise ValueError(f"Invalid recompute_advantage value: {recompute_advantage!r}")


def check_adam_options(adam_options) -> bool:
    """The switch that reads betas, eps, amsgrad and decoupled_weight_decay as a bool; ValueError for anything but a
    bool or 0 / 1."""
    if isinstance(adam_options, (bool, np.bool_)) or (isinstance(adam_options, (int, np.integer))
                                                       and adam_options in (0, 1)):
        return bool(adam_options)
    raise ValueError(f"Invalid adam_options value: {adam_options!r}")


def check_value_norm(value_norm, beta) -> Tuple[bool, float]:
    """The value-target normalisation's switch and EMA weight as (bool, float); ValueError for a switch other than a bool
    or 0 / 1, and for a beta that is not finite or not in (0, 1).  beta is checked whether or not the switch is on."""
    if not (isinstance(value_norm, (bool, np.bool_)) or (isinstance(value_norm, (int, np.integer))
                                                          and value_norm in (0, 1))):
        raise ValueError(f"Invalid value_norm value: {value_norm!r}")
    if isinstance(beta, (bool, np.bool_)) or not isinstance(beta, (int, float, np.integer, np.floating)):
        raise ValueError(f"Invalid value_norm_beta value: {beta!r}")
    b = float(beta)
    if not (math.isfinite(b) and 0.0 < b < 1.0):
        raise ValueError(f"Invalid value_norm_beta value: {beta!r} (in (0, 1))")
    return bool(value_norm), b


def value_norm_stats(m1: float, m2: float, d: float) -> Tuple[float, float]:
    """(mean, std) of a value-target normaliser state {m1, m2, d} in float64, as the kernels form them
    (include/upb200.h: upb_set_value_norm): (0, 1) while d == 0."""
    if d == 0.0:
        return 0.0, 1.0
    dd = max(d, 1e-5)
    mu = m1 / dd
    return mu, math.sqrt(max(m2 / dd - mu * mu, 1e-2))


def check_grad_noise_every(grad_noise_every) -> Optional[int]:
    """The gradient-noise measurement's period k as an int (minibatch step i of every epoch is measured when
    i % k == 0), None meaning off; ValueError for a bool and anything that is not an integer >= 1."""
    if grad_noise_every is None:
        return None
    if isinstance(grad_noise_every, (bool, np.bool_)) or not isinstance(grad_noise_every, (int, np.integer)) \
            or grad_noise_every < 1:
        raise ValueError(f"Invalid grad_noise_every value: {grad_noise_every!r} (None or an integer >= 1)")
    return int(grad_noise_every)


def cta_group_sizes(count: int, grid: int) -> np.ndarray:
    """n_c, the number of items each CTA of a launch over `count` items takes under the kernels' static schedule: the
    launch has min(count, grid) CTAs and CTA c takes the items c, c + min(count, grid), ... (include/upb200.h:
    upb_ppo_grad_noise's Q = sum n_c^2)."""
    g = min(int(count), int(grid))
    if g <= 0:
        return np.zeros(0, np.int64)
    q, r = divmod(int(count), g)
    return np.where(np.arange(g) < r, q + 1, q).astype(np.int64)


def grad_noise_terms(noise) -> Tuple[float, float, float]:
    """(U, V, D) of gradient-noise measurements `noise` (rows {A, S, Q, N} of upb_ppo_grad_noise), summed in float64 over
    the rows: D = N^2 - Q, U = S - A (estimates D |mu|^2) and V = (N^2 A - Q S) / N (estimates D tr Sigma_x), where x_i is
    one graph's term of the summed minibatch gradient, mu its mean and Sigma_x its covariance.  A row with N = 0 (no
    sample) adds nothing.  With CTA groups of equal size this is McCandlish et al.'s two-batch estimator."""
    rows = np.asarray(noise, np.float64).reshape(-1, 4)
    U = V = D = 0.0
    for A, S, Q, N in rows.tolist():
        if N == 0.0:
            continue
        U += S - A
        V += (N * N * A - Q * S) / N
        D += N * N - Q
    return U, V, D


def grad_noise_estimate(U: float, V: float, D: float, batch: int, samples: int) -> dict:
    """The update's gradient-noise report from the (U, V, D) sums of its counted measurements over every rank:
    grad_noise_scale = V / U (B_simple = tr Sigma / |G|^2, in graphs; reported as computed, so negative or infinite when
    the mean gradient is not resolved), grad_noise_g2 = batch^2 U / D and grad_noise_trace = batch^2 V / D (|G|^2 and
    tr Sigma in the units of one graph's gradient, batch times its term), grad_noise_samples = samples.  NaN where a
    denominator is 0 and nothing counted (float64 division otherwise, so x / 0 is +-inf)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        U, V, D = np.float64(U), np.float64(V), np.float64(D)
        b2 = np.float64(batch) ** 2
        return dict(grad_noise_scale=float(V / U), grad_noise_g2=float(b2 * U / D), grad_noise_trace=float(b2 * V / D),
                    grad_noise_samples=int(samples))


def check_clip_epsilon(clip_epsilon) -> float:
    """The PPO clip epsilon as a float; ValueError for a negative or non-finite one."""
    eps = float(clip_epsilon)
    if not math.isfinite(eps) or eps < 0.0:
        raise ValueError(f"Invalid clip_epsilon value: {clip_epsilon}")
    return eps


def check_lr(lr) -> float:
    """The learning rate as a float; ValueError for a negative or non-finite one, as torch.optim.Adam raises.  0 is
    legal: the moments and step counters still advance."""
    r = float(lr)
    if not math.isfinite(r) or r < 0.0:
        raise ValueError(f"Invalid learning rate: {lr}")
    return r


def check_adam(betas, eps, amsgrad=False, decoupled_weight_decay=False) -> Tuple[float, float, float, bool, bool]:
    """torch.optim.Adam's betas, eps, amsgrad and decoupled_weight_decay as (beta1, beta2, eps, amsgrad, decoupled);
    ValueError for a tensor-valued beta or eps, a beta outside [0, 1) (also once rounded to fp32, as the kernels keep it)
    or a negative or non-finite eps."""
    if isinstance(eps, torch.Tensor) or any(isinstance(b, torch.Tensor) for b in betas):
        raise ValueError("betas and eps must be Python floats, not tensors")
    b1, b2 = (float(b) for b in betas)
    for i, b in enumerate((b1, b2)):
        if not (0.0 <= b < 1.0 and float(np.float32(b)) < 1.0):
            raise ValueError(f"Invalid beta parameter at index {i}: {b}")
    e = float(eps)
    if not math.isfinite(e) or e < 0.0:
        raise ValueError(f"Invalid epsilon value: {eps}")
    return b1, b2, e, bool(amsgrad), bool(decoupled_weight_decay)


def check_loss_coef(name: str, coef) -> float:
    """A loss coefficient (value_pred_coef, entropy_coef) as a float; ValueError for a non-finite one.  Any finite value
    is accepted, a negative one included."""
    c = float(coef)
    if not math.isfinite(c):
        raise ValueError(f"Invalid {name} value: {coef}")
    return c


def clip_range(clip_epsilon: float) -> Tuple[float, float]:
    """torch.clamp(ratio, 1.0 - eps, 1.0 + eps)'s bounds on an fp32 ratio (urban_planning_agent.py:368): each formed in
    double from the Python float and rounded once to fp32.  1.f -/+ fp32(eps) is one ulp off for 47 of the values
    eps = 0.01 ... 0.99."""
    return float(np.float32(1.0 - clip_epsilon)), float(np.float32(1.0 + clip_epsilon))


class Engine:
    def __init__(self, device, n_cap: int, e_cap: int, lr: float = 4e-4, betas=(0.9, 0.999), eps: float = 1e-5,
                 clip_epsilon: float = 0.2, value_pred_coef: float = 0.5, entropy_coef: float = 0.01,
                 clip_mode: int = _lib.CLIP_REFERENCE, grid_limit: int = 0, max_graphs: int = 1 << 20,
                 model: str = "sgnn", weight_decay: float = 0.0, diagnostics: bool = False, target_kl=None,
                 value_clip=None, max_grad_norm=None, kl_coef=None, skip_nonfinite: bool = False,
                 value_norm: bool = False, value_norm_beta: float = 0.99999, dual_clip=None, huber_delta=None,
                 desired_kl=None, lr_bounds=LR_BOUNDS, grad_noise_every=None, prox_ewma=None):
        if model not in ("sgnn", "mlp"):
            raise ValueError("model must be 'sgnn' (rl-sgnn) or 'mlp' (rl-mlp ablation)")
        # grad_noise_every: the period of the gradient-noise measurement the updater driving this engine runs
        # (PPOUpdater); the engine itself measures when ppo_grad_noise is called and configures nothing for it.  None = off
        self.grad_noise_every = check_grad_noise_every(grad_noise_every)
        # weight_decay: torch.optim.Adam's coupled L2 term (urban_planning_agent.py:145-149), for both models
        weight_decay = check_weight_decay(weight_decay)
        # target_kl: end an update at the first step whose approximate KL exceeds 1.5 * target_kl (upb_set_target_kl);
        # None or 0 = off
        target_kl = check_target_kl(target_kl)
        # value_clip: the clipped value loss of OpenAI baselines' ppo2 / CleanRL's clip_vloss with range c
        # (upb_set_value_clip); the training calls then take the pre-pass values as old_values.  None = off
        value_clip = check_value_clip(value_clip)
        # dual_clip: dual-clip PPO, the surrogate of a negative advantage bounded below by c A (upb_set_dual_clip); None =
        # off.  huber_delta: the Huber value loss 2 huber_loss(V, R, delta) in place of (V - R)^2 (upb_set_huber_delta);
        # None = off
        dual_clip = check_dual_clip(dual_clip)
        huber_delta = check_huber_delta(huber_delta)
        # prox_ewma: the EWMA proximal policy (PPO-EWMA) with weight beta (upb_set_prox_ewma): the clip's anchor is an
        # exponential moving average of the weights over optimiser steps, the behaviour policy weights the surrogate.
        # The proximal parameters must be set (init_prox_params / set_prox_params) before training.  None = off
        prox_ewma = check_prox_ewma(prox_ewma)
        # desired_kl / lr_bounds: the KL-adaptive lr of RSL-RL's adaptive schedule, decided by every optimiser step inside
        # its kernels (upb_set_adaptive_lr); None = off
        desired_kl, lr_min, lr_max = check_adaptive_lr(desired_kl, lr_bounds)
        # max_grad_norm: torch.nn.utils.clip_grad_norm_(parameters(), max_grad_norm) on every step, one global group
        # (upb_set_max_grad_norm); needs clip_mode=CLIP_NEVER.  None = off
        max_grad_norm = check_max_grad_norm(max_grad_norm, clip_mode)
        # kl_coef: the KL penalty beta * KL(pi_old || pi) on the exact categorical KL (upb_set_kl_penalty); the training
        # calls then take the pre-pass candidate log-probs as old_cand_log_probs.  None = off
        kl_coef, _ = check_kl_penalty(kl_coef)
        # skip_nonfinite: a step whose statistics count a non-finite result or whose reduced gradient is not finite
        # changes nothing and marks statistics slot 19 (upb_set_nonfinite_guard); any clip_mode.  False = off
        skip_nonfinite = check_skip_nonfinite(skip_nonfinite)
        # value_norm: the value head predicts values normalised by running return statistics with EMA weight
        # value_norm_beta (upb_set_value_norm: denormalize_values, value_norm_update).  False = off
        value_norm, value_norm_beta = check_value_norm(value_norm, value_norm_beta)
        clip_epsilon = check_clip_epsilon(clip_epsilon)
        lr = check_lr(lr)
        value_pred_coef = check_loss_coef("value_pred_coef", value_pred_coef)
        entropy_coef = check_loss_coef("entropy_coef", entropy_coef)
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
        # The Python values last passed to the library, which the setters below compare against.  The context starts
        # from upb_create's fp32 copies (lr: (double)(float)lr), so a run that never calls a setter keeps that arithmetic.
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        self.lr, self.value_pred_coef, self.entropy_coef = lr, value_pred_coef, entropy_coef
        # the clip range as the reference's torch.clamp forms it from the double epsilon (upb_create's default forms it
        # from the fp32 one)
        self.set_clip_epsilon(clip_epsilon)
        if weight_decay != 0.0:
            _lib.check(_lib.lib().upb_set_weight_decay_double(self._ctx, weight_decay), "upb_set_weight_decay_double")
        self.weight_decay = weight_decay
        # diagnostics: the step kernels also fill statistics slots 8-12 (PPO diagnostics, upb_set_diagnostics)
        if diagnostics:
            _lib.check(_lib.lib().upb_set_diagnostics(self._ctx, 1), "upb_set_diagnostics")
        self.diagnostics = bool(diagnostics)
        if target_kl != 0.0:
            _lib.check(_lib.lib().upb_set_target_kl(self._ctx, target_kl), "upb_set_target_kl")
        self.target_kl = target_kl
        if value_clip != 0.0:
            # torch.clamp(d, -c, c) with a Python float c clamps an fp32 tensor at +-fp32(c)
            _lib.check(_lib.lib().upb_set_value_clip(self._ctx, float(np.float32(value_clip))), "upb_set_value_clip")
        self.value_clip = value_clip
        if dual_clip != 0.0:
            # c * A with a Python float c and an fp32 tensor A is fp32(c) * A
            _lib.check(_lib.lib().upb_set_dual_clip(self._ctx, float(np.float32(dual_clip))), "upb_set_dual_clip")
        self.dual_clip = dual_clip
        if huber_delta != 0.0:
            # huber_loss(..., delta) compares and clamps an fp32 tensor at fp32(delta)
            _lib.check(_lib.lib().upb_set_huber_delta(self._ctx, float(np.float32(huber_delta))),
                       "upb_set_huber_delta")
        self.huber_delta = huber_delta
        if prox_ewma is not None:
            _lib.check(_lib.lib().upb_set_prox_ewma(self._ctx, 1, float(np.float32(prox_ewma))), "upb_set_prox_ewma")
        self.prox_ewma = prox_ewma
        if desired_kl != 0.0:
            _lib.check(_lib.lib().upb_set_adaptive_lr(self._ctx, desired_kl, lr_min, lr_max), "upb_set_adaptive_lr")
        self.desired_kl, self.lr_bounds = desired_kl, (lr_min, lr_max)
        if max_grad_norm != 0.0:
            # clip_grad_norm_ multiplies by an fp32 coefficient formed with fp32(max_norm)
            _lib.check(_lib.lib().upb_set_max_grad_norm(self._ctx, float(np.float32(max_grad_norm))),
                       "upb_set_max_grad_norm")
        self.max_grad_norm = max_grad_norm
        self.kl_coef = 0.0
        if kl_coef != 0.0:
            self.set_kl_coef(kl_coef)
        if skip_nonfinite:
            _lib.check(_lib.lib().upb_set_nonfinite_guard(self._ctx, 1), "upb_set_nonfinite_guard")
        self.skip_nonfinite = skip_nonfinite
        if value_norm:
            _lib.check(_lib.lib().upb_set_value_norm(self._ctx, value_norm_beta), "upb_set_value_norm")
        self.value_norm, self.value_norm_beta = value_norm, value_norm_beta
        self.n_cap, self.e_cap = n_cap, e_cap
        self.peers, self.peers_ok = 1, False          # multi-GPU fused step: see connect_peers
        # the per-tensor table last passed to set_param_groups: (lr, weight_decay, trained) tuples, None = none, and
        # its per-tensor Adam settings (check_adam tuples), None = the context's
        self.param_groups = None
        self.param_group_adam = None
        # Adam's betas, eps, amsgrad and decoupled flag last passed to set_adam (upb_create's until then)
        self.adam = (self.betas[0], self.betas[1], self.eps, False, False)
        if desired_kl != 0.0:
            # the adaptive lr starts from the Python lr itself (upb_set_adaptive_lr seeds upb_create's fp32 copy)
            self.set_lr_state([lr])

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            _lib.lib().upb_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_kl_coef(self, beta: float) -> None:
        """The KL penalty's coefficient for the steps issued from now on (upb_set_kl_penalty, rounded once to fp32);
        0 turns the penalty off.  ValueError for a negative or non-finite value."""
        b = float(beta)
        if not math.isfinite(b) or b < 0.0:
            raise ValueError(f"Invalid kl_coef value: {beta}")
        _lib.check(_lib.lib().upb_set_kl_penalty(self._ctx, b), "upb_set_kl_penalty")
        self.kl_coef = b

    def set_lr(self, lr: float) -> None:
        """Adam's learning rate for the optimiser steps issued from now on, both models (upb_set_lr).  Kept as a double,
        as torch keeps param_groups' lr: each step scales by (float)(lr / bias_correction1).  ValueError for a negative or
        non-finite value."""
        r = check_lr(lr)
        self._refuse_with_param_groups("lr")
        _lib.check(_lib.lib().upb_set_lr(self._ctx, r), "upb_set_lr")
        self.lr = r

    def set_loss_coefs(self, value_pred_coef: float, entropy_coef: float) -> None:
        """The value-loss and entropy coefficients of the training steps issued from now on, and of read_losses, both
        models (upb_set_loss_coefs, each rounded once to fp32).  ValueError for a non-finite value."""
        v = check_loss_coef("value_pred_coef", value_pred_coef)
        e = check_loss_coef("entropy_coef", entropy_coef)
        _lib.check(_lib.lib().upb_set_loss_coefs(self._ctx, v, e), "upb_set_loss_coefs")
        self.value_pred_coef, self.entropy_coef = v, e

    def set_clip_epsilon(self, clip_epsilon: float) -> None:
        """The surrogate's clip epsilon for the training steps issued from now on: the bounds clip_range() forms, as
        torch.clamp(ratio, 1.0 - eps, 1.0 + eps) does (upb_set_clip_range).  ValueError for a negative or non-finite
        value."""
        eps = check_clip_epsilon(clip_epsilon)
        lo_hi = clip_range(eps)
        _lib.check(_lib.lib().upb_set_clip_range(self._ctx, *lo_hi), "upb_set_clip_range")
        self.clip_epsilon, self.clip_range = eps, lo_hi

    def set_weight_decay(self, weight_decay: float) -> None:
        """Adam's weight decay for the optimiser steps issued from now on, both models (upb_set_weight_decay_double: the
        coupled L2 term rounded once to fp32, set_adam's decoupled factor formed from the double).  ValueError for a
        negative or non-finite value."""
        wd = check_weight_decay(weight_decay)
        self._refuse_with_param_groups("weight_decay")
        _lib.check(_lib.lib().upb_set_weight_decay_double(self._ctx, wd), "upb_set_weight_decay_double")
        self.weight_decay = wd

    def set_adam(self, betas, eps: float, amsgrad: bool = False, decoupled_weight_decay: bool = False) -> None:
        """Adam's betas, eps, AMSGrad and decoupled weight decay (torch.optim.AdamW) for the optimiser steps issued from
        now on, both models (upb_set_adam).  At the engine's own betas and eps, coupled and without AMSGrad, the steps
        are exactly those of an engine that never called it.  ValueError (check_adam) before any CUDA call, and while
        the engine has parameter groups, whose groups carry these settings."""
        adam = check_adam(betas, eps, amsgrad, decoupled_weight_decay)
        self._refuse_with_param_groups("Adam settings")
        _lib.check(_lib.lib().upb_set_adam(self._ctx, adam[0], adam[1], adam[2], int(adam[3]), int(adam[4])),
                   "upb_set_adam")
        self.adam = adam

    def lr_state_count(self) -> int:
        """Entries of the KL-adaptive lr state this engine reads and writes: one per tensor with parameter groups, else 1."""
        return len(self.layout.slots) if self.param_groups is not None else 1

    def read_lr_state_async(self, out: torch.Tensor) -> torch.Tensor:
        """Queue a copy of the KL-adaptive lr state the next optimiser step reads (lr_state_count() float64 values) into
        `out`, a pinned CPU float64 tensor, on the current stream (upb_get_lr_state); read it after the stream gets
        there.  Needs desired_kl."""
        name = self._p + "get_lr_state"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, out.data_ptr(), out.numel(), self._stream()), name)
        return out

    def get_lr_state(self) -> np.ndarray:
        """The KL-adaptive lr state (float64[lr_state_count()], slot order with parameter groups).  Synchronises the
        stream."""
        out = torch.zeros(self.lr_state_count(), dtype=torch.float64, pin_memory=True)
        self.read_lr_state_async(out)
        torch.cuda.current_stream(self.device).synchronize()
        return out.numpy().copy()

    def set_lr_state(self, lr) -> None:
        """Restore the KL-adaptive lr state: 1 value, or one per tensor with parameter groups (check_lr each), in stream
        order.  Needs desired_kl."""
        v = np.ascontiguousarray(lr, np.float64).reshape(-1)
        if v.size not in (1, self.lr_state_count()):
            raise ValueError(f"lr state: need 1 or {self.lr_state_count()} values, got {v.size}")
        for x in v:
            check_lr(x)
        name = self._p + "set_lr_state"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, v.ctypes.data, v.size, self._stream()), name)
        # the Python lrs follow the state, so that an unchanged live lr issues no set_lr / set_param_groups call
        if self.param_groups is not None:
            vals = v.tolist() * (self.lr_state_count() if v.size == 1 else 1)
            self.param_groups = (tuple(vals),) + tuple(self.param_groups[1:])
        else:
            self.lr = float(v[0])

    def init_prox_params(self, params: torch.Tensor) -> None:
        """theta_prox <- params (the model's flat fp32 parameters on this device), queued on the current stream."""
        if params.dtype != torch.float32 or params.device != self.device or params.numel() < self.num_params \
                or not params.is_contiguous():
            raise ValueError(f"init_prox_params: need contiguous float32 params on {self.device}")
        name = self._p + "init_prox_params"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, params.data_ptr(), self._stream()), name)

    def get_prox_params(self) -> np.ndarray:
        """theta_prox (float32[num_params]); UpbError while it was never set.  Synchronises the device."""
        out = np.zeros(self.num_params, np.float32)
        name = self._p + "get_prox_params"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, out.ctypes.data, out.size), name)
        return out

    def set_prox_params(self, prox) -> None:
        """Restore theta_prox from a host copy of num_params floats."""
        v = np.ascontiguousarray(prox, np.float32).reshape(-1)
        if v.size != self.num_params:
            raise ValueError(f"prox params: need {self.num_params} values, got {v.size}")
        name = self._p + "set_prox_params"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, v.ctypes.data, v.size), name)

    def get_amsgrad_state(self) -> Optional[np.ndarray]:
        """AMSGrad's max_exp_avg_sq (float32[num_params]), None while no tensor has had amsgrad.  Synchronises."""
        name = self._p + "get_amsgrad_state"
        has = getattr(_lib.lib(), name)(self._ctx, None, self.num_params)       # 1 / 0: whether the buffer exists
        _lib.check(min(has, 0), name)
        if not has:
            return None
        out = np.zeros(self.num_params, np.float32)
        _lib.check(getattr(_lib.lib(), name)(self._ctx, out.ctypes.data, out.size), name)
        return out

    def set_amsgrad_state(self, vmax) -> None:
        """Restore AMSGrad's max_exp_avg_sq (num_params values).  Synchronises."""
        v = np.ascontiguousarray(vmax, np.float32).reshape(-1)
        if v.size != self.num_params:
            raise ValueError(f"max_exp_avg_sq: need {self.num_params} values, got {v.size}")
        name = self._p + "set_amsgrad_state"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, v.ctypes.data, v.size), name)

    def _refuse_with_param_groups(self, what: str) -> None:
        if getattr(self, "param_groups", None) is not None:
            raise ValueError(f"this engine has parameter groups (set_param_groups), which set each tensor's {what}")

    # ---- parameter groups (include/upb200.h: upb_set_param_groups) ---------------------------------------------------
    @property
    def layout(self) -> "PL.Layout":
        return PL.MLP if self.model == "mlp" else PL.SGNN

    def set_param_groups(self, lr, weight_decay, trained, adam=None) -> None:
        """Per-tensor Adam settings for the optimiser steps issued from now on (upb_set_param_groups): one lr, weight
        decay and trained flag per tensor, in the layout's slot order (32 SGNN / 18 rl-mlp tensors).  A frozen tensor
        (trained false) gets no Adam step and a zero gradient column; each trained one steps with its own lr, weight decay
        and step count.  adam: one (beta1, beta2, eps, amsgrad, decoupled) per tensor (upb_set_param_groups_adam; the
        weight decays are then passed as doubles), None = every tensor at the engine's settings (set_adam).  Once set,
        set_lr, set_weight_decay and set_adam raise ValueError.  ValueError, before any CUDA call, for a table of another
        length, an invalid lr, weight decay or Adam setting (check_lr, check_weight_decay, check_adam), no trained tensor,
        or a frozen val_w2 / val_b2 while value_norm is on (its rescale writes them every update).  Synchronises the
        device."""
        names = list(self.layout.slots)
        lr, weight_decay, trained = list(lr), list(weight_decay), list(trained)
        if not len(lr) == len(weight_decay) == len(trained) == len(names):
            raise ValueError(f"parameter groups: need {len(names)} values of lr, weight_decay and trained (one per "
                             f"tensor), got {len(lr)}, {len(weight_decay)}, {len(trained)}")
        lr = tuple(check_lr(x) for x in lr)
        weight_decay = tuple(check_weight_decay(x) for x in weight_decay)
        trained = tuple(bool(x) for x in trained)
        if adam is not None:
            adam = list(adam)
            if len(adam) != len(names):
                raise ValueError(f"parameter groups: need {len(names)} Adam settings (one per tensor), got {len(adam)}")
            adam = tuple(check_adam(a[:2], *a[2:]) for a in adam)
        if not any(trained):
            raise ValueError("parameter groups: no tensor is trained")
        if self.value_norm:
            frozen = [n for n in ("val_w2", "val_b2") if not trained[names.index(n)]]
            if frozen:
                raise ValueError(f"value_norm rescales {' and '.join(frozen)} every update: they cannot be frozen")
        n = len(names)
        lr_c = (C.c_double * n)(*lr)
        tr_c = (C.c_uint8 * n)(*trained)
        if adam is None:
            wd_c = (C.c_float * n)(*weight_decay)
            name = self._p + "set_param_groups"
            _lib.check(getattr(_lib.lib(), name)(self._ctx, lr_c, wd_c, tr_c, n), name)
        else:
            col = lambda k, ty: (ty * n)(*[a[k] for a in adam])
            name = self._p + "set_param_groups_adam"
            _lib.check(getattr(_lib.lib(), name)(self._ctx, lr_c, (C.c_double * n)(*weight_decay), tr_c,
                                                 col(0, C.c_float), col(1, C.c_float), col(2, C.c_float),
                                                 col(3, C.c_uint8), col(4, C.c_uint8), n), name)
        self.param_groups = (lr, weight_decay, trained)
        self.param_group_adam = adam

    def get_tensor_steps(self) -> np.ndarray:
        """Each tensor's Adam step count (int64, slot order); needs a table (set_param_groups).  Synchronises."""
        out = np.zeros(len(self.layout.slots), np.int64)
        name = self._p + "get_tensor_steps"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, out.ctypes.data, out.size), name)
        return out

    def set_tensor_steps(self, steps) -> None:
        """Restore each tensor's Adam step count (slot order, >= 0); needs a table (set_param_groups)."""
        st = np.ascontiguousarray(steps, np.int64).reshape(-1)
        if st.size != len(self.layout.slots) or (st < 0).any():
            raise ValueError(f"tensor steps: need {len(self.layout.slots)} counts >= 0")
        name = self._p + "set_tensor_steps"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, st.ctypes.data, st.size), name)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _check_blob(self, blob: PackedGraphs):
        if blob.n_cap > self.n_cap or blob.e_cap > self.e_cap:
            raise _lib.UpbError(f"blob caps ({blob.n_cap},{blob.e_cap}) exceed the engine's ({self.n_cap},{self.e_cap})")

    # ------------------------------------------------------------------ no-grad passes
    def forward(self, blob: PackedGraphs, params: torch.Tensor, actions: Optional[torch.Tensor] = None,
                ids: Optional[torch.Tensor] = None, want_greedy: bool = False, cand_log_probs: bool = False):
        """value, log_prob, entropy (and greedy action index) per graph of the blob, each shaped (count,).
        Outputs are indexed by blob position; entries not listed in `ids` are left untouched (zero).  cand_log_probs:
        also return every candidate's log-probability, (blob.cand_len,) indexed by candidate position
        (upb_forward_cand), last in the tuple."""
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
        cand = torch.zeros(blob.cand_len, dtype=torch.float32, device=dev) if cand_log_probs else None
        name = self._p + ("forward_cand" if cand_log_probs else "forward")
        extra = (cand.data_ptr(),) if cand_log_probs else ()
        _lib.check(getattr(_lib.lib(), name)(self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(),
                                             _ptr(actions), value.data_ptr(), logp.data_ptr(), ent.data_ptr(),
                                             _ptr(greedy), *extra, self._stream()), name)
        out = (value, logp, ent) + ((greedy,) if want_greedy else ())
        return out + (cand,) if cand_log_probs else out

    def values(self, blob: PackedGraphs, params: torch.Tensor, ids: Optional[torch.Tensor] = None,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The value of every graph `ids` (all if None) from a value-only sweep (upb_values): forward(...)[0] bit for bit,
        without the policy heads.  (count,) float32 indexed by blob position; entries not listed in `ids` keep the values
        of `out` (zeros when None).  With value_norm on, the head's normalised outputs.  One launch, no
        synchronisation."""
        self._check_blob(blob)
        assert params.numel() == self.num_params, "flat parameter vector of the wrong model"
        if out is None:
            out = torch.zeros(blob.count, dtype=torch.float32, device=self.device)
        assert (out.dtype == torch.float32 and out.is_contiguous() and out.numel() == blob.count
                and out.device == self.device)
        cnt = blob.count if ids is None else int(ids.numel())
        name = self._p + "values"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(),
                                             out.data_ptr(), self._stream()), name)
        return out

    def policy_logits(self, blob: PackedGraphs, params: torch.Tensor, ids: Optional[torch.Tensor] = None):
        """The masked logits of both policy heads (policy.py:45-65, upb_policy_logits): (land_use, road, stage).
        land_use is (B0, e_cap) and road (B1, n_cap) float32 on the device, or None for a stage without a graph; the
        widths are this engine's caps.  Row r of a matrix belongs to the r-th graph of that stage in `ids` order (blob
        order when None), as the reference's x[stage[:, s].bool()]: -2^32+1 except at the mask-true candidates, which
        hold their logits, and NaN for a graph larger than the engine's caps.  stage: (count,) int32 numpy, the stage
        (0 land use, 1 road) of every graph of the blob.  Rows and shapes come from the host copy of the blob, so with
        ids None the call does not synchronise with the device."""
        self._check_blob(blob)
        assert params.numel() == self.num_params, "flat parameter vector of the wrong model"
        stage = blob.info[:, 3].copy()
        order = np.arange(blob.count) if ids is None else ids.cpu().numpy().astype(np.int64)
        rows = np.full(blob.count, -1, np.int32)
        out = []
        for s, width in ((0, self.e_cap), (1, self.n_cap)):
            mine = order[stage[order] == s]
            rows[mine] = np.arange(mine.size, dtype=np.int32)
            out.append(torch.empty(mine.size, width, dtype=torch.float32, device=self.device) if mine.size else None)
        rows_d = torch.from_numpy(rows).pin_memory().to(self.device, non_blocking=True)
        cnt = blob.count if ids is None else int(ids.numel())
        _lib.check(getattr(_lib.lib(), self._p + "policy_logits")(
            self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(), rows_d.data_ptr(), _ptr(out[0]),
            _ptr(out[1]), self._stream()), self._p + "policy_logits")
        return out[0], out[1], stage

    # ------------------------------------------------------------------ training step pieces
    def new_grad_buffer(self) -> torch.Tensor:
        return torch.zeros(self.grad_stride, dtype=torch.float32, device=self.device)

    def ppo_grad(self, blob: PackedGraphs, params: torch.Tensor, actions: torch.Tensor, advantages: torch.Tensor,
                 returns: torch.Tensor, fixed_log_probs: torch.Tensor, exps: torch.Tensor, inv_batch: float,
                 inv_ind: float, ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                 old_values: Optional[torch.Tensor] = None,
                 old_cand_log_probs: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Gradient of the PPO loss of the graphs `ids` (all if None) w.r.t. the flat parameters, plus the loss
        statistics, in one flat buffer (see upb200.h).  Per-sample arrays are indexed by blob position; old_values are
        the pre-pass values the clipped value loss needs (required while value_clip is set, ignored otherwise);
        old_cand_log_probs the pre-pass candidate log-probs of forward(cand_log_probs=True) the KL penalty needs
        (required while kl_coef is set, ignored otherwise)."""
        return self._train_call("ppo_grad", blob, params, actions, advantages, returns, fixed_log_probs, exps,
                                inv_batch, inv_ind, ids, out, old_values, old_cand_log_probs)

    def _train_call(self, what, blob, params, actions, advantages, returns, fixed_log_probs, exps, inv_batch, inv_ind,
                    ids, out, old_values, old_cand_log_probs=None):
        self._check_blob(blob)
        dev = self.device
        if out is None:
            out = self.new_grad_buffer()
        cnt = blob.count if ids is None else int(ids.numel())
        # without reference data the entry points of a context that never clips its value loss (upb_ppo_grad, ...);
        # with the candidate log-probs upb_step_refs (upb_ppo_grad_refs, ...)
        ov_t = None if old_values is None else _f32(old_values.reshape(-1), dev)
        if old_cand_log_probs is not None:
            oc_t = _f32(old_cand_log_probs.reshape(-1), dev)
            if oc_t.numel() < blob.cand_len:
                raise ValueError(f"old_cand_log_probs must hold blob.cand_len = {blob.cand_len} values")
            refs = _lib.StepRefs(_ptr(ov_t), oc_t.data_ptr())
            ov, name = (C.byref(refs),), self._p + what + "_refs"
        else:
            ov = () if ov_t is None else (ov_t.data_ptr(),)
            name = self._p + what + ("_vclip" if ov else "")
        _lib.check(getattr(_lib.lib(), name)(
            self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(), _f32(actions, dev).data_ptr(),
            _f32(advantages, dev).data_ptr(), _f32(returns, dev).data_ptr(), _f32(fixed_log_probs, dev).data_ptr(),
            _f32(exps, dev).data_ptr(), *ov, float(inv_batch), float(inv_ind), out.data_ptr(), self._stream()), name)
        return out

    def ppo_grad_noise(self, blob: PackedGraphs, params: torch.Tensor, actions: torch.Tensor, advantages: torch.Tensor,
                       returns: torch.Tensor, fixed_log_probs: torch.Tensor, exps: torch.Tensor, inv_batch: float,
                       inv_ind: float, ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                       noise_out: Optional[torch.Tensor] = None, old_values: Optional[torch.Tensor] = None,
                       old_cand_log_probs: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """ppo_grad of the graphs `ids` into `out`, plus the gradient-noise measurement of that launch
        (upb_ppo_grad_noise): noise_out, a device float64 tensor of 4 (None: a new one), receives {A, S, Q, N} -- the
        summed squared norms of the CTAs' partial gradients, the squared norm of the reduced gradient, the sum of the
        squared CTA group sizes (cta_group_sizes) and the graph count; {0, 0, 0, 0} while the KL stop word is set.  CTA c
        takes the graphs ids[c], ids[c + grid], ..., so pass `ids` in a random order.  Returns (out, noise_out).  Three
        launches, no synchronisation; arguments as for ppo_grad."""
        self._check_blob(blob)
        dev = self.device
        if out is None:
            out = self.new_grad_buffer()
        if noise_out is None:
            noise_out = torch.zeros(4, dtype=torch.float64, device=dev)
        if not (noise_out.dtype == torch.float64 and noise_out.is_contiguous() and noise_out.numel() == 4
                and noise_out.device == dev):
            raise ValueError("noise_out must be a contiguous float64 tensor of 4 on the engine's device")
        cnt = blob.count if ids is None else int(ids.numel())
        ov_t = None if old_values is None else _f32(old_values.reshape(-1), dev)
        oc_t = None if old_cand_log_probs is None else _f32(old_cand_log_probs.reshape(-1), dev)
        if oc_t is not None and oc_t.numel() < blob.cand_len:
            raise ValueError(f"old_cand_log_probs must hold blob.cand_len = {blob.cand_len} values")
        refs = _lib.StepRefs(_ptr(ov_t), _ptr(oc_t))
        name = self._p + "ppo_grad_noise"
        _lib.check(getattr(_lib.lib(), name)(
            self._ctx, blob.dev_ptr(), _ptr(ids), cnt, params.data_ptr(), _f32(actions, dev).data_ptr(),
            _f32(advantages, dev).data_ptr(), _f32(returns, dev).data_ptr(), _f32(fixed_log_probs, dev).data_ptr(),
            _f32(exps, dev).data_ptr(), C.byref(refs), float(inv_batch), float(inv_ind), out.data_ptr(),
            noise_out.data_ptr(), self._stream()), name)
        return out, noise_out

    def ppo_step(self, blob: PackedGraphs, params: torch.Tensor, actions: torch.Tensor, advantages: torch.Tensor,
                 returns: torch.Tensor, fixed_log_probs: torch.Tensor, exps: torch.Tensor, inv_batch: float,
                 inv_ind: float, ids: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                 old_values: Optional[torch.Tensor] = None,
                 old_cand_log_probs: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Single-GPU optimiser step in one launch (gradient + reduction + Adam, upb_ppo_step / upb_mlp_ppo_step);
        falls back to ppo_grad + apply inside the library on steps that clip.  Returns the gradient / statistics
        buffer.  old_values, old_cand_log_probs: as for ppo_grad."""
        return self._train_call("ppo_step", blob, params, actions, advantages, returns, fixed_log_probs, exps,
                                inv_batch, inv_ind, ids, out, old_values, old_cand_log_probs)

    def normalize_advantages(self, advantages: torch.Tensor, exps: torch.Tensor, order: torch.Tensor, batch: int,
                             out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Per-minibatch advantage normalisation over an epoch's sample order (upb_normalize_advantages): for each
        minibatch order[i*batch:(i+1)*batch], (A - mean) / (std + 1e-8) with mean and unbiased std over its exps != 0
        graphs, written at blob position for its graphs.  `order` is a device int32 tensor.  Entries of `out` outside
        those minibatches keep their values (`out` None: a copy of `advantages`).  One launch, no synchronisation."""
        dev = self.device
        adv = _f32(advantages.reshape(-1), dev)
        e = _f32(exps.reshape(-1), dev)
        if order.device != dev or order.dtype != torch.int32 or not order.is_contiguous():
            raise ValueError("order must be a contiguous int32 tensor on the engine's device")
        if out is None:
            out = adv.clone()
        assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() == adv.numel()
        assert out.data_ptr() != adv.data_ptr(), "out must not alias the advantages"
        _lib.check(_lib.lib().upb_normalize_advantages(self._ctx, adv.data_ptr(), e.data_ptr(), order.data_ptr(),
                                                       int(order.numel()), int(batch), out.data_ptr(),
                                                       self._stream()), "upb_normalize_advantages")
        return out

    # ---- value-target normalisation (include/upb200.h: upb_set_value_norm) ------------------------------------------
    def denormalize_values(self, normalized: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """fmaf(fp32(std), n, fp32(mean)) of the value head's normalised outputs with this model's current statistics
        (exactly n while the state is the identity).  One launch, no synchronisation."""
        n = _f32(normalized.reshape(-1), self.device)
        if out is None:
            out = torch.empty_like(n)
        assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() == n.numel()
        name = self._p + "value_norm_denormalize"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, n.data_ptr(), int(n.numel()), out.data_ptr(), self._stream()),
                   name)
        return out

    def value_norm_update(self, returns: torch.Tensor, params: torch.Tensor, values: Optional[torch.Tensor] = None):
        """One update of the running statistics from all the returns, PopArt's rescale of the value head's last layer in
        `params` (in place) and the returns (and `values`, when given) normalised with the new statistics.  Returns
        (normalised returns, normalised values or None, device float64 (2,) holding the new (mean, std)).  One launch,
        no synchronisation; needs value_norm on."""
        if not self.value_norm:
            raise ValueError("value-target normalisation is off: construct the engine with value_norm=True")
        assert params.numel() == self.num_params and params.dtype == torch.float32 and params.is_contiguous()
        r = _f32(returns.reshape(-1), self.device)
        v = None if values is None else _f32(values.reshape(-1), self.device)
        if v is not None and v.numel() != r.numel():
            raise ValueError("values must hold one value per return")
        r_out = torch.empty_like(r)
        v_out = None if v is None else torch.empty_like(v)
        mean_std = torch.empty(2, dtype=torch.float64, device=self.device)
        name = self._p + "value_norm_update"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, r.data_ptr(), _ptr(v), int(r.numel()), params.data_ptr(),
                                             r_out.data_ptr(), _ptr(v_out), mean_std.data_ptr(), self._stream()), name)
        return r_out, v_out, mean_std

    def get_value_norm_state(self) -> Tuple[float, float, float]:
        """This model's running state (m1, m2, d) as Python floats (synchronises the device)."""
        st = (C.c_double * 3)()
        name = self._p + "get_value_norm_state"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, st), name)
        return float(st[0]), float(st[1]), float(st[2])

    def set_value_norm_state(self, state) -> None:
        """Restore this model's running state (m1, m2, d); (0, 0, 0) is the identity.  ValueError for a non-finite value,
        m2 < 0 or d outside [0, 1]."""
        m1, m2, d = (float(x) for x in state)
        if not all(math.isfinite(x) for x in (m1, m2, d)) or m2 < 0.0 or not 0.0 <= d <= 1.0:
            raise ValueError(f"Invalid value-norm state: {state!r}")
        st = (C.c_double * 3)(m1, m2, d)
        name = self._p + "set_value_norm_state"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, st), name)

    def select_action(self, blob: PackedGraphs, params: torch.Tensor, uniforms: Optional[torch.Tensor] = None,
                      ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Action index per graph of the blob (int32, indexed by blob position): greedy arg-max when `uniforms` is
        None (policy.py:72-79 `mean_action`), else drawn by inverse CDF from one uniform in [0, 1) per graph
        (policy.py:81-83); a candidate of fp32 probability 0 is never drawn."""
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
        """True if the next ppo_step runs as one launch (it does not take the two-group clip; the global clip of
        max_grad_norm stays in the launch)."""
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

    def reset_kl_stop(self) -> None:
        """Clear this model's KL stop word on the current stream, so that the next steps train again."""
        _lib.check(getattr(_lib.lib(), self._p + "reset_kl_stop")(self._ctx, self._stream()), self._p + "reset_kl_stop")

    def read_losses(self, grad: torch.Tensor) -> Tuple[float, float, float, float]:
        out = (C.c_float * 4)()
        _lib.check(getattr(_lib.lib(), self._p + "read_losses")(self._ctx, grad.data_ptr(), out, self._stream()),
                   self._p + "read_losses")
        return tuple(float(x) for x in out)

    def grad_norms(self, rows: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Squared gradient norms of gradient buffers stacked as `rows` (R, grad_stride): (R, 3) float32 on the device,
        the sums of squares over the shared encoder, the policy heads and the value head (upb_grad_norms).  One launch,
        no synchronisation."""
        if rows.dim() != 2 or rows.shape[1] != self.grad_stride:
            raise ValueError(f"rows must be (R, {self.grad_stride}) gradient buffers of this model")
        rows = _f32(rows, self.device)
        n = rows.shape[0]
        if out is None:
            out = torch.empty(n, 3, dtype=torch.float32, device=self.device)
        assert out.shape == (n, 3) and out.dtype == torch.float32 and out.is_contiguous() and out.device == self.device
        _lib.check(getattr(_lib.lib(), self._p + "grad_norms")(self._ctx, rows.data_ptr(), n, out.data_ptr(),
                                                              self._stream()), self._p + "grad_norms")
        return out

    def gae(self, rewards: torch.Tensor, masks: torch.Tensor, values: torch.Tensor, gamma: float, tau: float):
        dev = self.device
        r, m, v = _f32(rewards.reshape(-1), dev), _f32(masks.reshape(-1), dev), _f32(values.reshape(-1), dev)
        T = r.numel()
        adv = torch.empty(T, dtype=torch.float32, device=dev)
        ret = torch.empty(T, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().upb_gae(self._ctx, r.data_ptr(), m.data_ptr(), v.data_ptr(), T, float(gamma),
                                      float(tau), adv.data_ptr(), ret.data_ptr(), self._stream()), "upb_gae")
        return adv, ret

    def gae_targets(self, rewards: torch.Tensor, masks: torch.Tensor, head_values: torch.Tensor, gamma: float,
                    tau: float):
        """(advantages, returns, anchors) of the raw head outputs `head_values` (values()) in one launch
        (upb_gae_targets): gae() on the values, with value_norm on denormalised with this model's current statistics and
        the returns normalised with them (neither the statistics nor the head move); anchors are the head values, the
        clipped value loss's old values.  No synchronisation."""
        dev = self.device
        r, m = _f32(rewards.reshape(-1), dev), _f32(masks.reshape(-1), dev)
        n = _f32(head_values.reshape(-1), dev)
        T = r.numel()
        if m.numel() != T or n.numel() != T:
            raise ValueError("rewards, masks and head_values must hold one value per sample")
        adv, ret, anchor = (torch.empty(T, dtype=torch.float32, device=dev) for _ in range(3))
        name = self._p + "gae_targets"
        _lib.check(getattr(_lib.lib(), name)(self._ctx, r.data_ptr(), m.data_ptr(), n.data_ptr(), T, float(gamma),
                                             float(tau), adv.data_ptr(), ret.data_ptr(), anchor.data_ptr(),
                                             self._stream()), name)
        return adv, ret, anchor

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
