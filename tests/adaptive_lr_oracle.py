"""Host mirror of the KL-adaptive learning rate (include/upb200.h: upb_set_adaptive_lr): the decision on a statistics
row's reduced slots 8 and 4 in fp32, as the kernels take it, and the new lr in float64, per tensor with parameter
groups.  RSL-RL's rule (schedule="adaptive"): with kl = slot8 / max(slot4, 1),

    kl > 2 desired_kl                -> lr = max(lr_min, lr / 1.5)
    0 < kl < desired_kl / 2          -> lr = min(lr_max, lr * 1.5)

where the kernels compare the sum with the fp32 threshold times max(slot4, 1) instead of dividing."""
import numpy as np

from drl_urban_planning_b200.engine import adapt_lr


def decision(s8, s4, desired_kl) -> int:
    """+1, -1 or 0 for one row: fp32 products and comparisons, as lr_decision (optim_kernels.cuh)."""
    s8, s4 = np.float32(s8), np.float32(s4)
    n = np.float32(max(s4, np.float32(1.0))) if not np.isnan(s4) else np.float32(1.0)
    down = np.float32(np.float32(2.0 * desired_kl) * n)
    up = np.float32(np.float32(desired_kl / 2.0) * n)
    if s8 > down:
        return -1
    if s8 > 0 and s8 < up:
        return 1
    return 0


def step(lrs, dec, bounds, trained=None):
    """Every tensor's lr after a step with decision dec that applied Adam; a frozen tensor's lr does not move."""
    trained = [True] * len(lrs) if trained is None else trained
    return [adapt_lr(x, dec, *bounds) if t else x for x, t in zip(lrs, trained)]


def replay(lrs, rows, desired_kl, bounds, applied=None, trained=None):
    """The decisions and the lrs each step applies over statistics rows (slot 8, slot 4); applied[i] False: the step
    applied nothing (its decision is 0, the lrs stay).  Returns (decisions, per-step lrs, final lrs)."""
    decs, per_step = [], []
    for i, (s8, s4) in enumerate(rows):
        d = decision(s8, s4, desired_kl) if applied is None or applied[i] else 0
        lrs = step(lrs, d, bounds, trained)
        decs.append(d)
        per_step.append(list(lrs))
    return decs, per_step, lrs
