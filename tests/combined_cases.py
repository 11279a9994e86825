"""Builders and host models of tests/test_gpu_options_combined.py: the training options used together, as
a fine-tuning run uses them -- per-tensor parameter groups with frozen tensors, value normalisation (PopArt), live
schedules of the per-group lr and the PPO coefficients, the clipped value loss, the KL penalty, advantage
normalisation, the global clip, weight decay and the non-finite guard -- on both models.

The minibatch with every PPO option is tests/ppo_oracle.py's; this module holds the parameter-group table and its
schedule, the host model of each tensor's Adam count, the element-wise Adam bar, and the rule that tells which samples
a non-finite reward reaches."""
import types

import numpy as np

import decay_oracle as DO
import scale_cases as SC
from drl_urban_planning_b200 import params as PL
from harness import reproducible_states
from oracle import sgnn_numpy as ON


# ---- the parameter-group table and its schedule ----------------------------------------------------------------------
# Frozen at the first update, the first of them trained again from the second on: none is a prefix of the layout, and
# each sits between trained tensors (gcn1_w mid-encoder, mha_out_b, lu_w1 the land-use head's last tensor; enc_b the
# rl-mlp encoder's last, val_b1 inside the value head).  val_w2 and val_b2 stay trained: value_norm rescales them.
FROZEN = {"sgnn": ["gcn1_w", "mha_out_b", "lu_w1"], "mlp": ["enc_b", "lu_w1", "val_b1"]}
LR_BASE = 2.0 ** -12


def layout_of(model):
    return PL.MLP if model == "mlp" else PL.SGNN


def base_lr(k):
    """Tensor k's lr before any schedule: 2^-12 (1 + (5k mod 16) / 16), so neighbours differ by at least 5/31."""
    return LR_BASE * (1.0 + ((5 * k) % 16) / 16.0)


def base_wd(k):
    """Tensor k's weight decay: 0 for every fourth tensor, else 2^-8 (1 + k / 16), distinct and fp32-exact."""
    return 0.0 if k % 4 == 1 else 2.0 ** -8 * (1.0 + k / 16.0)


def lr_lambda(k):
    """Tensor k's LambdaLR factor: (1 - (k mod 3) / 64)^epoch, its own per group."""
    f = 1.0 - (k % 3) / 64.0
    return lambda epoch: f ** epoch


def frozen_at(model, it):
    return FROZEN[model] if it == 0 else FROZEN[model][1:]


def groups_at(model, it):
    """One group per tensor, as PPOUpdater.set_param_groups takes them, at update `it`: each lr as LambdaLR forms it
    (base_lr * lambda(it)), a frozen tensor in no group."""
    frozen = frozen_at(model, it)
    return [dict(params=[name], lr=base_lr(k) * lr_lambda(k)(it), weight_decay=base_wd(k))
            for k, name in enumerate(layout_of(model).slots) if name not in frozen]


def table(model, it):
    """Per tensor (lr, fp32 weight decay, trained) at update `it`: what the kernels use."""
    names = list(layout_of(model).slots)
    g = {x["params"][0]: x for x in groups_at(model, it)}
    lr = np.array([g[n]["lr"] if n in g else 0.0 for n in names])
    wd = np.array([np.float32(g[n]["weight_decay"]) if n in g else 0.0 for n in names], np.float64)
    return lr, wd, np.array([n in g for n in names])


# clip_epsilon, value_pred_coef and entropy_coef changed through set_hyperparameters before the second and third update;
# the changed clip epsilons are binary fractions, so that 1 -/+ eps, the clamp's bounds, are the fp32 values the kernel
# uses (the first update's 0.2, the default, is not: fp32(1 -/+ 0.2) differ from 1 -/+ 0.2 by less than 3e-8, and a
# ratio would have to fall between the two to move the oracle's gradient)
COEFS = [dict(clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01),
         dict(clip_epsilon=0.25, value_pred_coef=0.8, entropy_coef=0.03),
         dict(clip_epsilon=0.125, value_pred_coef=0.3, entropy_coef=0.002)]


def kernel_coefs(it):
    """COEFS[it] as the kernels hold them: the loss coefficients rounded once to fp32."""
    c = COEFS[it]
    return dict(clip_epsilon=c["clip_epsilon"], value_pred_coef=float(np.float32(c["value_pred_coef"])),
                entropy_coef=float(np.float32(c["entropy_coef"])))


def seg_of(layout):
    """Each tensor's segment: 0 encoder / value, 1 land-use head, 2 road head."""
    return np.array([0 if sl.owner != "pol" else (1 if sl.name.startswith("lu_") else 2) for sl in layout.slots.values()])


def entry_table(layout, per_tensor):
    """A per-tensor array spread over the flat columns."""
    return np.repeat(np.asarray(per_tensor), [sl.size for sl in layout.slots.values()])


# ---- the host model of each tensor's Adam count ----------------------------------------------------------------------
def next_counts(counts, trained, seg, stages, skipped):
    """Each tensor's count after one step: +1 when it is trained, its segment is live (the encoder and value always, a
    policy head when a graph of its stage is in the minibatch) and the step was not skipped."""
    live = np.array([True, bool((np.asarray(stages) == 0).any()), bool((np.asarray(stages) == 1).any())])
    return np.asarray(counts) + (np.asarray(trained) & live[np.asarray(seg)] & (not skipped)).astype(np.int64)


# ---- where a non-finite reward reaches -------------------------------------------------------------------------------
def episodes(masks):
    """(first, last) of every episode: an episode ends where masks == 0, and the last one at T - 1."""
    masks = np.asarray(masks).reshape(-1)
    ends = np.flatnonzero(masks == 0)
    if not ends.size or ends[-1] != masks.size - 1:
        ends = np.r_[ends, masks.size - 1]
    return list(zip(np.r_[0, ends[:-1] + 1], ends))


def gae_per_episode(rewards, masks, values, gamma, tau):
    """ON.estimate_advantages on each episode on its own, from zero, as k_gae scans them.  For finite inputs this is
    the whole-buffer scan bit for bit (masks == 0 cuts the chain); a non-finite advantage stays in its episode here,
    where the whole-buffer scan's prev_advantage * 0 turns it into NaN for every earlier sample."""
    r, m, v = (np.asarray(x, np.float32).reshape(-1) for x in (rewards, masks, values))
    adv, ret = np.zeros(r.size, np.float32), np.zeros(r.size, np.float32)
    for a, e in episodes(m):
        x, y = ON.estimate_advantages(r[a:e + 1], m[a:e + 1], v[a:e + 1], gamma, tau)
        adv[a:e + 1], ret[a:e + 1] = x.ravel(), y.ravel()
    return adv, ret


def nonfinite_positions(rewards, masks, values, gamma, tau):
    """The samples whose advantage or return is not finite."""
    with np.errstate(invalid="ignore", over="ignore"):
        adv, ret = gae_per_episode(rewards, masks, values, gamma, tau)
    return np.flatnonzero(~(np.isfinite(adv) & np.isfinite(ret)))


def poison(ro, episode=2):
    """+inf reward at the first step of episode `episode` (an exps != 0 sample); its position."""
    pos = int(episodes(ro.masks)[episode][0])
    ro.rewards[pos] = np.inf
    ro.exps[pos] = 1.0
    return pos


# ---- rollouts --------------------------------------------------------------------------------------------------------
# (states, seed, reward scale, reward shift) of the three updates: the statistics leave the identity at the second
UPDATES = [(SC.T_PRODUCT, 41, 1.0, 0.0), (6561, 42, 30.0, 200.0), (SC.T_PRODUCT, 43, 5.0, -50.0)]


def thin_exps(ro, frac, seed):
    """exps = 0 for a further seeded `frac` of the samples."""
    ro.exps = np.where(np.random.default_rng(seed + 7).random(ro.T) < frac, 0.0, ro.exps).astype(np.float32)
    return ro


def scaled(ro, scale, shift):
    ro.rewards = (ro.rewards * np.float32(scale) + np.float32(shift)).astype(np.float32)
    return ro


def small_rollout(seed, T, scale, shift):
    """T graphs of harness.reproducible_states (rl-mlp rows reproducible run to run), episodes ended at T / 40 random
    steps, 5 % exps 0, rewards N(shift, scale^2)."""
    states, actions = reproducible_states(seed, T)
    rng = np.random.default_rng(seed)
    masks = np.ones(T, np.float32)
    masks[rng.choice(T - 1, T // 40, replace=False)] = 0.0
    exps = np.where(rng.random(T) < 0.05, 0.0, 1.0).astype(np.float32)
    rewards = (rng.standard_normal(T) * scale + shift).astype(np.float32)
    return types.SimpleNamespace(T=T, states=states, actions=actions, rewards=rewards, masks=masks, exps=exps)


# ---- instrumenting the update ----------------------------------------------------------------------------------------
class Recorder(SC.Recorder):
    """scale_cases.Recorder that also snapshots engine.get_tensor_steps(): tsteps[0] before the first step, tsteps[k + 1]
    after step k."""

    def __init__(self, up, sample, nb):
        super().__init__(up, sample, nb)
        self.tsteps = [up.engine.get_tensor_steps()]

    def step(self, ids, global_batch, global_ind):
        super().step(ids, global_batch, global_ind)
        self.tsteps.append(self.up.engine.get_tensor_steps())


# ---- the element-wise Adam bar ---------------------------------------------------------------------------------------
# A step delta = x1 - x0 (exact in float64) is checked element by element against delta64, the float64 step:
# |delta - delta64| <= 2 ulp(x1) + 1e-4 |delta64|.  For the first moment delta64 is one float64 Adam step from the
# fp32 state before the step (the weight decay enters here); for the parameters it is formed from the kernel's own new
# moments (param_step_want: each element's lr and count enter here).  The 2 ulp are the rounding of x1 itself and of
# the fp32 step; 1e-4 covers the fp32 arithmetic, the fp32 clip coefficient and step size, and the second moment's
# weight 1 - fp32(beta2) (1.29e-5 relative in v, so 6.5e-6 in the step; see V_BAR).  A wrong lr moves delta by the
# lr's error: 1/32 = 3e-2 relative, tens to hundreds of times the bar on a typical element.
ELEM_RTOL, ELEM_ULPS = 1e-4, 2.0


def elem_excess(got1, got0, want1):
    """Per element (|delta - delta64|) / (2 ulp(got1) + 1e-4 |delta64|): above 1 fails the bar."""
    got1, got0, want1 = (np.asarray(x, np.float64) for x in (got1, got0, want1))
    d, d64 = got1 - got0, want1 - got0
    ulp = np.spacing(np.abs(got1).astype(np.float32)).astype(np.float64)
    return np.abs(d - d64) / (ELEM_ULPS * ulp + ELEM_RTOL * np.abs(d64))


def elem_excess_v(got, want, vbar):
    """Per element |v - v64| / (vbar |v64| + 2 ulp(v)): above 1 fails."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    ulp = np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)
    return np.abs(got - want) / (vbar * np.abs(want) + ELEM_ULPS * ulp)


def param_step_want(p0, m1, v1, t, live, lr, b1=0.9, b2=0.999, eps=1e-5):
    """The parameter step in float64 from the kernel's own new moments (checked on their own): each element's error is
    then the step's arithmetic alone, not a small first moment's rounding, which after a cancelling update can be
    large relative to the moment."""
    p0, m1, v1 = (np.asarray(x, np.float64) for x in (p0, m1, v1))
    tt = np.maximum(np.asarray(t, np.float64) + live, 1)
    step = lr / (1 - b1 ** tt)
    return np.where(live, p0 - step * m1 / (np.sqrt(v1) / np.sqrt(1 - b2 ** tt) + eps), p0)


def adam_want(before, grad, live, lr, wd, t):
    """decay_oracle.adam_step with per-entry lr, weight decay and counts."""
    p0, m0, v0 = before
    return DO.adam_step(p0, m0, v0, t, grad, live, wd, lr=lr)
