"""Drop-in for the update half of `UrbanPlanningAgent` (reference urban_planning/agents/urban_planning_agent.py).

Usage in the reference tree (see INTEGRATION.md):

    from drl_urban_planning_b200.agent import use_b200_update
    agent = UrbanPlanningAgent(cfg, dtype, device, num_threads, ...)      # unchanged reference constructor
    use_b200_update(agent)                                                 # update_params now runs on the H100 path

`use_b200_update` replaces `agent.update_params` (reference :248-271, which calls estimate_advantages and
update_policy :281-361).  Sampling (`sample_worker`), evaluation, logging and checkpointing stay the reference's;
after every update the new weights are written back into `agent.actor_critic_net` so `save_checkpoint` /
`sample` see them.  `estimate_advantages` is also exported with the reference's signature.
"""
from __future__ import annotations

import time
from typing import Optional

import numpy as np
import torch

from . import _lib, params as PL
from .ppo import PPOUpdater


def estimate_advantages(rewards, masks, values, gamma, tau, engine=None):
    """khrylib/rl/core/common.py:5-26 on the GPU: rewards (T,), masks (T,), values (T,1) -> (T,1), (T,1) on the
    input's device.  Bit-identical to the reference's sequential fp32 scan (tests/test_gpu_parity.py)."""
    from .engine import Engine
    device = rewards.device
    if engine is None:
        dev = device if device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        engine = _default_engine(dev)
    adv, ret = engine.gae(rewards, masks, values, gamma, tau)
    return adv.reshape(-1, 1).to(device), ret.reshape(-1, 1).to(device)


# Adam keys other than lr and weight_decay that change the arithmetic, and the value each takes when the engine was built
# with `betas` and `eps` (foreach, fused, capturable and differentiable choose an implementation, not the result)
def _fixed_adam_keys(betas, eps):
    return dict(betas=tuple(float(b) for b in betas), eps=float(eps), amsgrad=False, maximize=False,
                decoupled_weight_decay=False)


def _check_fixed_adam_keys(groups, betas, eps):
    fixed = _fixed_adam_keys(betas, eps)
    for g in groups:
        for key, want in fixed.items():
            if key not in g:
                continue
            got = g[key]
            got = tuple(float(b) for b in got) if key == "betas" else (float(got) if key == "eps" else bool(got))
            if got != want:
                raise ValueError(f"agent.optimizer's {key} is {g[key]!r}, the H100 update was built with {want!r}: only "
                                 "lr and weight_decay may change between updates")


def _optimizer_values(optimizer, betas, eps, adam_options: bool = False):
    """(lr, weight_decay) of `optimizer`'s param_groups, where torch.optim.Adam.step reads them; ValueError when the
    groups disagree on either or, with adam_options off, when a group holds another Adam setting than the engine was
    built with."""
    groups = optimizer.param_groups
    if not adam_options:
        _check_fixed_adam_keys(groups, betas, eps)
    out = []
    for key in ("lr", "weight_decay"):
        vals = [float(g.get(key, 0.0)) for g in groups]
        if not np.array_equal(vals, [vals[0]] * len(vals), equal_nan=True):     # a NaN everywhere is set_lr's to refuse
            raise ValueError(f"agent.optimizer's param_groups disagree on {key} ({vals}): the H100 update trains every "
                             "parameter with one value")
        out.append(vals[0])
    return out[0], out[1]


def _check_adam_optimizer(optimizer) -> None:
    """adam_options reads torch.optim.Adam's keys: ValueError for another optimizer (AdamW is an Adam)."""
    if not isinstance(optimizer, torch.optim.Adam):
        raise ValueError(f"adam_options needs agent.optimizer to be a torch.optim.Adam or AdamW, not "
                         f"{type(optimizer).__name__}")


def _group_adam(g, i, betas, eps) -> tuple:
    """Group i's (beta1, beta2, eps, amsgrad, decoupled_weight_decay) as torch.optim.Adam.step reads them (a missing
    key: the engine's betas / eps, False); ValueError for maximize=True or an invalid value (engine.check_adam)."""
    from .engine import check_adam
    if g.get("maximize", False):
        raise ValueError(f"agent.optimizer.param_groups[{i}] has maximize=True: the H100 update minimises the loss")
    try:
        return check_adam(g.get("betas", betas), g.get("eps", eps), g.get("amsgrad", False),
                          g.get("decoupled_weight_decay", False))
    except ValueError as e:
        raise ValueError(f"agent.optimizer.param_groups[{i}]: {e}") from None


def _optimizer_adam(optimizer, betas, eps) -> dict:
    """adam_options: the Adam settings every group of `optimizer` holds, as keywords of
    PPOUpdater.set_hyperparameters; ValueError, naming the key, when the groups disagree on one."""
    _check_adam_optimizer(optimizer)
    vals = [_group_adam(g, i, betas, eps) for i, g in enumerate(optimizer.param_groups)]
    out = {}
    for k, key in enumerate(("betas", "eps", "amsgrad", "decoupled_weight_decay")):
        got = [(v[0], v[1]) if key == "betas" else v[k + 1] for v in vals]
        if any(x != got[0] for x in got):
            raise ValueError(f"agent.optimizer's param_groups disagree on {key} ({got}): without param_groups the H100 "
                             "update trains every parameter with one value")
        out[key] = got[0]
    return out


def live_param_groups(agent, layout, betas=(0.9, 0.999), eps=None, adam_options: bool = False) -> list:
    """agent.optimizer's param_groups as the tensors torch.optim.Adam.step would train, for PPOUpdater.set_param_groups:
    one {"params": [slot names], "lr", "weight_decay"} per group, holding its tensors with requires_grad=True.  The
    Parameters map to the flat layout's slots through agent.actor_critic_net.named_parameters(), whose names are
    state_dict_keys(slot)[0].  ValueError, naming the tensor or the key, for a parameter of the optimizer that is not
    one of agent.actor_critic_net's, a parameter with requires_grad=True in no group (torch would accumulate its .grad
    across steps, as zero_grad never clears it), no trained tensor, groups with another betas / eps / amsgrad / maximize
    / decoupled_weight_decay than the engine's (eps None = cfg.eps), and an invalid lr or weight_decay in any group.
    adam_options: each group also carries its "betas", "eps", "amsgrad" and "decoupled_weight_decay" (_group_adam),
    and ValueError for an optimizer that is not a torch.optim.Adam and for maximize=True instead."""
    from .engine import check_lr, check_weight_decay
    opt = getattr(agent, "optimizer", None)
    if opt is None:
        raise ValueError("param_groups reads agent.optimizer's param_groups: the agent has no optimizer")
    eps = agent.cfg.eps if eps is None else eps
    if adam_options:
        _check_adam_optimizer(opt)
    else:
        _check_fixed_adam_keys(opt.param_groups, betas, eps)
    by_key = {PL.state_dict_keys(sl)[0]: sl.name for sl in layout.slots.values()}
    slot_of, named = {}, []
    for key, p in agent.actor_critic_net.named_parameters():
        if key not in by_key:
            raise ValueError(f"agent.actor_critic_net's parameter {key!r} is not in the flat layout")
        slot_of[id(p)] = by_key[key]
        named.append((key, p))
    out, grouped = [], set()
    for i, g in enumerate(opt.param_groups):
        try:
            lr = check_lr(g["lr"])
            wd = check_weight_decay(g.get("weight_decay", 0.0))
        except ValueError as e:
            raise ValueError(f"agent.optimizer.param_groups[{i}]: {e}") from None
        names = []
        for p in g["params"]:
            if id(p) not in slot_of:
                raise ValueError(f"agent.optimizer.param_groups[{i}] holds a parameter of shape {tuple(p.shape)} that is "
                                 "not one of agent.actor_critic_net's")
            grouped.add(id(p))
            if p.requires_grad:
                names.append(slot_of[id(p)])
        out.append(dict(params=names, lr=lr, weight_decay=wd))
        if adam_options:
            b1, b2, e, ams, dec = _group_adam(g, i, betas, eps)
            out[-1].update(betas=(b1, b2), eps=e, amsgrad=ams, decoupled_weight_decay=dec)
    for key, p in named:
        if p.requires_grad and id(p) not in grouped:
            raise ValueError(f"{key} has requires_grad=True but is in no group of agent.optimizer: freeze it with "
                             "requires_grad_(False) or add it to a group")
    if not any(g["params"] for g in out):
        raise ValueError("agent.optimizer trains no tensor: every parameter of its groups has requires_grad=False")
    return out


def live_hyperparameters(agent, betas=(0.9, 0.999), eps=None, param_groups: bool = False,
                         adam_options: bool = False) -> dict:
    """The hyperparameters the reference's update_params / update_policy read from the agent at the top of an update
    (urban_planning_agent.py:248-361): lr and weight_decay from agent.optimizer.param_groups (see _optimizer_values;
    `betas` and `eps` are the engine's, eps None = cfg.eps), clip_epsilon, value_pred_coef, entropy_coef, gamma, tau,
    opt_num_epochs and mini_batch_size from the agent's attributes.  Each falls back to the cfg when the agent lacks it.
    Keyword arguments of PPOUpdater.set_hyperparameters.  param_groups: leave lr and weight_decay out (they come per
    tensor from live_param_groups).  adam_options (without param_groups): also betas, eps, amsgrad and
    decoupled_weight_decay, on which every group must agree (_optimizer_adam)."""
    cfg = agent.cfg
    opt = getattr(agent, "optimizer", None)
    if param_groups:
        out = {}
    else:
        if opt is not None:
            lr, wd = _optimizer_values(opt, betas, cfg.eps if eps is None else eps, adam_options)
        else:
            lr, wd = cfg.lr, getattr(cfg, "weightdecay", 0.0)
        out = dict(lr=lr, weight_decay=wd)
        if adam_options and opt is not None:
            out.update(_optimizer_adam(opt, betas, cfg.eps if eps is None else eps))
    for name, cfg_name in (("clip_epsilon", "clip_epsilon"), ("value_pred_coef", "value_pred_coef"),
                           ("entropy_coef", "entropy_coef"), ("gamma", "gamma"), ("tau", "tau"),
                           ("opt_num_epochs", "num_optim_epoch"), ("mini_batch_size", "mini_batch_size")):
        out[name] = getattr(agent, name) if hasattr(agent, name) else getattr(cfg, cfg_name)
    return out


_ENGINES = {}


def _default_engine(dev):
    from .engine import Engine
    key = (dev.type, dev.index)
    if key not in _ENGINES:
        _ENGINES[key] = Engine(dev, 64, 64)
    return _ENGINES[key]


class B200Update:
    """Owns the PPOUpdater of one agent and mirrors the weights between it and the agent's torch modules."""

    def __init__(self, agent, clip_mode: int = _lib.CLIP_REFERENCE, process_group="auto", device=None,
                 diagnostics: bool = False, target_kl=None, value_clip=None, normalize_advantage: bool = False,
                 max_grad_norm=None, kl_coef=None, kl_target=None, skip_nonfinite: bool = False,
                 value_norm: bool = False, value_norm_beta: float = 0.99999, param_groups: bool = False,
                 recompute_advantage: bool = False, adam_options: bool = False, dual_clip=None, huber_delta=None,
                 desired_kl=None, lr_bounds=None, grad_noise_every=None, prox_ewma=None):
        cfg = agent.cfg
        self.agent = agent
        dev = torch.device(device) if device is not None else agent.device
        if dev.type != "cuda":
            raise _lib.UpbError("use_b200_update needs agent.device to be a CUDA device (train.py --use_nvidia_gpu)")
        # everything the kernels are specialised for is checked BEFORE a CUDA context / updater is built
        # (heads = 2 or another layer count has the same flat shapes but different maths)
        kind = getattr(cfg, "agent", "rl-sgnn")
        if kind == "rl-sgnn":
            from .model import _check_specs
            _check_specs(cfg)
            self.layout, model = PL.SGNN, "sgnn"
        elif kind == "rl-mlp":                     # the ablation agent of train.py:18 (models/model.py:22-33)
            from .mlp import _check_mlp_specs
            _check_mlp_specs(cfg)
            self.layout, model = PL.MLP, "mlp"
        else:
            raise NotImplementedError(f"agent '{kind}' has no learned update (rule / GA baselines)")
        from .engine import (check_adam_options, check_adaptive_lr, check_clip_epsilon, check_dual_clip, check_huber_delta,
                             check_grad_noise_every, check_kl_penalty, check_max_grad_norm, check_prox_ewma,
                             check_recompute_advantage, check_skip_nonfinite,
                             check_target_kl, check_value_clip, check_value_norm, check_weight_decay)
        weight_decay = check_weight_decay(getattr(cfg, "weightdecay", 0.0))    # Adam's weight_decay (:145-149)
        check_target_kl(target_kl)
        # keyword arguments, not cfg keys: the reference would ignore such a key and train the same yaml differently
        check_value_clip(value_clip)
        check_dual_clip(dual_clip)
        check_huber_delta(huber_delta)
        check_adaptive_lr(desired_kl, lr_bounds)
        check_grad_noise_every(grad_noise_every)
        check_prox_ewma(prox_ewma)
        check_max_grad_norm(max_grad_norm, clip_mode)
        check_kl_penalty(kl_coef, kl_target)
        check_skip_nonfinite(skip_nonfinite)
        check_value_norm(value_norm, value_norm_beta)
        check_recompute_advantage(recompute_advantage)
        if check_adam_options(adam_options) and getattr(agent, "optimizer", None) is not None:
            _check_adam_optimizer(agent.optimizer)
        check_clip_epsilon(cfg.clip_epsilon)
        se = cfg.state_encoder_specs
        self.updater = PPOUpdater(
            self.layout.from_state_dict(agent.actor_critic_net.state_dict()), se["max_num_nodes"], se["max_num_edges"], dev,
            lr=cfg.lr, eps=cfg.eps, clip_epsilon=cfg.clip_epsilon, value_pred_coef=cfg.value_pred_coef,
            entropy_coef=cfg.entropy_coef, gamma=cfg.gamma, tau=cfg.tau, opt_num_epochs=cfg.num_optim_epoch,
            mini_batch_size=cfg.mini_batch_size, clip_mode=clip_mode, process_group=process_group,
            batch_stage=bool(cfg.agent_specs.get("batch_stage", False)), model=model, weight_decay=weight_decay,
            diagnostics=diagnostics, target_kl=target_kl, value_clip=value_clip,
            normalize_advantage=normalize_advantage, max_grad_norm=max_grad_norm, kl_coef=kl_coef,
            kl_target=kl_target, skip_nonfinite=skip_nonfinite, value_norm=value_norm,
            value_norm_beta=value_norm_beta, param_groups=param_groups, recompute_advantage=recompute_advantage,
            adam_options=adam_options, dual_clip=dual_clip, huber_delta=huber_delta, desired_kl=desired_kl,
            lr_bounds=lr_bounds, grad_noise_every=grad_noise_every, prox_ewma=prox_ewma)
        self.param_groups = bool(param_groups)
        self.adam_options = bool(adam_options)

    def push_weights(self):
        """agent modules -> updater (e.g. after load_checkpoint / freeze_*)."""
        flat = self.layout.from_state_dict(self.agent.actor_critic_net.state_dict())
        self.updater.params.copy_(torch.as_tensor(flat, device=self.updater.params.device))

    def pull_weights(self):
        sd = self.layout.to_state_dict(self.updater.flat_params())
        ref = self.agent.actor_critic_net.state_dict()
        self.agent.actor_critic_net.load_state_dict({k: torch.as_tensor(v).to(ref[k].device) for k, v in sd.items()})

    # ---- optimiser state (SURVEY 8f-4).  The reference's checkpoints hold no Adam state (save_checkpoint :172-193): a
    # resumed run restarts the moments, and so does a fresh B200Update.  These calls keep them, inside the reference's
    # own checkpoint files under a key the reference ignores.
    CHECKPOINT_KEY = "b200_optimizer"

    def optimizer_state(self) -> dict:
        """The Adam state, with the KL penalty on its current (possibly adapted) coefficient under "kl_coef", and with
        value_norm on the normaliser's running state under "value_norm" ({"m1", "m2", "d"})."""
        m, v, steps = self.updater.engine.get_opt_state()
        state = {"exp_avg": m, "exp_avg_sq": v, "steps": steps}
        if self.updater.kl_coef is not None:
            state["kl_coef"] = self.updater.kl_coef
        if getattr(self.updater, "value_norm", False):
            state["value_norm"] = dict(zip(("m1", "m2", "d"), self.updater.engine.get_value_norm_state()))
        if getattr(self, "param_groups", False):
            state["tensor_steps"] = self.updater.engine.get_tensor_steps()
        if getattr(self, "adam_options", False):
            vmax = self.updater.engine.get_amsgrad_state()
            if vmax is not None:
                state["max_exp_avg_sq"] = vmax
        if getattr(self.updater, "desired_kl", None) is not None:
            state["lr_state"] = self.updater.engine.get_lr_state()
        if getattr(self.updater, "prox_ewma", None) is not None and self.updater._prox_ready:
            state["prox_params"] = self.updater.engine.get_prox_params()
        return state

    def _read_param_groups(self):
        """The agent's parameter groups and requires_grad flags -> the updater (param_groups on)."""
        eng = self.updater.engine
        self._groups = live_param_groups(self.agent, self.layout, eng.betas, eng.eps, getattr(self, "adam_options", False))
        self.updater.set_param_groups(self._groups)

    def load_optimizer_state(self, state: dict, clip_like_new_process: bool = True) -> None:
        """Restore the Adam moments / step counts.  `clip_like_new_process` (default) keeps the reference's behaviour
        that the FIRST optimiser step of every process clips gradients (the parameters() generators of
        urban_planning_agent.py:46 are fresh in a new process, SURVEY A.6-2): the restored global step count is kept
        for Adam's bias correction but the clip-once latch is re-armed.  False = continue as if never interrupted."""
        self.updater.engine.set_opt_state(state["exp_avg"], state["exp_avg_sq"], state["steps"],
                                          rearm_first_step_clip=clip_like_new_process)
        # the KL penalty's coefficient where the run left it; a checkpoint without it restarts from the configured one
        if self.updater.kl_coef is not None:
            self.updater.set_kl_coef(state.get("kl_coef", self.updater.kl_coef_init))
        # the value normaliser where the run left it (the checkpointed value head predicts in its units); a checkpoint
        # without it starts from the identity
        if getattr(self.updater, "value_norm", False):
            vn = state.get("value_norm", dict(m1=0.0, m2=0.0, d=0.0))
            self.updater.engine.set_value_norm_state((vn["m1"], vn["m2"], vn["d"]))
        # each tensor's count where the run left it; a checkpoint without them starts each from its segment's count.
        # The table exists from the updater's construction; the agent's groups are read at the next update
        if getattr(self, "param_groups", False):
            ts = state.get("tensor_steps")
            if ts is None:      # steps [1] encoder and value, [2] land-use head, [3] road head
                seg = lambda sl: 0 if sl.owner != "pol" else (1 if sl.name.startswith("lu_") else 2)
                ts = [state["steps"][1 + seg(sl)] for sl in self.layout.slots.values()]
            self.updater.engine.set_tensor_steps(ts)
        # AMSGrad's running maximum where the run left it; a checkpoint without it starts from zeros
        if getattr(self, "adam_options", False):
            vmax = state.get("max_exp_avg_sq")
            if vmax is None and self.updater.engine.get_amsgrad_state() is not None:
                vmax = np.zeros(self.updater.engine.num_params, np.float32)
            if vmax is not None:
                self.updater.engine.set_amsgrad_state(vmax)
        # the adaptive lr where the run left it; a checkpoint without it starts from agent.optimizer's lr, which the next
        # update reads
        if getattr(self.updater, "desired_kl", None) is not None and state.get("lr_state") is not None:
            self.updater.engine.set_lr_state(state["lr_state"])
            self._write_back_lr()
        # the EWMA proximal parameters where the run left them; a checkpoint without them starts them from the live
        # parameters at the top of the next update
        if getattr(self.updater, "prox_ewma", None) is not None:
            prox = state.get("prox_params")
            if prox is not None:
                self.updater.engine.set_prox_params(prox)
            self.updater._prox_ready = prox is not None

    def _write_back_lr(self) -> None:
        """The adaptive lr into agent.optimizer.param_groups, so that the next update starts from it and a scheduler that
        multiplies lr composes with it: one lr into every group, or with param_groups each group's from its first
        trained tensor (a group without one keeps its lr).  The groups map to tensors as the last update read them or,
        before the first update (a checkpoint restored into a fresh controller), as live_param_groups reads them now."""
        opt = getattr(self.agent, "optimizer", None)
        eng = self.updater.engine
        if opt is None:
            return
        if eng.param_groups is None:
            for g in opt.param_groups:
                g["lr"] = eng.lr
            return
        names = list(eng.layout.slots)
        lrs, _, trained = eng.param_groups
        groups = getattr(self, "_groups", None)
        if groups is None:
            groups = live_param_groups(self.agent, self.layout, eng.betas, eng.eps, getattr(self, "adam_options", False))
        for g, lg in zip(opt.param_groups, groups):
            ks = [names.index(n) for n in lg["params"] if trained[names.index(n)]]
            if ks:
                g["lr"] = lrs[ks[0]]

    def value_stats(self):
        """(mean, std) of the value normaliser now: with value_norm on, agent.value_net(states) returns normalised
        values, and mean + std * value_net(states) is the value in reward units.  (0.0, 1.0) while the option is off or
        before the first update.  Synchronises the device."""
        if not getattr(self.updater, "value_norm", False):
            return 0.0, 1.0
        from .engine import value_norm_stats
        return value_norm_stats(*self.updater.engine.get_value_norm_state())

    def checkpoint_paths(self, iteration: int):
        """The files `UrbanPlanningAgent.save_checkpoint(iteration)` writes (urban_planning_agent.py:185-193)."""
        cfg, agent = self.agent.cfg, self.agent
        paths = []
        if cfg.save_model_interval > 0 and (iteration + 1) % cfg.save_model_interval == 0:
            paths.append("{}/iteration_{:04d}.p".format(cfg.model_dir, iteration + 1))
        if getattr(agent, "save_best_flag", False):
            paths.append("{}/best.p".format(cfg.model_dir))
            paths.append("{}/best_reward{:.2f}_iteration_{:04d}.p".format(cfg.model_dir, agent.best_rewards, iteration + 1))
        return paths

    def save_checkpoint(self, iteration: int):
        """`agent.save_checkpoint` (:172-193) followed by adding the Adam state to every file it wrote."""
        import os
        import pickle
        paths = self.checkpoint_paths(iteration)
        self._ref_save_checkpoint(iteration)
        state = None
        for p in paths:
            if os.path.exists(p):
                if state is None:
                    state = self.optimizer_state()
                with open(p, "rb") as f:
                    cp = pickle.load(f)
                cp[self.CHECKPOINT_KEY] = state
                with open(p, "wb") as f:
                    pickle.dump(cp, f)

    def load_checkpoint(self, checkpoint, restore_best_rewards: bool = True):
        """`agent.load_checkpoint` (:153-170) followed by restoring the Adam state if the file carries it."""
        import pickle
        start = self._ref_load_checkpoint(checkpoint, restore_best_rewards)
        cfg = self.agent.cfg
        cp_path = ("%s/iteration_%04d.p" % (cfg.model_dir, checkpoint)) if isinstance(checkpoint, int) else \
            ("%s/%s.p" % (cfg.model_dir, checkpoint))
        with open(cp_path, "rb") as f:
            cp = pickle.load(f)
        self.push_weights()
        if self.CHECKPOINT_KEY in cp:
            self.load_optimizer_state(cp[self.CHECKPOINT_KEY])
        return start

    def update_params(self, batch, iteration):
        """Signature and effects of UrbanPlanningAgent.update_params (:248-271), with the hyperparameters the agent holds
        now (live_hyperparameters): an lr scheduler stepped on agent.optimizer or an annealed agent.entropy_coef takes
        effect here, as in the reference."""
        t0 = time.time()
        agent = self.agent
        eng = self.updater.engine
        groups = getattr(self, "param_groups", False)
        if groups:
            self._read_param_groups()
        self.updater.set_hyperparameters(**live_hyperparameters(agent, eng.betas, eng.eps, groups,
                                                                getattr(self, "adam_options", False)))
        self.push_weights()
        tb = getattr(agent, "tb_logger", None)
        log_fn = (lambda tag, val, step: tb.add_scalar(tag, val, step)) if tb is not None else None
        self.updater.loss_iter = getattr(agent, "loss_iter", 0)
        self.updater.update_params(batch.states, batch.actions, batch.rewards, batch.masks, batch.exps,
                                   log_fn=log_fn, iteration=iteration)
        agent.loss_iter = self.updater.loss_iter
        self.pull_weights()
        if getattr(self.updater, "desired_kl", None) is not None:
            self._write_back_lr()
        return time.time() - t0


def use_b200_update(agent, **kw) -> B200Update:
    """Route `agent.update_params` through the H100 path; returns the controller object.  Keywords go to B200Update:
    clip_mode, process_group, device, diagnostics (True: PPO diagnostics under diag/* in the agent's tb_logger),
    target_kl (end each update before the first step whose approximate KL exceeds 1.5 * target_kl; None = off),
    value_clip (the clipped value loss of OpenAI baselines' ppo2 with range value_clip; None = off) and
    normalize_advantage (normalise each minibatch's advantages, as Stable-Baselines3 does; default False) and
    max_grad_norm (clip_grad_norm_ of all parameters to max_grad_norm on every step; needs clip_mode=CLIP_NEVER; None =
    off) and kl_coef / kl_target (the KL penalty kl_coef * KL(pi_old || pi) on the exact categorical KL; kl_target adapts
    the coefficient after every update by the PPO paper's rule; None = off / a fixed coefficient) and skip_nonfinite
    (True: a minibatch step whose statistics or reduced gradient are not finite changes no parameter, Adam moment or
    step counter -- the decision is on the gradient, not on the inputs or the losses: an infinite advantage whose ratio
    the surrogate clips gives a zero policy gradient, and that step is applied and logs an infinite surrogate loss --, is left out of the logged losses and is counted under diag/nonfinite_skips; an update whose every
    step was skipped raises FloatingPointError; default False: such a minibatch raises FloatingPointError after its
    epoch, or passes NaN into the parameters) and value_norm / value_norm_beta (True: value targets normalised by
    running return statistics with EMA weight value_norm_beta, default 0.99999, and PopArt's output-preserving rescale
    of the value head's last layer; agent.value_net(states) then returns normalised values, see
    B200Update.value_stats; default False) and param_groups (True: train exactly the tensors torch's Adam.step would --
    those with requires_grad=True in agent.optimizer's param_groups -- each with its group's lr and weight_decay and its
    own step count, read at the top of every update (live_param_groups); default False: every tensor is trained with one
    lr and weight_decay, and requires_grad is ignored) and recompute_advantage (True: every epoch after the first trains
    on advantages, returns and value-clip anchors recomputed from a value-only sweep at the parameters the previous epoch
    left, as Tianshou's recompute_advantage; default False: all from the update's pre-pass) and adam_options (True: each
    update also applies the betas, eps, amsgrad and decoupled_weight_decay of agent.optimizer's param_groups, so that
    agent.optimizer = torch.optim.AdamW(...) or Adam(..., amsgrad=True) trains as torch would; default False: those
    keys must keep the engine's values) and dual_clip (dual-clip PPO as Tianshou's PPOPolicy(dual_clip=c): the
    surrogate of a negative advantage A is bounded below by dual_clip * A; finite and > 1; None = off) and huber_delta
    (the Huber value loss 2 huber_loss(V, R, delta) in place of (V - R)^2, as MAPPO's use_huber_loss; finite and > 0;
    None = off) and desired_kl / lr_bounds (RSL-RL's adaptive lr schedule: every minibatch step divides the lr by 1.5
    when its approximate KL, measured at the parameters it starts from, is above 2 * desired_kl and multiplies it by 1.5
    when it is below desired_kl / 2, within lr_bounds, default (1e-5, 1e-2); decided inside the step kernels.  The
    adapted lr is written back into agent.optimizer.param_groups after every update, so a scheduler that multiplies lr
    composes with it, while a LambdaLR, which sets lr from its base value, overrides it; None = off) and
    grad_noise_every (an integer k >= 1: measure the gradient noise scale B_noise of McCandlish et al. 2018 before
    minibatch step i of every epoch when i % k == 0, from one extra gradient launch of the minibatch in a random order;
    update_params returns grad_noise_scale, grad_noise_g2, grad_noise_trace and grad_noise_samples and logs them under
    diag/ once per iteration; training is unchanged; None = off) and prox_ewma (a weight beta in [0, 1): PPO-EWMA, the
    clip keeps the policy close to an exponential moving average of the weights over optimiser steps while the behaviour
    policy weights the surrogate; its mean age is beta / (1 - beta) steps, mini_batch_size * beta / (1 - beta) graphs,
    so a run that changes mini_batch_size keeps its behaviour with engine.prox_ewma_for_batch; the average is kept in
    checkpoints under "prox_params"; with diagnostics, diag/prox_weight and diag/prox_kl; None = off).  Every update
    reads the agent's current hyperparameters first
    (live_hyperparameters): an lr scheduler on agent.optimizer or a changed agent.entropy_coef takes effect there."""
    ctl = B200Update(agent, **kw)
    agent.update_params = ctl.update_params
    # checkpoints: the reference's files, plus the Adam moments under a key it ignores (SURVEY 8f-4)
    if hasattr(agent, "save_checkpoint"):
        ctl._ref_save_checkpoint = agent.save_checkpoint
        agent.save_checkpoint = ctl.save_checkpoint
    if hasattr(agent, "load_checkpoint"):
        ctl._ref_load_checkpoint = agent.load_checkpoint
        agent.load_checkpoint = ctl.load_checkpoint
    agent._b200_update = ctl
    return ctl
