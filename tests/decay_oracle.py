"""Adam weight decay (cfg `weightdecay`, torch.optim.Adam(weight_decay=...) at urban_planning_agent.py:145-149) for the
oracles, which themselves run Adam without it.

torch adds the term inside `Adam.step` as `grad = grad.add(param, alpha=weight_decay)`: coupled L2, after
clip_policy_grad has scaled `.grad`, from the parameter before the step, and only for tensors whose `.grad` is not
None (a skipped policy head gets none)."""
from __future__ import annotations

import numpy as np

import ppo_oracle as PPO
from oracle import sgnn_numpy as ON


def adam_step(flat, m, v, t, grad, live, wd, **kw):
    """oracle/sgnn_numpy.adam_step with the decay term added to the live entries' (already clipped) gradient."""
    grad = np.where(live, np.asarray(grad, np.float64) + wd * np.asarray(flat, np.float64), grad)
    return ON.adam_step(flat, m, v, t, grad, live, **kw)


def port_agent(flat, wd, **kw):
    """ppo_oracle.PortAgent on torch.optim.Adam(weight_decay=wd)."""
    return PPO.PortAgent(flat, weight_decay=wd, **kw)


def mlp_port_agent(flat, wd, **kw):
    """ppo_oracle.MLPPortAgent on torch.optim.Adam(weight_decay=wd)."""
    return PPO.MLPPortAgent(flat, weight_decay=wd, **kw)
