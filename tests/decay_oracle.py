"""Adam weight decay (cfg `weightdecay`, torch.optim.Adam(weight_decay=...) at urban_planning_agent.py:145-149) for the
oracles, which themselves run Adam without it.

torch adds the term inside `Adam.step` as `grad = grad.add(param, alpha=weight_decay)`: coupled L2, after
clip_policy_grad has scaled `.grad`, from the parameter before the step, and only for tensors whose `.grad` is not
None (a skipped policy head gets none)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP


def adam_step(flat, m, v, t, grad, live, wd, **kw):
    """oracle/sgnn_numpy.adam_step with the decay term added to the live entries' (already clipped) gradient."""
    grad = np.where(live, np.asarray(grad, np.float64) + wd * np.asarray(flat, np.float64), grad)
    return ON.adam_step(flat, m, v, t, grad, live, **kw)


def _decayed_adam(params, wd, lr=4e-4, eps=1e-5):
    return torch.optim.Adam(params, lr=lr, eps=eps, weight_decay=wd)


def port_agent(flat, wd, lr=4e-4, eps=1e-5, **kw) -> TP.PortAgent:
    """oracle/torch_port.PortAgent whose optimiser is torch.optim.Adam(lr, eps, weight_decay=wd)."""
    agent = TP.PortAgent(flat, lr=lr, eps=eps, **kw)
    agent.opt = _decayed_adam(list(agent.P.values()), wd, lr, eps)
    return agent


def mlp_port_agent(flat, wd, lr=4e-4, eps=1e-5, **kw) -> MP.MLPPortAgent:
    """oracle/mlp_port.MLPPortAgent whose optimiser is torch.optim.Adam(lr, eps, weight_decay=wd)."""
    agent = MP.MLPPortAgent(flat, lr=lr, eps=eps, **kw)
    agent.opt = _decayed_adam(list(agent.P.values()), wd, lr, eps)
    return agent
