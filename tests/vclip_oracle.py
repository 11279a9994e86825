"""Per-minibatch advantage normalisation (Stable-Baselines3's normalize_advantage) for the oracles, which do not
implement it, and the clipped value loss (OpenAI baselines' ppo2, CleanRL's clip_vloss) in torch's operations:
    d = V - V_old,  Vc = V_old + clamp(d, -c, c),  a = (V - R)^2,  b = (Vc - R)^2,  loss = max(a, b)
averaged over the minibatch's B graphs.  The minibatch with the clipped value loss is tests/ppo_oracle.py's."""
from __future__ import annotations

import numpy as np
import torch


def clipped_value_loss(v, ret, old_values, c):
    """The torch form: mean of torch.max(a, b), all tensors of one shape."""
    d = v - old_values
    vc = old_values + torch.clamp(d, -c, c)
    return torch.max((v - ret).pow(2), (vc - ret).pow(2)).mean()


def normalize64(adv, exps, order, B):
    """float64 normalisation of every minibatch order[i B, (i + 1) B), i < len(order) // B, rounded as the kernel does:
    mean and unbiased std to fp32 once each, then (A - mean) / (std + 1e-8) in fp32.  Other entries keep their values."""
    adv = np.asarray(adv, np.float32).reshape(-1)
    exps = np.asarray(exps).reshape(-1)
    out = adv.copy()
    for i in range(len(order) // B):
        idx = np.asarray(order[i * B:(i + 1) * B])
        sel = adv[idx[exps[idx] != 0]].astype(np.float64)
        if sel.size < 2:
            continue
        mean = np.float32(sel.mean())
        std = np.float32(np.sqrt(((sel - sel.mean()) ** 2).sum() / (sel.size - 1)))
        out[idx] = (adv[idx] - mean) / np.float32(std + np.float32(1e-8))
    return out


def normalize_torch(adv, exps, order, B):
    """The Stable-Baselines3 formula in torch fp32 on each minibatch's exps != 0 advantages, written to all its graphs."""
    adv = torch.as_tensor(np.asarray(adv, np.float32).reshape(-1))
    exps = torch.as_tensor(np.asarray(exps).reshape(-1))
    out = adv.clone()
    for i in range(len(order) // B):
        idx = torch.as_tensor(np.asarray(order[i * B:(i + 1) * B]), dtype=torch.long)
        sel = adv[idx][exps[idx] != 0]
        if sel.numel() < 2:
            continue
        out[idx] = (adv[idx] - sel.mean()) / (sel.std() + 1e-8)
    return out.numpy()
