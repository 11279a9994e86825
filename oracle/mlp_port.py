"""TEST INFRASTRUCTURE ONLY.  CPU restatement of the reference's rl-mlp ablation model and its PPO losses.

Follows, op for op on padded batches, `MLPStateEncoder.forward` (reference
urban_planning/models/state_encoder.py:217-308), the policy heads (urban_planning/models/policy.py:45-104), the value
head (urban_planning/models/value.py:36-39) and the PPO losses of agent_pg.py:19-23 / urban_planning_agent.py:363-371.
Gradients come from autograd, as in the reference.  Pinned to golden vectors produced by the reference's own
`create_mlp_model` (tests/golden/mlp_*.npz, tests/test_mlp.py).  Parameters are a dict keyed by the short names of
drl_urban_planning_b200/params.py (`PL.MLP`).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from drl_urban_planning_b200 import params as PL
from oracle.torch_port import stack_states          # tensorfy + batch_data (state_encoder.py:163-177)

MASK_FILL = -2.0 ** 32 + 1        # policy.py:50
FEASIBLE = 1                      # city_config.py:24
NUM_TYPE_SLOTS = 14               # city_config.NUM_TYPES + 1


def params_from_flat(flat, dtype=torch.float32, requires_grad=False) -> Dict[str, torch.Tensor]:
    flat = np.asarray(flat, np.float32)
    return {s.name: torch.tensor(flat[s.offset:s.offset + s.size].reshape(s.shape).copy(), dtype=dtype,
                                 requires_grad=requires_grad) for s in PL.MLP.slots.values()}


def _mean(h, mask):                                  # SGNNStateEncoder.mean_features (state_encoder.py:179-182)
    m = mask.unsqueeze(-1).to(h.dtype)
    return (h * m).sum(1) / mask.to(h.dtype).sum(1, keepdim=True)


def encode(P, b):
    """MLPStateEncoder.forward (state_encoder.py:278-308) -> land-use features, road features, value features."""
    dt = P["enc_w"].dtype
    x, ei = b["node_features"].to(dt), b["edge_index"]
    h_num = torch.tanh(torch.tanh(b["numerical"].to(dt) @ P["num_w0"].T + P["num_b0"]) @ P["num_w1"].T + P["num_b1"])
    D = x.shape[-1]
    f1 = torch.gather(x, 1, ei[:, :, 0].unsqueeze(-1).expand(-1, -1, D))          # :269-270
    f2 = torch.gather(x, 1, ei[:, :, 1].unsqueeze(-1).expand(-1, -1, D))
    feas = torch.argmax(f2[:, :, :NUM_TYPE_SLOTS], dim=-1) == FEASIBLE              # :271
    fe = torch.where(feas.unsqueeze(-1), f2, f1)
    fe = torch.where(b["edge_mask"].unsqueeze(-1), fe, torch.zeros_like(fe))        # :274-275
    h_nodes = x @ P["enc_w"].T + P["enc_b"]
    h_edges = fe @ P["enc_w"].T + P["enc_b"]
    hc = (b["current_node"].to(dt) @ P["enc_w"].T + P["enc_b"]).unsqueeze(1)
    sv = torch.cat([h_num, _mean(h_nodes, b["node_mask"]), _mean(h_edges, b["edge_mask"]), b["stage"].to(dt)], 1)
    hcr = hc.expand(-1, h_edges.shape[1], -1)
    lu = torch.cat([h_edges, hcr, h_edges * hcr, h_edges - hcr], -1)
    return lu, h_nodes, sv


def value(P, b):
    _, _, sv = encode(P, b)
    y = torch.tanh(sv @ P["val_w0"].T + P["val_b0"])
    y = torch.tanh(y @ P["val_w1"].T + P["val_b1"])
    return y @ P["val_w2"].T + P["val_b2"]


def masked_logits(P, b):
    lu, hn, _ = encode(P, b)
    z_lu = (torch.tanh(lu @ P["lu_w0"].T + P["lu_b0"]) @ P["lu_w1"].T).squeeze(-1)
    z_rd = (torch.tanh(hn @ P["road_w0"].T + P["road_b0"]) @ P["road_w1"].T).squeeze(-1)
    fill = torch.tensor(MASK_FILL, dtype=z_lu.dtype)
    return torch.where(b["land_use_mask"], z_lu, fill), torch.where(b["road_mask"], z_rd, fill)


def log_prob_entropy(P, b, actions):
    zl, zr = masked_logits(P, b)
    st0 = b["stage"][:, 0] > 0
    B = st0.shape[0]
    lp = torch.zeros(B, dtype=zl.dtype)
    ent = torch.zeros(B, dtype=zl.dtype)
    for sel, z, col in ((st0, zl, 0), (~st0, zr, 1)):
        if sel.any():
            d = torch.distributions.Categorical(logits=z[sel])
            lp = lp.index_put((sel.nonzero().squeeze(1),), d.log_prob(actions[sel, col]))
            ent = ent.index_put((sel.nonzero().squeeze(1),), d.entropy())
    return lp.unsqueeze(1), ent.unsqueeze(1)


def greedy_action(P, b):
    zl, zr = masked_logits(P, b)
    st0 = b["stage"][:, 0] > 0
    out = torch.zeros(st0.shape[0], 2)
    out[st0, 0] = torch.softmax(zl[st0], -1).argmax(-1).float()
    out[~st0, 1] = torch.softmax(zr[~st0], -1).argmax(-1).float()
    return out


def ppo_losses(P, b, actions, adv, ret, fixed_lp, ind, clip_epsilon=0.2):
    v = value(P, b)
    value_loss = (v - ret.to(v.dtype)).pow(2).mean()
    lp, ent = log_prob_entropy(P, b, actions)
    ratio = torch.exp(lp[ind] - fixed_lp.to(lp.dtype)[ind])
    a = adv.to(lp.dtype)[ind]
    surr = -torch.min(ratio * a, torch.clamp(ratio, 1 - clip_epsilon, 1 + clip_epsilon) * a).mean()
    return surr, value_loss, -ent[ind].mean()


class MLPPortAgent:
    """Update half of the rl-mlp agent: Adam over the 18 tensors + the reference's first-step-only clipping."""

    def __init__(self, flat, lr=4e-4, eps=1e-5, dtype=torch.float32, clip_epsilon=0.2, value_pred_coef=0.5,
                 entropy_coef=0.01):
        self.P = params_from_flat(flat, dtype, requires_grad=True)
        self.opt = torch.optim.Adam(list(self.P.values()), lr=lr, eps=eps)
        self.clip_epsilon, self.value_pred_coef, self.entropy_coef = clip_epsilon, value_pred_coef, entropy_coef
        self.steps_done = 0
        self.groups = [[s.name for s in PL.MLP.slots.values() if s.owner in ("enc", "pol")],
                       [s.name for s in PL.MLP.slots.values() if s.owner in ("enc", "val")]]

    def flat(self):
        return PL.MLP.flatten({k: v.detach().numpy() for k, v in self.P.items()})

    def flat_grad(self):
        return PL.MLP.flatten({k: (v.grad.numpy() if v.grad is not None else np.zeros(tuple(v.shape)))
                               for k, v in self.P.items()})

    def backward(self, b, actions, adv, ret, fixed, ind):
        surr, vl, el = ppo_losses(self.P, b, actions, adv, ret, fixed, ind, self.clip_epsilon)
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el
        self.opt.zero_grad()
        loss.backward()
        return loss.item(), vl.item(), surr.item(), el.item()

    def step(self, *args):
        out = self.backward(*args)
        if self.steps_done == 0:
            for names in self.groups:
                torch.nn.utils.clip_grad_norm_([self.P[n] for n in names], 1.0)
        self.opt.step()
        self.steps_done += 1
        return out
