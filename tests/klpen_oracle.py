"""The KL penalty on the exact categorical KL (upb_set_kl_penalty) for the oracles, which do not implement it.

For one graph with candidates c (masked entries have probability exactly 0), old log-probs lp_old at the update's
pre-pass parameters and lp at the current ones:
    KL_g = sum_c p_old(c) (lp_old(c) - lp(c)),   d KL_g / d z(c) = p(c) - p_old(c)
(autograd gives p sum(p_old) - p_old; sum(p_old) = 1).  The sum is taken in log space, so a new probability that
underflows gives a large finite term (torch.distributions.kl_divergence would give inf); a p_old that underflows adds
0.  The minibatch's penalty is beta * (1/|ind|) sum over ind of KL_g."""
from __future__ import annotations

import numpy as np
import torch

from drl_urban_planning_b200 import params as PL
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP


def kl64(lp_old, lp):
    """float64 (KL_g, d KL_g / d z) of one graph from its candidates' old and new log-probs (any order, same for both)."""
    lo, ln = np.asarray(lp_old, np.float64), np.asarray(lp, np.float64)
    po, p = np.exp(lo), np.exp(ln)
    return float(np.where(po > 0, po * (lo - ln), 0.0).sum()), p - po


def cand_layout(blob):
    """Per graph of a packed blob: (cand_off, k) and the blob's cand_idx section, from the host copy (csrc/blob.h)."""
    h = blob.host.numpy() if hasattr(blob.host, "numpy") else blob.host
    h = np.asarray(h[:blob.nbytes])
    hdr = np.frombuffer(h[:128].tobytes(), np.uint64)
    off_desc, off_cuv, off_cidx = int(hdr[3]), int(hdr[9]), int(hdr[10])
    desc = np.frombuffer(h[off_desc:off_desc + 64 * blob.count].tobytes(), np.int32).reshape(blob.count, 16)
    cidx = np.frombuffer(h[off_cidx:off_cidx + (off_cidx - off_cuv)].tobytes(), np.int32)
    return desc[:, 7].astype(np.int64), desc[:, 3].astype(np.int64), cidx


def per_graph(cand, blob):
    """Split a per-candidate array (candidate positions of `blob`) into one array per graph, each in mask-index order
    (the order of ON.forward's candidates), with those indices."""
    off, k, cidx = cand_layout(blob)
    out = []
    for i in range(blob.count):
        idx = cidx[off[i]:off[i] + k[i]]
        order = np.argsort(idx, kind="stable")
        out.append((np.asarray(cand)[off[i]:off[i] + k[i]][order], idx[order]))
    return out


def to_positions(per_graph_lp, blob):
    """The inverse of per_graph: a flat float32 per-candidate array of blob.cand_len from per-graph arrays in
    mask-index order."""
    off, k, cidx = cand_layout(blob)
    out = np.zeros(blob.cand_len, np.float32)
    for i in range(blob.count):
        idx = cidx[off[i]:off[i] + k[i]]
        order = np.argsort(idx, kind="stable")
        dst = np.zeros(k[i], np.float32)
        dst[order] = np.asarray(per_graph_lp[i], np.float32)
        out[off[i]:off[i] + k[i]] = dst
    return out


# ---- float64: the SGNN's numpy oracle -------------------------------------------------------------------------------
def cand_logp64(flat, states):
    """float64 log-softmax over every graph's candidates (mask-index order) with the SGNN's numpy oracle."""
    P = ON._p64(flat)
    out = []
    for st in states:
        fw = ON.forward(P, ON.unpad(st), keep=True)
        out.append(np.asarray(fw["cache"].get("logp", np.zeros(0)), np.float64) if fw["stage_id"] >= 0 else np.zeros(0))
    return out


def mlp_params64(flat, requires_grad=False):
    """The rl-mlp port's tensors in float64 from a float64 flat vector (mlp_port.params_from_flat rounds it to fp32)."""
    flat = np.asarray(flat, np.float64)
    return {s.name: torch.tensor(flat[s.offset:s.offset + s.size].reshape(s.shape).copy(), dtype=torch.float64,
                                 requires_grad=requires_grad) for s in PL.MLP.slots.values()}


def mlp_cand_logp64(flat, states):
    """float64 log-softmax over every graph's candidates (mask-index order) with the rl-mlp torch port in float64."""
    P = mlp_params64(flat)
    b = MP.stack_states(states)
    with torch.no_grad():
        zl, zr = MP.masked_logits(P, b)
    out = []
    for i in range(len(states)):
        lu = bool(b["stage"][i, 0] > 0)
        mask = (b["land_use_mask"] if lu else b["road_mask"])[i].numpy()
        z = (zl if lu else zr)[i].numpy()[mask]
        out.append(z - z.max() - np.log(np.exp(z - z.max()).sum()) if z.size else np.zeros(0))
    return out


def ppo_minibatch(flat, states, actions, advantages, returns, fixed_log_probs, exps, lp_old, beta,
                  clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01):
    """oracle/sgnn_numpy.ppo_minibatch plus beta * kl: float64 losses (loss includes beta * kl), the flat gradient and
    slot 18's sum (kl_sum) and per-graph KL_g (kl_g).  lp_old: per graph, its candidates' old log-probs in mask-index
    order.  The penalty's logit seed enters sgnn_numpy.backward as a second call whose g_z is exactly that seed (the
    backward is linear in g_z: with g_logp = -1, g_ent = 0 and no action, g_z = the cached p, replaced by the seed)."""
    P = ON._p64(flat)
    B = len(states)
    adv, ret, flp = (np.asarray(x, np.float64).reshape(-1) for x in (advantages, returns, fixed_log_probs))
    ind = set(np.flatnonzero(np.asarray(exps).reshape(-1) != 0).tolist())
    n_ind = max(len(ind), 1)
    Gtot = {k: np.zeros_like(v) for k, v in P.items()}
    surr = eloss = vsum = 0.0
    kl_g = np.zeros(B)
    for i, st in enumerate(states):
        g = ON.unpad(st)
        sid = int(np.argmax(g.stage[:2]))
        fw = ON.forward(P, g, action=int(actions[i, sid]), keep=True)
        V = fw["value"]
        vsum += (V - ret[i]) ** 2
        g_lp = g_en = 0.0
        if i in ind:
            r = np.exp(fw["log_prob"] - flp[i])
            s1, s2 = r * adv[i], np.clip(r, 1 - clip_epsilon, 1 + clip_epsilon) * adv[i]
            surr += -min(s1, s2) / n_ind
            eloss += -fw["entropy"] / n_ind
            if (1 - clip_epsilon) <= r <= (1 + clip_epsilon) or s1 < s2:
                g_lp = -adv[i] * r / n_ind
            g_en = -entropy_coef / n_ind
        Gi = ON.backward(P, g, fw, value_pred_coef * 2.0 * (V - ret[i]) / B, g_lp, g_en)
        c = fw["cache"]
        if i in ind and c.get("logp") is not None and c["logp"].size:
            kl_g[i], seed = kl64(lp_old[i], c["logp"])
            fw2 = dict(fw, cache=dict(c, p=beta / n_ind * seed), action_pos=-1)
            G2 = ON.backward(P, g, fw2, 0.0, -1.0, 0.0)
            for k in Gi:
                Gi[k] = Gi[k] + G2[k]
        for k in Gtot:
            Gtot[k] += Gi[k]
    vloss = vsum / B
    kl = kl_g.sum() / n_ind
    grad = np.zeros(PL.NUM_PARAMS)
    for s in PL.SLOTS.values():
        grad[s.offset:s.offset + s.size] = Gtot[s.name].reshape(-1)
    return dict(loss=surr + value_pred_coef * vloss + entropy_coef * eloss + beta * kl, value_loss=vloss,
                surr_loss=surr, entropy_loss=eloss, kl_loss=kl, grad=grad, kl_sum=kl_g.sum(), kl_g=kl_g)


# ---- the torch form ---------------------------------------------------------------------------------------------------
def kl_rows(lo, ln):
    """Per row of masked, normalised log-probs (old without gradient, new): sum p_old (lp_old - lp), in log space."""
    return (lo.exp() * (lo - ln)).sum(-1)


def sgnn_kl(P, P_old, b):
    """(B,) per-graph exact KL of the SGNN torch port (oracle/torch_port._distributions) against P_old's policy."""
    d0, d1, sel0, sel1 = TP._distributions(P, b)
    with torch.no_grad():
        o0, o1, _, _ = TP._distributions(P_old, b)
    kl = torch.zeros(b["stage"].shape[0], dtype=torch.float32)
    for d, o, sel in ((d0, o0, sel0), (d1, o1, sel1)):
        if d is not None:
            kl = kl.index_put((sel.nonzero().squeeze(1),), kl_rows(o.logits, d.logits))
    return kl


def mlp_kl(P, P_old, b):
    """(B,) per-graph exact KL of the rl-mlp port (oracle/mlp_port.masked_logits) against P_old's policy."""
    zl, zr = MP.masked_logits(P, b)
    with torch.no_grad():
        ol, orr = MP.masked_logits(P_old, b)
    st0 = b["stage"][:, 0] > 0
    kl = torch.zeros(st0.shape[0], dtype=zl.dtype)
    for sel, z, o in ((st0, zl, ol), (~st0, zr, orr)):
        if sel.any():
            kl = kl.index_put((sel.nonzero().squeeze(1),),
                              kl_rows(torch.log_softmax(o[sel], -1), torch.log_softmax(z[sel], -1)))
    return kl


class PortAgent(TP.PortAgent):
    """oracle/torch_port.PortAgent with beta * kl against the policy of `P_old` (the update's pre-pass parameters, set
    with snapshot()); `beta` may change between steps."""

    def __init__(self, flat, beta, **kw):
        super().__init__(flat, **kw)
        self.beta, self.P_old, self.last_kl = beta, None, None

    def snapshot(self):
        self.P_old = {k: v.detach().clone() for k, v in self.P.items()}

    def backward(self, b, actions, advantages, returns, fixed_log_probs, ind):
        surr, vl, el = TP.ppo_losses(self.P, b, actions, advantages, returns, fixed_log_probs, ind, self.clip_epsilon)
        kl = sgnn_kl(self.P, self.P_old, b)[ind].mean()
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el + self.beta * kl
        self.opt.zero_grad()
        loss.backward()
        self.last_kl = kl.item()
        return loss.item(), vl.item(), surr.item(), el.item()


class MLPPortAgent(MP.MLPPortAgent):
    """oracle/mlp_port.MLPPortAgent with beta * kl against the policy of `P_old` (snapshot())."""

    def __init__(self, flat, beta, **kw):
        super().__init__(flat, **kw)
        self.beta, self.P_old, self.last_kl = beta, None, None

    def snapshot(self):
        self.P_old = {k: v.detach().clone() for k, v in self.P.items()}

    def backward(self, b, actions, adv, ret, fixed, ind):
        surr, vl, el = MP.ppo_losses(self.P, b, actions, adv, ret, fixed, ind, self.clip_epsilon)
        kl = mlp_kl(self.P, self.P_old, b)[ind].mean()
        loss = surr + self.value_pred_coef * vl + self.entropy_coef * el + self.beta * kl
        self.opt.zero_grad()
        loss.backward()
        self.last_kl = kl.item()
        return loss.item(), vl.item(), surr.item(), el.item()
