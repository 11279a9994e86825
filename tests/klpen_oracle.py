"""The KL penalty's (upb_set_kl_penalty) candidate log-probs and its torch form for both models.

For one graph with candidates c (masked entries have probability exactly 0), old log-probs lp_old at the update's
pre-pass parameters and lp at the current ones:
    KL_g = sum_c p_old(c) (lp_old(c) - lp(c)),   d KL_g / d z(c) = p(c) - p_old(c)
(autograd gives p sum(p_old) - p_old; sum(p_old) = 1).  The sum is taken in log space, so a new probability that
underflows gives a large finite term (torch.distributions.kl_divergence would give inf); a p_old that underflows adds
0.  The float64 per-graph term (kl64) and the minibatch with the penalty are tests/ppo_oracle.py's."""
from __future__ import annotations

import numpy as np
import torch

from drl_urban_planning_b200 import params as PL
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON
from oracle import torch_port as TP


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
