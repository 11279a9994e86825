"""Float64 host helpers of the gradient-noise tests: the kernels' static item-to-CTA assignment written as the loop the
step kernels run, the four values {A, S, Q, N} of one measurement from per-item gradient terms grouped by it,
McCandlish et al.'s two-batch estimator in its own notation, and per-graph float64 gradient terms of the SGNN from the
torch port."""
import numpy as np
import torch


def assignment(count, grid):
    """The items each CTA takes: a launch has min(count, grid) CTAs, and CTA c runs `for item = c; item < count;
    item += gridDim.x` (sgnn_kernel.cuh, mlp_kernel.cuh)."""
    g = min(count, grid)
    groups = [[] for _ in range(g)]
    for c in range(g):
        item = c
        while item < count:
            groups[c].append(item)
            item += g
    return groups


def measure(x, grid):
    """{A, S, Q, N} of the summed-gradient terms x (N rows, one per item in launch order) grouped by assignment()."""
    x = np.asarray(x, np.float64)
    groups = assignment(x.shape[0], grid)
    A = sum(float(np.square(x[g].sum(0)).sum()) for g in groups)
    S = float(np.square(x.sum(0)).sum())
    Q = float(sum(len(g) ** 2 for g in groups))
    return np.array([A, S, Q, float(x.shape[0])])


def mccandlish(g_small_sq, g_big_sq, b_small, b_big):
    """McCandlish et al. 2018, appendix A.1: unbiased |G|^2 and tr(Sigma) from the squared norms of the mean gradients
    of a small batch (|G_small|^2, averaged over small batches) and of a big batch; (|G|^2, S, S / |G|^2)."""
    g2 = (b_big * g_big_sq - b_small * g_small_sq) / (b_big - b_small)
    tr = (g_small_sq - g_big_sq) / (1.0 / b_small - 1.0 / b_big)
    return g2, tr, tr / g2


def sgnn_graph_terms(flat, states, actions, adv, ret, fixed, exps, value_pred_coef=0.5, entropy_coef=0.01,
                     clip_epsilon=0.2):
    """x_i of every graph through the torch port (whose model runs in fp32), as float64: the gradient of graph i's share
    of the minibatch loss c_v (V_i - R_i)^2 / B + [exps_i != 0] (surr_i + c_e (-entropy_i)) / |ind|, so that the
    minibatch gradient is sum x_i.  Each graph is its own autograd pass: no graph's rounding enters another's term."""
    from oracle import torch_port as TP
    B = len(states)
    adv, ret, fixed = (np.asarray(a, np.float64).reshape(-1) for a in (adv, ret, fixed))
    n_ind = max(int((np.asarray(exps) != 0).sum()), 1)
    out = np.zeros((B, flat.size), np.float64)
    for i in range(B):
        p = torch.tensor(np.asarray(flat, np.float32), requires_grad=True)
        P = TP.params_from_flat(p)
        b = TP.stack_states([states[i]])
        act = torch.tensor(np.asarray(actions[i:i + 1], np.float32))
        ind = torch.tensor([bool(exps[i] != 0)])
        one = lambda v: torch.tensor([[float(v)]], dtype=torch.float32)
        surr, vl, ent = TP.ppo_losses(P, b, act, one(adv[i]), one(ret[i]), one(fixed[i]), ind, clip_epsilon)
        loss = value_pred_coef * vl / B
        if exps[i] != 0:
            loss = loss + (surr + entropy_coef * ent) / n_ind
        loss.backward()
        out[i] = p.grad.numpy().astype(np.float64)
    return out
