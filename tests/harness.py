"""Helpers shared by the test modules: error measures, golden-fixture loading, the `dev` fixture, the minibatch builder
and step drivers of the fused-against-two-call checks, the reference-agent stand-ins and a multi-process launcher.

Test modules import the fixture by name (`from harness import dev`), which registers it in that module."""
import os
import queue
import socket
import time
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states


# ---- error measures --------------------------------------------------------------------------------------------------
def rel(a, b, floor=1e-9):
    """max|a - b| / max|b| (the denominator at least `floor`)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


def tensor_errors(got, want, layout=PL.SGNN):
    """Per tensor of `layout`, max|delta| / max|want|.  Tensors whose gradient is (nearly) a sum of cancelling terms --
    attention key biases (exactly zero, SURVEY A.7) and, on tiny batches, head biases (the softmax logit gradients sum
    to zero) -- count as 0 while their error is within an absolute floor of 1e-7 x the largest entry of the whole of
    `want`: fp32 cancellation noise, present in the fp32 reference itself."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    floor = 1e-7 * max(np.abs(want).max(), 1e-9)
    out = {}
    for s in layout.slots.values():
        a, b = got[s.offset:s.offset + s.size], want[s.offset:s.offset + s.size]
        d = np.abs(a - b).max()
        out[s.name] = 0.0 if d <= floor else float(d / max(np.abs(b).max(), 1e-30))
    return out


def per_tensor_rel(got, want, layout=PL.SGNN):
    """(worst tensor_errors value, that tensor's name); (0.0, None) when every tensor is within the floor."""
    errs = tensor_errors(got, want, layout)
    name = max(errs, key=errs.get)
    return (errs[name], name) if errs[name] > 0 else (0.0, None)


def lp_tol(lp64, zabs):
    """Per-candidate log-prob tolerance: fp32 rounding of logits of magnitude `zabs` and of the log-prob itself."""
    return 2e-6 * (8.0 + np.abs(lp64) + zabs)


# ---- fixtures and device tensors -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need an H100"
    return torch.device("cuda", 0)


def t(x, dev):
    return torch.as_tensor(np.ascontiguousarray(x), device=dev)


def load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def update_losses(logged):
    """The per-minibatch loss/* values an update logged, one row (loss, value, surr, entropy) per step."""
    return np.array([[v for tag, v, s in logged if tag == k] for k in
                     ("loss/loss", "loss/value_loss", "loss/surr_loss", "loss/entropy_loss")]).T


def heads(layout):
    """Stage -> the parameter range of that stage's policy head."""
    return {0: slice(layout.slots["lu_w0"].offset, layout.slots["road_w0"].offset),
            1: slice(layout.slots["road_w0"].offset, layout.policy_end)}


# ---- minibatches and step drivers ------------------------------------------------------------------------------------
def reproducible_states(seed, count, spec=synth.COMMUNITIES["small"]):
    """`count` graphs of both stages, in random order, whose k_mlp gradient rows are run-to-run reproducible.

    The rl-mlp land-use head backward adds each candidate's input gradient to its selected node with shared-memory
    atomics from several warps, so a node selected by three or more candidates receives its sum in a run-dependent
    order (two additions onto zero commute exactly).  Road candidates are distinct nodes.  So: road graphs of the
    generator's sizes, and land-use graphs with one or two candidates."""
    rng = np.random.default_rng(seed)
    stages = rng.integers(0, 2, count)
    states, actions = [], np.zeros((count, 2), np.float32)
    for i, s in enumerate(stages):
        if s == 1:
            st, a = synth.make_state(rng, spec, stage=1)
        else:
            n = int(rng.integers(8, spec.max_num_nodes + 1))
            e = int(rng.integers(n, min(2 * n, spec.max_num_edges) + 1))
            st, a = synth.make_exact_state(rng, spec, n, e, 1 + i % 2, 0)
        states.append(st)
        actions[i, s] = a
    return states, actions


class Case:
    """A minibatch resident on the device: the states packed into one blob, PPO targets seeded by `seed` with
    exps = 0 at `zero_exps`, old log-probs N(-3, 0.3) (or `fixed`), and the model's initial parameters for `seed`."""

    def __init__(self, dev, model, states, actions, seed, zero_exps=(7,), fixed=None):
        self.dev, self.model = dev, model
        self.layout = PL.MLP if model == "mlp" else PL.SGNN
        self.count = len(states)
        self.states, self.actions = states, actions
        self.adv, self.ret, self.exps = synth.make_ppo_targets(seed, self.count)
        for i in zero_exps:
            self.exps[i] = 0.0
        self.fixed = (np.random.default_rng(seed).normal(-3.0, 0.3, size=(self.count, 1)).astype(np.float32)
                      if fixed is None else fixed)
        self.flat = PL.MLP.default_init(seed) if model == "mlp" else PL.default_init(seed)
        self.blob = pack_states(states).to(dev)
        self.info = self.blob.info.astype(np.int64)
        self.stage = self.info[:, 3]
        self.dev_args = tuple(t(x, dev) for x in (self.actions, self.adv, self.ret, self.fixed, self.exps))

    def engine(self, **kw):
        return Engine(self.dev, self.blob.n_cap, self.blob.e_cap, model=self.model, **kw)

    def step_args(self, sel=None):
        """The per-sample arrays and the minibatch's 1/B and 1/|ind| for the graphs `sel` (None: all of them)."""
        exps = self.exps if sel is None else self.exps[sel]
        return self.dev_args + (1.0 / len(exps), 1.0 / max(int((exps != 0).sum()), 1))

    def ids(self, sel):
        return None if sel is None else t(np.asarray(sel, np.int32), self.dev)


def nan_buffer(eng):
    """A gradient buffer whose every entry must be written by the step (NaN otherwise)."""
    return torch.full((eng.grad_stride,), float("nan"), dtype=torch.float32, device=eng.device)


def two_call_step(eng, case, params, sel=None):
    """ppo_grad + apply on the graphs `sel` (None: the whole blob, no index list); the gradient buffer."""
    g = nan_buffer(eng)
    eng.ppo_grad(case.blob, params, *case.step_args(sel), ids=case.ids(sel), out=g)
    eng.apply(params, g)
    return g


def fused_step(eng, case, params, sel=None):
    """ppo_step on the graphs `sel` (None: the whole blob, no index list); the gradient buffer."""
    g = nan_buffer(eng)
    eng.ppo_step(case.blob, params, *case.step_args(sel), ids=case.ids(sel), out=g)
    return g


def assert_same_state(e1, p1, g1, e2, p2, g2, what):
    """Bit for bit: the whole gradient / statistics buffer (every entry written), parameters, both Adam moments and
    the step counters.  Returns the step counters."""
    torch.cuda.synchronize()
    a, b = g1.cpu().numpy(), g2.cpu().numpy()
    assert np.isfinite(b).all(), (what, np.flatnonzero(~np.isfinite(b))[:8])
    assert np.array_equal(a, b), (what, np.flatnonzero(a != b)[:8])
    assert np.array_equal(p1.cpu().numpy(), p2.cpu().numpy()), what
    m1, v1, s1 = e1.get_opt_state()
    m2, v2, s2 = e2.get_opt_state()
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2), what
    assert s1.tolist() == s2.tolist(), (what, s1.tolist(), s2.tolist())
    return s2


# ---- stand-ins for the reference's agent -----------------------------------------------------------------------------
class Cfg:
    """The model specs of the reference's cfg; tests add the training attributes they need."""

    def __init__(self, n, e):
        self.state_encoder_specs = dict(state_encoder_hidden_size=[64, 16], gcn_node_dim=16, num_gcn_layers=2,
                                        num_edge_fc_layers=1, max_num_nodes=n, max_num_edges=e, num_attention_heads=1)
        self.policy_specs = dict(policy_land_use_head_hidden_size=[32, 1], policy_road_head_hidden_size=[32, 1])
        self.value_specs = dict(value_head_hidden_size=[32, 32, 1])


class Agent:
    node_dim, numerical_feature_size, dtype = 23, 52, torch.float32


def tensorfy(states):
    return [[torch.tensor(x) for x in s] for s in states]


SHIPPED_CFG = dict(lr=4e-4, eps=1e-5, clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01, gamma=0.99, tau=0.95,
                   num_optim_epoch=1, mini_batch_size=16)


def sgnn_agent(dev, n_cap, e_cap, flat, logged, **cfg):
    """A reference-shaped rl-sgnn agent as use_b200_update sees it: a cfg with SHIPPED_CFG's values unless `cfg` names
    others, the device, a tb_logger appending (tag, value, step) to `logged`, and actor-critic modules holding
    `flat`."""
    from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
    c = Cfg(n_cap, e_cap)
    c.agent_specs, c.agent = {}, "rl-sgnn"
    for k, v in {**SHIPPED_CFG, **cfg}.items():
        setattr(c, k, v)
    ag = Agent()
    ag.cfg, ag.device, ag.loss_iter = c, dev, 0
    ag.tb_logger = types.SimpleNamespace(add_scalar=lambda tag, v, s: logged.append((tag, v, s)))
    torch.manual_seed(0)
    p, v = create_sgnn_model(c, ag)
    ag.policy_net, ag.value_net, ag.actor_critic_net = p, v, ActorCritic(p, v)
    ag.actor_critic_net.load_flat_parameters(flat)
    return ag


# ---- worker processes ------------------------------------------------------------------------------------------------
def _stop(procs, grace):
    """Join every started process, terminating (then killing) whatever is still alive after `grace` seconds."""
    for p in procs:
        if p.pid is None:
            continue
        p.join(timeout=grace)
        if p.is_alive():
            p.terminate()
            p.join(timeout=30)
        if p.is_alive():
            p.kill()
            p.join()


def _spawned(target, rank, world, port, args, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    q.put((rank, target(rank, world, *args)))


def spawn(world, target, *args, timeout=600):
    """Run target(rank, world, *args) in `world` spawned processes, with MASTER_ADDR / MASTER_PORT set to a free local
    port for torch.distributed; {rank: what target returned}.  Raises as soon as a worker exits without a result, or
    after `timeout` seconds.  On every path each worker is joined, and terminated if it is still running, before this
    returns or raises."""
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_spawned, args=(target, r, world, port, args, q)) for r in range(world)]
    out = {}
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + timeout
        while len(out) < world:
            try:
                rank, res = q.get(timeout=1.0)
                out[rank] = res
            except queue.Empty:
                failed = [p.exitcode for p in procs if p.exitcode not in (None, 0)]
                assert not failed, f"a worker exited with code {failed} before returning its result"
                assert time.monotonic() < deadline, f"{world - len(out)} worker(s) gave no result within {timeout} s"
        return out
    finally:
        _stop(procs, 120 if len(out) == world else 0)


def _client(client, states, mean_action, q, wid):
    client.seed(100 + wid)
    got = [client.select_action([s], mean_action).numpy().copy() for s in states]
    q.put((wid, np.concatenate(got)))


def run_clients(server, per_worker, mean_action, timeout=120):
    """One forked rollout worker per entry of `per_worker`, each asking `server` for an action per state (worker w
    seeded with client.seed(100 + w)); {w: the actions it received}.  Every worker is joined, and terminated if it is
    still running, before this returns or raises."""
    import multiprocessing as mp
    ctx = mp.get_context("fork")
    q = ctx.Queue()
    procs = [ctx.Process(target=_client, args=(server.client(w), per_worker[w], mean_action, q, w))
             for w in range(len(per_worker))]
    res = {}
    try:
        for p in procs:
            p.start()
        for _ in procs:
            w, got = q.get(timeout=timeout)
            res[w] = got
        return res
    finally:
        _stop(procs, 30 if len(res) == len(procs) else 0)
