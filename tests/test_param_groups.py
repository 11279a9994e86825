"""CPU: parameter groups and frozen tensors (use_b200_update(param_groups=True)): live_param_groups maps agent.optimizer's
param_groups and requires_grad flags to the per-tensor table PPOUpdater.set_param_groups / Engine.set_param_groups pass
to the library, every ValueError comes before the library or the device is touched, the default path keeps refusing
groups that disagree on lr, and data-parallel ranks with different tables raise."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL
from drl_urban_planning_b200.agent import B200Update, live_hyperparameters, live_param_groups
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.ppo import PPOUpdater
from harness import SHIPPED_CFG, Agent, Cfg, sgnn_agent, spawn

ENCODER = {"sgnn": [n for n, s in PL.SGNN.slots.items() if s.owner == "enc"],
           "mlp": [n for n, s in PL.MLP.slots.items() if s.owner == "enc"]}


def agent(model):
    """A reference-shaped agent of `model` on the CPU, with setup_optimizer's Adam over actor_critic_net.parameters()."""
    if model == "sgnn":
        ag = sgnn_agent(torch.device("cpu"), 64, 64, PL.default_init(1), [])
    else:
        from drl_urban_planning_b200.mlp import ActorCritic, create_mlp_model
        c = Cfg(64, 64)
        c.agent, c.agent_specs = "rl-mlp", {}
        for k, v in SHIPPED_CFG.items():
            setattr(c, k, v)
        torch.manual_seed(5)
        p, v = create_mlp_model(c, Agent())
        ag = types.SimpleNamespace(cfg=c, actor_critic_net=ActorCritic(p, v), policy_net=p, value_net=v)
    ag.cfg.weightdecay = 0.0
    ag.optimizer = torch.optim.Adam(ag.actor_critic_net.parameters(), lr=ag.cfg.lr, eps=ag.cfg.eps)
    return ag


def layout(model):
    return PL.SGNN if model == "sgnn" else PL.MLP


def encoder_params(ag):
    return list(ag.actor_critic_net.actor_net.shared_net.parameters())


def head_params(ag):
    enc = {id(p) for p in encoder_params(ag)}
    return [p for p in ag.actor_critic_net.parameters() if id(p) not in enc]


def table(model, groups):
    """The per-tensor table of `groups` as PPOUpdater.set_param_groups forms it."""
    names = list(layout(model).slots)
    lr, wd, tr = [0.0] * len(names), [0.0] * len(names), [False] * len(names)
    for g in groups:
        for n in g["params"]:
            k = names.index(n)
            lr[k], wd[k], tr[k] = g["lr"], g["weight_decay"], True
    return lr, wd, tr


# ---- the mapping -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_one_group_trains_every_tensor(model):
    ag = agent(model)
    groups = live_param_groups(ag, layout(model))
    assert groups == [dict(params=list(layout(model).slots), lr=4e-4, weight_decay=0.0)]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_two_groups_with_their_own_lr_and_weight_decay(model):
    ag = agent(model)
    ag.optimizer = torch.optim.Adam([dict(params=encoder_params(ag), lr=1e-4, weight_decay=1e-4),
                                     dict(params=head_params(ag), lr=4e-4)], lr=ag.cfg.lr, eps=ag.cfg.eps)
    groups = live_param_groups(ag, layout(model))
    heads = [n for n in layout(model).slots if n not in ENCODER[model]]
    assert groups == [dict(params=ENCODER[model], lr=1e-4, weight_decay=1e-4),
                      dict(params=heads, lr=4e-4, weight_decay=0.0)]
    lr, wd, tr = table(model, groups)
    assert all(tr) and lr.count(1e-4) == len(ENCODER[model]) and wd.count(1e-4) == len(ENCODER[model])


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_requires_grad_false_on_the_shared_encoder_freezes_it(model):
    ag = agent(model)
    ag.actor_critic_net.actor_net.shared_net.requires_grad_(False)
    groups = live_param_groups(ag, layout(model))
    assert groups[0]["params"] == [n for n in layout(model).slots if n not in ENCODER[model]]
    _, _, tr = table(model, groups)
    assert [not x for x in tr] == [n in ENCODER[model] for n in layout(model).slots]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_optimizer_over_the_heads_only_freezes_the_encoder(model):
    ag = agent(model)
    ag.actor_critic_net.actor_net.shared_net.requires_grad_(False)    # else it would be trained outside any group
    ag.optimizer = torch.optim.Adam(head_params(ag), lr=2e-4, eps=ag.cfg.eps, weight_decay=1e-3)
    groups = live_param_groups(ag, layout(model))
    assert groups == [dict(params=[n for n in layout(model).slots if n not in ENCODER[model]], lr=2e-4,
                           weight_decay=1e-3)]


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_per_group_lambda_lr_after_a_step(model):
    ag = agent(model)
    ag.optimizer = torch.optim.Adam([dict(params=encoder_params(ag), lr=1e-4), dict(params=head_params(ag), lr=4e-4)],
                                    eps=ag.cfg.eps)
    sched = torch.optim.lr_scheduler.LambdaLR(ag.optimizer, [lambda it: 0.5 ** it, lambda it: 1.0 - it / 4])
    ag.optimizer.step()
    sched.step()
    groups = live_param_groups(ag, layout(model))
    assert [g["lr"] for g in groups] == [1e-4 * 0.5, 4e-4 * 0.75]


def test_the_default_path_still_refuses_groups_that_disagree_on_lr():
    ag = agent("sgnn")
    ag.optimizer = torch.optim.Adam([dict(params=encoder_params(ag), lr=1e-4), dict(params=head_params(ag), lr=4e-4)],
                                    eps=ag.cfg.eps)
    with pytest.raises(ValueError, match="disagree on lr"):
        live_hyperparameters(ag)
    assert "lr" not in live_hyperparameters(ag, param_groups=True)
    assert len(live_param_groups(ag, PL.SGNN)) == 2


# ---- ValueErrors, before the library or the device ---------------------------------------------------------------------
def _frozen_in_no_group(ag):
    ag.optimizer = torch.optim.Adam(head_params(ag), lr=4e-4, eps=ag.cfg.eps)      # the encoder keeps requires_grad


def _stranger(ag):
    ag.optimizer.add_param_group(dict(params=[torch.nn.Parameter(torch.zeros(3))]))


def _nothing_trained(ag):
    ag.actor_critic_net.requires_grad_(False)


def _set_all(key, value):
    return lambda ag: [g.__setitem__(key, value) for g in ag.optimizer.param_groups]


REFUSED = [
    (_frozen_in_no_group, "actor_net.shared_net.numerical_feature_encoder.linear_0.weight has requires_grad=True"),
    (_stranger, "not one of agent.actor_critic_net's"),
    (_nothing_trained, "trains no tensor"),
    (_set_all("betas", (0.8, 0.999)), "betas"),
    (_set_all("eps", 1e-8), "eps"),
    (_set_all("amsgrad", True), "amsgrad"),
    (_set_all("maximize", True), "maximize"),
    (_set_all("decoupled_weight_decay", True), "decoupled_weight_decay"),
    (_set_all("lr", -1e-4), "learning rate"),
    (_set_all("lr", float("nan")), "learning rate"),
    (_set_all("weight_decay", float("inf")), "weight_decay"),
]


class RecordingUpdater:
    """What B200Update.update_params calls on its updater, failing the test on any call."""

    def set_param_groups(self, groups):
        pytest.fail("the update passed a table to the library before checking it")

    set_hyperparameters = set_param_groups


@pytest.mark.parametrize("mutate, match", REFUSED)
def test_update_params_raises_before_cuda(mutate, match):
    ag = agent("sgnn")
    mutate(ag)
    ctl = B200Update.__new__(B200Update)
    ctl.agent, ctl.updater, ctl.layout, ctl.param_groups = ag, RecordingUpdater(), PL.SGNN, True
    ctl.updater.engine = types.SimpleNamespace(betas=(0.9, 0.999), eps=1e-5)
    ctl.push_weights = lambda: pytest.fail("the update touched the device before checking its groups")
    with pytest.raises(ValueError, match=match):
        ctl.update_params(types.SimpleNamespace(), 0)


def null_engine(model="sgnn", value_norm=False):
    """An Engine with a null context: a call that reached the library would raise UpbError."""
    eng = Engine.__new__(Engine)
    eng._ctx, eng.model, eng._p = C.c_void_p(), model, "upb_mlp_" if model == "mlp" else "upb_"
    eng.value_norm, eng.param_groups = value_norm, None
    return eng


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_engine_checks_the_table_before_the_library(model):
    n = len(layout(model).slots)
    eng = null_engine(model)
    with pytest.raises(ValueError, match=f"need {n} values"):
        eng.set_param_groups([4e-4] * (n - 1), [0.0] * n, [True] * n)
    with pytest.raises(ValueError, match="Invalid learning rate"):
        eng.set_param_groups([4e-4] * (n - 1) + [float("nan")], [0.0] * n, [True] * n)
    with pytest.raises(ValueError, match="Invalid weight_decay"):
        eng.set_param_groups([4e-4] * n, [0.0] * (n - 1) + [-1.0], [True] * n)
    with pytest.raises(ValueError, match="no tensor is trained"):
        eng.set_param_groups([4e-4] * n, [0.0] * n, [False] * n)
    vn = null_engine(model, value_norm=True)
    names = list(layout(model).slots)
    for frozen in ("val_w2", "val_b2"):
        tr = [name != frozen for name in names]
        with pytest.raises(ValueError, match=f"value_norm rescales {frozen}"):
            vn.set_param_groups([4e-4] * n, [0.0] * n, tr)
    with pytest.raises(_lib.UpbError, match="null context"):       # a valid table reaches the library
        eng.set_param_groups([4e-4] * n, [0.0] * n, [True] * n)
    assert eng.param_groups is None


class RecordingEngine:
    def __init__(self, model="sgnn"):
        self.model, self.lr, self.weight_decay, self.param_groups = model, 4e-4, 0.0, None
        self.layout = layout(model)
        self.calls = []

    def set_param_groups(self, lr, wd, trained):
        self.calls.append((lr, wd, trained))
        self.param_groups = (lr, wd, trained)


def recording_updater(model="sgnn"):
    up = PPOUpdater.__new__(PPOUpdater)
    up.engine, up.param_groups = RecordingEngine(model), True
    return up


def test_updater_groups_issue_one_call_per_change_and_check_first():
    up = recording_updater()
    names = list(PL.SGNN.slots)
    every = [dict(params=names, lr=4e-4)]
    up.set_param_groups(every)
    up.set_param_groups(every)                                   # unchanged: no call
    assert len(up.engine.calls) == 1 and up.engine.calls[0][2] == (True,) * 32
    heads = [dict(params=names[20:], lr=4e-4, weight_decay=1e-3)]
    up.set_param_groups(heads)
    assert up.engine.calls[1][2] == (False,) * 20 + (True,) * 12 and up.engine.calls[1][1][20:] == (1e-3,) * 12
    for bad, match in [([dict(params=["nope"], lr=1e-3)], "unknown tensor"),
                       ([dict(params=names, lr=1e-3), dict(params=names[:1], lr=1e-3)], "more than one group"),
                       ([dict(params=names, lr=-1.0)], "learning rate"),
                       ([dict(params=names, lr=1e-3, weight_decay=float("nan"))], "weight_decay")]:
        with pytest.raises(ValueError, match=match):
            up.set_param_groups(bad)
    assert len(up.engine.calls) == 2
    with pytest.raises(ValueError, match="each tensor's lr and weight_decay"):
        up.set_hyperparameters(lr=1e-3)
    with pytest.raises(ValueError, match="each tensor's lr and weight_decay"):
        up.set_hyperparameters(weight_decay=0.0)
    off = recording_updater()
    off.param_groups = False
    with pytest.raises(ValueError, match="param_groups=True"):
        off.set_param_groups(every)


def test_engine_lr_and_weight_decay_setters_refuse_a_table():
    eng = null_engine()
    eng.param_groups = ((4e-4,) * 32, (0.0,) * 32, (True,) * 32)
    with pytest.raises(ValueError, match="parameter groups"):
        eng.set_lr(1e-3)
    with pytest.raises(ValueError, match="parameter groups"):
        eng.set_weight_decay(0.0)


# ---- two gloo ranks ----------------------------------------------------------------------------------------------------
def _rank_worker(rank, world):
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    T = 12
    info = np.stack([np.arange(T) + 5, np.arange(T) * 3, np.arange(T) % 7, np.arange(T) % 2], 1).astype(np.int64)
    up = recording_updater()
    up.world, up.rank, up.pg, up.device = world, rank, None, torch.device("cpu")
    up.exps_host, up.actions = np.ones(T, np.float32), torch.zeros(T, 2)
    names = list(PL.SGNN.slots)
    out = []
    for groups in ([dict(params=names, lr=4e-4)],
                   [dict(params=names[20:] if rank else names, lr=4e-4)],                 # rank 1 freezes the encoder
                   [dict(params=names[:20], lr=1e-4 * (1 + rank)), dict(params=names[20:], lr=4e-4)]):
        up.set_param_groups(groups)
        try:
            PPOUpdater._check_same_buffer(up, info, up._param_group_signature())
            out.append(None)
        except _lib.UpbError as e:
            out.append(str(e))
    dist.destroy_process_group()
    return out


def test_ranks_with_different_tables_raise():
    res = spawn(2, _rank_worker, timeout=300)
    for r in (0, 1):
        same, frozen, lr = res[r]
        assert same is None
        assert "different hyperparameters" in frozen and "trained[num_w0]" in frozen
        assert "(lr[num_w0], lr[num_b0]" in lr
