"""CPU: the hyperparameters an update reads from the agent (B200Update.update_params -> live_hyperparameters ->
PPOUpdater.set_hyperparameters), as the reference's update_params / update_policy read them at every update: the values
and their cfg fallbacks, every ValueError before the library or the device is touched, the calls a change issues (and
that no change issues none), the loss coefficients of UpdateLog, and the cross-rank check on two gloo ranks."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.agent import B200Update, live_hyperparameters
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.ppo import PPOUpdater, UpdateLog
from harness import SHIPPED_CFG, Cfg, spawn


class RecordingEngine:
    """The Python face of Engine that set_hyperparameters uses, recording the library calls it would make."""

    def __init__(self, lr=4e-4, clip_epsilon=0.2, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-5):
        self.lr, self.clip_epsilon, self.weight_decay, self.betas, self.eps = lr, clip_epsilon, weight_decay, betas, eps
        self.calls = []

    def set_lr(self, lr):
        self.calls.append(("lr", lr)); self.lr = lr

    def set_clip_epsilon(self, eps):
        self.calls.append(("clip_epsilon", eps)); self.clip_epsilon = eps

    def set_loss_coefs(self, v, e):
        self.calls.append(("loss_coefs", v, e))

    def set_weight_decay(self, wd):
        self.calls.append(("weight_decay", wd)); self.weight_decay = wd


def updater(**cfg):
    """A PPOUpdater at SHIPPED_CFG's values (or `cfg`'s) whose engine records calls instead of making them."""
    c = {**SHIPPED_CFG, **cfg}
    up = PPOUpdater.__new__(PPOUpdater)
    up.engine = RecordingEngine(lr=c["lr"], clip_epsilon=c["clip_epsilon"], eps=c["eps"])
    up.value_pred_coef, up.entropy_coef = c["value_pred_coef"], c["entropy_coef"]
    up.gamma, up.tau, up.opt_num_epochs, up.mini_batch_size = c["gamma"], c["tau"], c["num_optim_epoch"], c["mini_batch_size"]
    return up


def ref_agent(with_attributes=True, **opt_kw):
    """A reference-shaped agent: the cfg, and (with_attributes) the attributes UrbanPlanningAgent.__init__ hands its
    base classes plus the torch.optim.Adam of setup_optimizer (urban_planning_agent.py:145-149)."""
    cfg = Cfg(64, 64)
    for k, v in SHIPPED_CFG.items():
        setattr(cfg, k, v)
    cfg.agent, cfg.weightdecay = "rl-sgnn", 0.0
    ag = types.SimpleNamespace(cfg=cfg)
    if with_attributes:
        ag.gamma, ag.tau, ag.clip_epsilon = cfg.gamma, cfg.tau, cfg.clip_epsilon
        ag.value_pred_coef, ag.entropy_coef = cfg.value_pred_coef, cfg.entropy_coef
        ag.opt_num_epochs, ag.mini_batch_size = cfg.num_optim_epoch, cfg.mini_batch_size
        net = torch.nn.Linear(3, 2)
        kw = dict(lr=cfg.lr, eps=cfg.eps, weight_decay=cfg.weightdecay, **opt_kw)
        ag.optimizer = torch.optim.Adam([{"params": [net.weight]}, {"params": [net.bias]}], **kw)
    return ag


# ---- reading the live values -----------------------------------------------------------------------------------------
def test_stand_in_agent_falls_back_to_the_cfg():
    """tests/harness.py's stand-ins have no optimizer and none of the attributes: every value is the cfg's."""
    ag = ref_agent(with_attributes=False)
    got = live_hyperparameters(ag)
    assert got == dict(lr=4e-4, weight_decay=0.0, clip_epsilon=0.2, value_pred_coef=0.5, entropy_coef=0.01,
                       gamma=0.99, tau=0.95, opt_num_epochs=1, mini_batch_size=16)
    ag.cfg.weightdecay = 1e-3
    assert live_hyperparameters(ag)["weight_decay"] == 1e-3


def test_reference_agent_values_are_read_where_the_reference_reads_them():
    ag = ref_agent()
    assert live_hyperparameters(ag) == live_hyperparameters(ref_agent(with_attributes=False))
    ag.entropy_coef, ag.clip_epsilon, ag.value_pred_coef = 0.003, 0.1, 0.25
    ag.gamma, ag.tau, ag.opt_num_epochs, ag.mini_batch_size = 0.9, 0.5, 3, 8
    for g in ag.optimizer.param_groups:
        g["weight_decay"] = 1e-4
    # CleanRL's anneal_lr: frac = 1 - (iteration - 1) / num_iterations, as a LambdaLR
    sched = torch.optim.lr_scheduler.LambdaLR(ag.optimizer, lambda it: 1.0 - it / 10)
    ag.optimizer.step()
    sched.step()
    got = live_hyperparameters(ag)
    assert got == dict(lr=4e-4 * 0.9, weight_decay=1e-4, clip_epsilon=0.1, value_pred_coef=0.25, entropy_coef=0.003,
                       gamma=0.9, tau=0.5, opt_num_epochs=3, mini_batch_size=8)
    # ReduceLROnPlateau lowers lr by its factor once the metric stops improving
    plateau = torch.optim.lr_scheduler.ReduceLROnPlateau(ag.optimizer, factor=0.2, patience=0)
    plateau.step(1.0)
    plateau.step(2.0)
    assert live_hyperparameters(ag)["lr"] == pytest.approx(4e-4 * 0.9 * 0.2, rel=1e-15)


def test_lr_given_as_a_tensor_is_read_as_a_float():
    ag = ref_agent()
    for g in ag.optimizer.param_groups:
        g["lr"] = torch.tensor(3e-4, dtype=torch.float64)
    assert live_hyperparameters(ag)["lr"] == 3e-4


# ---- ValueErrors, before the library or the device ---------------------------------------------------------------------
@pytest.mark.parametrize("mutate, match", [
    (lambda o: o.param_groups[1].__setitem__("lr", 1e-3), "disagree on lr"),
    (lambda o: o.param_groups[0].__setitem__("weight_decay", 1e-2), "disagree on weight_decay"),
    (lambda o: [g.__setitem__("betas", (0.8, 0.999)) for g in o.param_groups], "betas"),
    (lambda o: [g.__setitem__("eps", 1e-8) for g in o.param_groups], "eps"),
    (lambda o: [g.__setitem__("amsgrad", True) for g in o.param_groups], "amsgrad"),
    (lambda o: [g.__setitem__("maximize", True) for g in o.param_groups], "maximize"),
    (lambda o: [g.__setitem__("lr", -1e-4) for g in o.param_groups], "learning rate"),
    (lambda o: [g.__setitem__("lr", float("nan")) for g in o.param_groups], "learning rate"),
    (lambda o: [g.__setitem__("lr", float("inf")) for g in o.param_groups], "learning rate"),
    (lambda o: [g.__setitem__("weight_decay", -1.0) for g in o.param_groups], "weight_decay"),
])
def test_update_params_raises_before_cuda(mutate, match):
    """B200Update.update_params reads and checks every value before it touches the weights, the library or the device
    (push_weights is its first device work), and a refused update changes nothing."""
    ag = ref_agent()
    mutate(ag.optimizer)
    ctl = B200Update.__new__(B200Update)
    ctl.agent, ctl.updater = ag, updater()
    ctl.push_weights = lambda: pytest.fail("the update touched the device before checking its values")
    before = ctl.updater.hyperparameters()
    with pytest.raises(ValueError, match=match):
        ctl.update_params(types.SimpleNamespace(), 0)
    assert ctl.updater.engine.calls == [] and ctl.updater.hyperparameters() == before


BAD = [("lr", -1e-3), ("lr", float("nan")), ("clip_epsilon", -0.1), ("clip_epsilon", float("inf")),
       ("value_pred_coef", float("nan")), ("entropy_coef", float("-inf")), ("weight_decay", -1.0),
       ("gamma", float("nan")), ("tau", float("inf")), ("opt_num_epochs", 0), ("opt_num_epochs", 2.0),
       ("opt_num_epochs", True), ("mini_batch_size", 0), ("mini_batch_size", 16.5)]


@pytest.mark.parametrize("name, bad", BAD)
def test_set_hyperparameters_checks_every_value_first(name, bad):
    """One invalid value among valid changes: ValueError, no call, no value changed."""
    up = updater()
    before = up.hyperparameters()
    kw = dict(lr=1e-3, clip_epsilon=0.3, entropy_coef=0.0, weight_decay=1e-3, opt_num_epochs=2)
    kw[name] = bad
    with pytest.raises(ValueError):
        up.set_hyperparameters(**kw)
    assert up.engine.calls == [] and up.hyperparameters() == before


@pytest.mark.parametrize("bad", [-1e-3, float("nan"), float("inf")])
def test_engine_rejects_invalid_lr_before_the_library(bad):
    """Engine(lr=...) and Engine.set_lr check before any CUDA call; set_lr's message is torch.optim.Adam's."""
    with pytest.raises(ValueError, match="Invalid learning rate"):
        Engine("cuda:0", 64, 64, lr=bad)
    eng = Engine.__new__(Engine)
    eng._ctx = C.c_void_p()                       # a null context: a call that reached the library would raise UpbError
    with pytest.raises(ValueError, match="Invalid learning rate"):
        eng.set_lr(bad)
    if not math.isfinite(bad):                    # any finite coefficient is accepted
        with pytest.raises(ValueError, match="value_pred_coef"):
            eng.set_loss_coefs(bad, 0.01)
        with pytest.raises(ValueError, match="entropy_coef"):
            eng.set_loss_coefs(0.5, bad)
    with pytest.raises(ValueError, match="clip_epsilon"):
        eng.set_clip_epsilon(bad)
    with pytest.raises(ValueError, match="weight_decay"):
        eng.set_weight_decay(bad)


def test_library_refuses_invalid_values_and_a_null_context():
    """The C entry points refuse a null context; the Python checks let lr = 0 and a negative coefficient through."""
    L = _lib.lib()
    assert L.upb_set_lr(None, 1e-3) == -1 and L.upb_set_loss_coefs(None, 0.5, 0.01) == -1       # UPB_ERR_ARG
    eng = Engine.__new__(Engine)
    eng._ctx = C.c_void_p()
    with pytest.raises(_lib.UpbError, match="null context"):
        eng.set_lr(0.0)                           # lr = 0 passes the Python check (moments and counters still advance)
    with pytest.raises(_lib.UpbError, match="null context"):
        eng.set_loss_coefs(-1.0, 0.0)             # any finite coefficient passes


# ---- what a change issues -----------------------------------------------------------------------------------------------
def test_unchanged_values_issue_no_call():
    """Values equal to the Python values last passed: nothing is called.  The cfg's 4e-4 is compared as the Python float
    it is, not as the fp32 number the context holds."""
    up = updater()
    up.set_hyperparameters(**live_hyperparameters(ref_agent()))
    up.set_hyperparameters()
    assert up.engine.calls == []


def test_each_change_issues_its_own_call():
    up = updater()
    up.set_hyperparameters(lr=3.7e-4)
    up.set_hyperparameters(entropy_coef=0.0, gamma=0.9)
    up.set_hyperparameters(clip_epsilon=0.18, weight_decay=1e-2, opt_num_epochs=3, mini_batch_size=8, tau=0.5)
    up.set_hyperparameters(value_pred_coef=1.0)
    assert up.engine.calls == [("lr", 3.7e-4), ("loss_coefs", 0.5, 0.0), ("clip_epsilon", 0.18),
                               ("weight_decay", 1e-2), ("loss_coefs", 1.0, 0.0)]
    assert up.hyperparameters() == dict(lr=3.7e-4, clip_epsilon=0.18, value_pred_coef=1.0, entropy_coef=0.0,
                                        weight_decay=1e-2, gamma=0.9, tau=0.5, opt_num_epochs=3, mini_batch_size=8)


def test_update_log_forms_losses_with_the_update_coefficients():
    """The update's UpdateLog is built from the updater's coefficients at its start, so the logged loss of each update is
    surr + value_pred_coef * value + entropy_coef * entropy with that update's values."""
    rows = np.zeros((2, 20))
    rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3], rows[:, 4] = [8.0, 4.0], [1.0, -2.0], [-30.0, -20.0], 4, 2
    up = updater()
    got = []
    for coefs in [(0.5, 0.01), (1.0, 0.05), (0.25, 0.0)]:
        up.set_hyperparameters(value_pred_coef=coefs[0], entropy_coef=coefs[1])
        logged = []
        book = UpdateLog(up.opt_num_epochs, up.value_pred_coef, up.entropy_coef,
                         log_fn=lambda tag, v, s: logged.append((tag, v, s)))
        book.epoch(0, rows)
        got.append([v for tag, v, s in logged if tag == "loss/loss"])
        want = rows[:, 1] / 2 + coefs[0] * rows[:, 0] / 4 + coefs[1] * rows[:, 2] / 2
        assert np.allclose(got[-1], want, rtol=0, atol=1e-12), coefs
        assert book.finish(False)["total_loss"] == pytest.approx(want.sum())


# ---- two gloo ranks ----------------------------------------------------------------------------------------------------
def _rank_worker(rank, world):
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    T = 12
    info = np.stack([np.arange(T) + 5, np.arange(T) * 3, np.arange(T) % 7, np.arange(T) % 2], 1).astype(np.int64)
    duck = types.SimpleNamespace(world=world, rank=rank, pg=None, device=torch.device("cpu"),
                                 exps_host=np.ones(T, np.float32), actions=torch.zeros(T, 2))
    up = updater()
    out = []
    for change in [{}, dict(lr=4e-4 * (0.5 if rank else 1.0)), dict(lr=2e-4, entropy_coef=0.02 if rank else 0.01,
                                                                      mini_batch_size=8 + rank)]:
        up.set_hyperparameters(**change)
        try:
            PPOUpdater._check_same_buffer(duck, info, up.hyperparameters())
            out.append(None)
        except _lib.UpbError as e:
            out.append(str(e))
    dist.destroy_process_group()
    return out


def test_ranks_with_different_hyperparameters_raise():
    """A ReduceLROnPlateau fed per-rank rewards gives the ranks different lr: the signature check of load_states, which
    runs before the update's first step, raises on every rank and names what differs."""
    res = spawn(2, _rank_worker, timeout=300)
    for r in (0, 1):
        same, lr, two = res[r]
        assert same is None
        assert "different hyperparameters (lr differ)" in lr
        assert "(entropy_coef, mini_batch_size differ)" in two
