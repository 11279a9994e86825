"""CPU: the KL penalty's argument checks, the adaptive coefficient on synthetic statistics rows, its log tags and
checkpoint round trip, and the float64 oracle (tests/ppo_oracle.py) against torch autograd and finite differences."""
import types

import numpy as np
import pytest
import torch

import klpen_oracle as KO
import ppo_oracle as PPO
from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine, adapt_kl_coef, check_kl_penalty
from drl_urban_planning_b200.ppo import KL_STOP_SLOT, KL_SKIP_SLOT, KLPEN_SLOT, PPOUpdater, UpdateLog
from harness import Cfg, per_tensor_rel, rel
from oracle import mlp_port as MP
from oracle import torch_port as TP

BAD = [0.0, -0.1, float("nan"), float("inf"), -float("inf")]


def test_check_kl_penalty_values():
    assert check_kl_penalty(None) == (0.0, 0.0)
    assert check_kl_penalty(0.2) == (0.2, 0.0) and check_kl_penalty(np.float32(1.0), 0.01) == (1.0, 0.01)
    for bad in BAD:
        with pytest.raises(ValueError, match="kl_coef"):
            check_kl_penalty(bad)
        with pytest.raises(ValueError, match="kl_target"):
            check_kl_penalty(0.2, bad)
    with pytest.raises(ValueError, match="kl_target"):
        check_kl_penalty(None, 0.01)


def no_cuda(*a, **k):
    raise AssertionError("reached CUDA")


@pytest.mark.parametrize("kw", [dict(kl_coef=b) for b in BAD] + [dict(kl_coef=0.2, kl_target=b) for b in BAD]
                         + [dict(kl_target=0.01)])
def test_bad_kl_penalty_is_rejected_before_any_cuda_call(kw, monkeypatch):
    monkeypatch.setattr(_lib, "lib", no_cuda)
    if "kl_target" not in kw:
        with pytest.raises(ValueError, match="kl_coef"):
            Engine("cuda:0", 16, 16, **kw)
    with pytest.raises(ValueError, match="kl_"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", **kw)
    from drl_urban_planning_b200.agent import B200Update
    for kind in ("rl-sgnn", "rl-mlp"):
        cfg = Cfg(64, 64)
        cfg.agent, cfg.clip_epsilon = kind, 0.2
        with pytest.raises(ValueError, match="kl_"):
            B200Update(types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0)), **kw)


def test_c_entry_point_validates_without_a_context():
    import ctypes as C
    L = _lib.lib()
    assert L.upb_set_kl_penalty(None, C.c_float(0.2)) == -1 and b"set_kl_penalty" in L.upb_last_error()


# ---- the adaptive coefficient on synthetic statistics rows -----------------------------------------------------------
def kl_rows(nb, d, n_ind=28, seed=0):
    """nb statistics rows with n_ind graphs in ind each and a mean exact KL of d over the whole epoch."""
    rng = np.random.default_rng(seed)
    st = np.zeros((nb, 19))
    st[:, 1] = rng.normal(size=nb)
    st[:, 2] = -rng.random(nb) * 30
    st[:, 3], st[:, 4] = 32, n_ind
    w = rng.random(nb) + 0.5
    st[:, KLPEN_SLOT] = d * n_ind * nb * w / w.sum()
    return st


@pytest.mark.parametrize("d,factor", [(0.001, 0.5), (0.0066, 0.5), (0.007, 1.0), (0.01, 1.0), (0.0149, 1.0),
                                      (0.0151, 2.0), (0.2, 2.0)])
def test_adaptation_rule(d, factor):
    target, beta = 0.01, 0.3
    book = UpdateLog(2, 0.5, 0.01, kl_coef=beta)
    book.epoch(0, kl_rows(4, 10 * d, seed=1))      # an earlier epoch does not count
    book.epoch(1, kl_rows(4, d, seed=2))
    assert adapt_kl_coef(beta, *book.kl_rows, target) == beta * factor


def test_adaptation_keeps_beta_without_graphs_in_ind():
    book = UpdateLog(1, 0.5, 0.01, kl_coef=0.3)
    book.epoch(0, kl_rows(3, 0.5, n_ind=0))
    assert book.kl_rows[1] == 0 and adapt_kl_coef(0.3, *book.kl_rows, 0.01) == 0.3
    assert adapt_kl_coef(0.3, float("nan"), 5.0, 0.01) == 0.3


def test_adaptation_with_a_kl_stop_mid_epoch():
    """The KL stop ends the update at row 2 of epoch 1 (slot 13 on the stopping row, slot 14 on the skipped ones): d is
    measured over rows 0-2 of that epoch, the stopping step's row included, the skipped rows (all zeros) not."""
    target, beta = 0.01, 0.3
    book = UpdateLog(3, 0.5, 0.01, kl_stop=True, kl_coef=beta)
    assert not book.epoch(0, kl_rows(5, 0.001, seed=3))
    st = kl_rows(5, 0.0, seed=4)
    st[:3, KLPEN_SLOT] = [0.1 * 28, 0.5 * 28, 1.2 * 28]       # d = 0.6 over rows 0-2
    st[2, KL_STOP_SLOT] = 1.0
    st[3:] = 0.0
    st[3:, KL_SKIP_SLOT] = 1.0
    assert book.epoch(1, st)
    assert book.kl_rows == (pytest.approx(1.8 * 28), 3 * 28)
    assert adapt_kl_coef(beta, *book.kl_rows, target) == 2 * beta
    assert adapt_kl_coef(beta, *book.kl_rows, 0.5) == beta
    assert adapt_kl_coef(beta, *book.kl_rows, 2.0) == beta / 2


@pytest.mark.parametrize("beta", [None, 0.25])
def test_update_log_tags_and_totals(beta):
    VC, EC = 0.5, 0.01
    logged = []
    book = UpdateLog(2, VC, EC, 3, 10, lambda t, v, s: logged.append((t, v, s)), kl_coef=beta)
    eps = [kl_rows(3, 0.02 * (e + 1), seed=e) for e in range(2)]
    for e, st in enumerate(eps):
        book.epoch(e, st)
    out = book.finish(False)
    st = np.concatenate(eps)
    kl = st[:, KLPEN_SLOT] / 28
    loss = st[:, 1] / 28 + VC * st[:, 0] / 32 + EC * st[:, 2] / 28 + (beta or 0.0) * kl
    assert np.allclose([v for t, v, _ in logged if t == "loss/loss"], loss)
    if beta is None:
        ref = []
        plain = UpdateLog(2, VC, EC, 3, 10, lambda t, v, s: ref.append((t, v, s)))
        for e, st_e in enumerate(eps):
            plain.epoch(e, st_e)
        assert plain.finish(False) == out and ref == logged
        assert not any(t.startswith("loss/kl") or "kl_loss" in t or t == "diag/kl_coef" for t, _, _ in logged)
        return
    got = [(v, s) for t, v, s in logged if t == "loss/kl_loss"]
    assert np.allclose([v for v, _ in got], kl) and [s for _, s in got] == list(range(10, 16))
    ep = [(v, s) for t, v, s in logged if t == "loss/epoch_kl_loss"]
    assert np.allclose([v for v, _ in ep], [kl[:3].sum(), kl[3:].sum()]) and [s for _, s in ep] == [6, 7]
    assert [(t, s) for t, _, s in logged if t in ("loss/total_kl_loss", "diag/kl_coef")] == [
        ("loss/total_kl_loss", 3), ("diag/kl_coef", 3)]
    assert np.isclose(out["total_kl_loss"], kl.sum() / 2) and out["kl_coef"] == beta
    assert [v for t, v, _ in logged if t == "diag/kl_coef"] == [beta]
    assert np.isclose(out["total_loss"], loss.sum() / 2)


# ---- checkpoint round trip of beta (no device: the engine is a recording stand-in) ----------------------------------
class FakeEngine:
    def __init__(self):
        self.kl_coef = None

    def get_opt_state(self):
        return np.zeros(3, np.float32), np.ones(3, np.float32), np.array([5, 5, 2, 3])

    def set_opt_state(self, m, v, steps, rearm_first_step_clip=False):
        self.restored = (m, v, steps)

    def set_kl_coef(self, beta):
        self.kl_coef = beta


def controller(beta0, beta):
    from drl_urban_planning_b200.agent import B200Update
    up = PPOUpdater.__new__(PPOUpdater)
    up.engine, up.kl_coef_init, up.kl_coef = FakeEngine(), beta0, beta
    ctl = B200Update.__new__(B200Update)
    ctl.updater = up
    return ctl


def test_checkpoint_carries_beta():
    state = controller(0.1, 0.4).optimizer_state()
    assert state["kl_coef"] == 0.4
    ctl = controller(0.1, 0.1)
    ctl.load_optimizer_state(state)
    assert ctl.updater.kl_coef == 0.4 and ctl.updater.engine.kl_coef == 0.4
    old = {k: v for k, v in state.items() if k != "kl_coef"}          # a checkpoint written without the penalty
    ctl = controller(0.1, 0.8)
    ctl.load_optimizer_state(old)
    assert ctl.updater.kl_coef == 0.1 and ctl.updater.engine.kl_coef == 0.1
    off = controller(None, None)
    assert "kl_coef" not in off.optimizer_state()
    off.load_optimizer_state(state)                                     # the penalty stays off
    assert off.updater.kl_coef is None and off.updater.engine.kl_coef is None


# ---- the oracle ---------------------------------------------------------------------------------------------------------
def test_per_candidate_seed_against_autograd():
    rng = np.random.default_rng(3)
    for k, spread in ((1, 1.0), (7, 1.0), (40, 5.0), (12, 80.0)):
        zo, zn = rng.normal(0, spread, k), rng.normal(0, spread, k)
        zn[0] = zo[0] - 150.0 if k > 1 else zn[0]          # a new probability that underflows in fp32
        lo = torch.log_softmax(torch.tensor(zo), -1)
        z = torch.tensor(zn, requires_grad=True)
        kl = KO.kl_rows(lo, torch.log_softmax(z, -1))
        kl.backward()
        want_kl, seed = PPO.kl64(lo.numpy(), torch.log_softmax(torch.tensor(zn), -1).numpy())
        assert np.isclose(kl.item(), want_kl, rtol=1e-12, atol=1e-15) and np.isfinite(want_kl)
        assert np.allclose(z.grad.numpy(), seed, rtol=1e-10, atol=1e-14)
    assert PPO.kl64(np.zeros(0), np.zeros(0))[0] == 0.0                 # k = 0: no term
    lo = np.array([0.0, -800.0])                                       # p_old underflows to 0 in float64: adds 0
    assert PPO.kl64(lo, np.array([-1e-3, -7.0]))[0] == pytest.approx(1e-3)


def sgnn_case(seed=4, count=8):
    states, actions = synth.make_states(seed, "small", count, stages=[i % 2 for i in range(count)])
    adv, ret, exps = synth.make_ppo_targets(seed, count)
    exps[1] = 0.0
    fixed = np.random.default_rng(seed).normal(-3.0, 0.3, size=(count, 1)).astype(np.float32)
    flat0 = PL.default_init(seed)
    flat1 = (flat0 + np.random.default_rng(seed + 1).normal(0, 0.05, flat0.shape)).astype(np.float32)
    return states, actions, adv, ret, exps, fixed, flat0, flat1


def test_sgnn_oracle_gradient_against_torch_autograd():
    """The float64 oracle with beta * kl against autograd of the torch form (oracle/torch_port, fp32) at the policy the
    update moved to (flat1) with the pre-pass at flat0; the penalty's gradient is far above the tolerance."""
    states, actions, adv, ret, exps, fixed, flat0, flat1 = sgnn_case()
    beta = 2.0
    lp_old = KO.cand_logp64(flat0.astype(np.float64), states)
    r = PPO.sgnn_minibatch(flat1.astype(np.float64), states, actions, adv, ret, fixed, exps, lp_old=lp_old,
                           kl_coef=beta)
    agent = PPO.PortAgent(flat0, kl_coef=beta)
    agent.snapshot()
    agent.P = {k: torch.tensor(flat1[s.offset:s.offset + s.size].reshape(s.shape), requires_grad=True)
               for k, s in PL.SLOTS.items()}
    agent.opt = torch.optim.Adam(list(agent.P.values()))
    b = TP.stack_states(states)
    ind = torch.tensor(exps).nonzero(as_tuple=False).squeeze(1)
    losses = agent.backward(b, torch.tensor(actions), torch.tensor(adv), torch.tensor(ret), torch.tensor(fixed), ind)
    worst, where = per_tensor_rel(agent.flat_grad(), r["grad"])
    assert worst < 1e-4, (worst, where)
    assert np.allclose(losses, [r["loss"], r["value_loss"], r["surr_loss"], r["entropy_loss"]], rtol=1e-5, atol=1e-6)
    assert np.isclose(agent.last_kl, r["kl_loss"], rtol=1e-4) and r["kl_loss"] > 1e-4
    r0 = PPO.sgnn_minibatch(flat1.astype(np.float64), states, actions, adv, ret, fixed, exps, lp_old=lp_old)
    assert per_tensor_rel(r0["grad"], r["grad"])[0] > 1e-2


def test_sgnn_oracle_penalty_gradient_against_finite_differences():
    states, actions, adv, ret, exps, fixed, flat0, flat1 = sgnn_case(6, 6)
    beta = 1.0
    f0, f1 = flat0.astype(np.float64), flat1.astype(np.float64)
    lp_old = KO.cand_logp64(f0, states)
    ind = np.flatnonzero(exps != 0)
    args = (states, actions, adv, ret, fixed, exps)
    g = PPO.sgnn_minibatch(f1, *args, lp_old=lp_old, kl_coef=beta)["grad"] - PPO.sgnn_minibatch(f1, *args)["grad"]

    def kl(f):
        lp = KO.cand_logp64(f, states)
        return beta * sum(PPO.kl64(lp_old[i], lp[i])[0] for i in ind) / len(ind)

    rng = np.random.default_rng(0)
    picks = [PL.SLOTS[n].offset + int(rng.integers(PL.SLOTS[n].size))
             for n in ("lu_w1", "lu_w0", "road_w0", "road_b0", "gcn1_w", "enc_w", "att_q_w", "mha_out_w")]
    h = 1e-6
    for j in picks:
        e = np.zeros_like(f1)
        e[j] = h
        fd = (kl(f1 + e) - kl(f1 - e)) / (2 * h)
        assert abs(fd - g[j]) <= 1e-6 + 1e-4 * abs(fd), (j, fd, g[j])
    assert np.abs(g).max() > 1e-3


def test_mlp_torch_form_against_finite_differences_in_float64():
    states, actions = synth.make_states(8, "small", 6, stages=[i % 2 for i in range(6)])
    flat0 = PL.MLP.default_init(8).astype(np.float64)
    flat1 = flat0 + np.random.default_rng(9).normal(0, 0.05, flat0.shape)
    b = MP.stack_states(states)
    P0, P1 = KO.mlp_params64(flat0), KO.mlp_params64(flat1, requires_grad=True)
    kl = KO.mlp_kl(P1, P0, b)
    kl.sum().backward()
    lp_old, lp_new = KO.mlp_cand_logp64(flat0, states), KO.mlp_cand_logp64(flat1, states)
    want = [PPO.kl64(lp_old[i], lp_new[i])[0] for i in range(len(states))]
    assert np.allclose(kl.detach().numpy(), want, rtol=1e-10, atol=1e-14) and max(want) > 1e-4
    grad = np.zeros(PL.MLP.num_params)
    for s in PL.MLP.slots.values():
        if P1[s.name].grad is not None:
            grad[s.offset:s.offset + s.size] = P1[s.name].grad.numpy().reshape(-1)
    rng = np.random.default_rng(1)
    h = 1e-6
    for name in ("lu_w1", "lu_w0", "road_w0", "enc_w"):
        j = PL.MLP.slots[name].offset + int(rng.integers(PL.MLP.slots[name].size))
        e = np.zeros_like(flat1)
        e[j] = h
        fd = (sum(PPO.kl64(lp_old[i], x)[0] for i, x in enumerate(KO.mlp_cand_logp64(flat1 + e, states)))
              - sum(PPO.kl64(lp_old[i], x)[0] for i, x in enumerate(KO.mlp_cand_logp64(flat1 - e, states)))) / (2 * h)
        assert abs(fd - grad[j]) <= 1e-7 + 1e-5 * abs(fd), (name, fd, grad[j])


def test_cand_positions_round_trip():
    from drl_urban_planning_b200.packing import pack_states
    states, _ = synth.make_states(2, "small", 7, stages=[i % 2 for i in range(7)])
    blob = pack_states(states, pinned=False)
    lp = KO.cand_logp64(PL.default_init(2).astype(np.float64), states)
    flat = KO.to_positions(lp, blob)
    assert flat.shape == (blob.cand_len,)
    back = KO.per_graph(flat, blob)
    for i, st in enumerate(states):
        mask = st[6] if int(np.argmax(st[8][:2])) == 0 else st[7]
        assert np.array_equal(back[i][1], np.flatnonzero(mask))
        assert np.allclose(back[i][0], lp[i], rtol=1e-6, atol=1e-6)
