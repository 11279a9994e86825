"""CPU: the KL stop's argument checks (Engine, PPOUpdater, upb_set_target_kl) and the update's host bookkeeping of the
statistics rows the step kernels mark with slot 13 (the step that stopped) and slot 14 (steps skipped after it)."""
import numpy as np
import pytest

from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.diagnostics import NAMES
from drl_urban_planning_b200.engine import Engine, check_target_kl
from drl_urban_planning_b200.ppo import KL_SKIP_SLOT, KL_STOP_SLOT, UpdateLog

BAD = [-1.0, -1e-30, float("nan"), float("inf"), -float("inf")]
VC, EC = 0.5, 0.01


def test_check_target_kl_values():
    assert check_target_kl(None) == 0.0
    assert check_target_kl(0) == 0.0
    assert check_target_kl(0.01) == 0.01
    assert check_target_kl(np.float32(2.5)) == 2.5
    for bad in BAD:
        with pytest.raises(ValueError):
            check_target_kl(bad)


@pytest.mark.parametrize("bad", BAD)
def test_engine_and_updater_reject_a_bad_target_before_any_cuda_call(bad, monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    with pytest.raises(ValueError):
        Engine("cuda:0", 16, 16, target_kl=bad)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", target_kl=bad)


def test_c_entry_point_validates_without_a_context():
    import ctypes as C
    L = _lib.lib()
    assert L.upb_set_target_kl(None, C.c_float(0.1)) == -1 and b"set_target_kl" in L.upb_last_error()
    assert L.upb_reset_kl_stop(None, None) == -1 and b"reset_kl_stop" in L.upb_last_error()
    assert L.upb_mlp_reset_kl_stop(None, None) == -1 and b"mlp_reset_kl_stop" in L.upb_last_error()


def rows(nb, seed, stop=None, skipped_from=None):
    """Statistics rows (nb, 16) with known sums; `stop` marks slot 13 of that row, rows from `skipped_from` on are
    skipped rows (zeros but slot 14)."""
    rng = np.random.default_rng(seed)
    st = np.zeros((nb, 16))
    st[:, 0] = rng.random(nb) * 4
    st[:, 1] = rng.normal(size=nb)
    st[:, 2] = -rng.random(nb) * 30
    st[:, 3] = 32
    st[:, 4] = 28
    st[:, 8] = rng.random(nb)
    if stop is not None:
        st[stop, KL_STOP_SLOT] = 1
    if skipped_from is not None:
        st[skipped_from:] = 0
        st[skipped_from:, KL_SKIP_SLOT] = 1
    return st


def losses(st):
    vl, sl, el = st[:, 0] / st[:, 3], st[:, 1] / st[:, 4], st[:, 2] / st[:, 4]
    return np.stack([sl + VC * vl + EC * el, vl, sl, el], 1)


def run(epochs, kl_stop, opt_num_epochs=4, iteration=2, loss_iter=10, diag=False):
    logged = []
    book = UpdateLog(opt_num_epochs, VC, EC, iteration, loss_iter, lambda t, v, s: logged.append((t, v, s)),
                     kl_stop=kl_stop)
    ran = 0
    for e, st in enumerate(epochs):
        d = {n: st[:, 8] / np.maximum(st[:, 4], 1) + k for k, n in enumerate(NAMES)} if diag else None
        ran += 1
        if book.epoch(e, st, d):
            break
    return book, book.finish(diag), logged, ran


def test_no_stop_logs_every_row_of_every_epoch():
    eps = [rows(5, s) for s in range(4)]
    for on in (False, True):
        book, out, logged, ran = run(eps, on)
        assert ran == 4
        steps = [s for t, _, s in logged if t == "loss/loss"]
        assert steps == list(range(10, 30))
        assert book.loss_iter == 30
        want = np.mean([losses(st).sum(0) for st in eps], 0)
        assert np.allclose([out["total_loss"], out["total_value_loss"], out["total_surr_loss"],
                            out["total_entropy_loss"]], want, rtol=1e-14)
        assert [s for t, _, s in logged if t == "loss/epoch_loss"] == [8, 9, 10, 11]
        if on:
            assert out["steps_applied"] == 20 and out["kl_stop"] is None
            assert ("diag/steps_applied", 20.0, 2) in logged
        else:
            assert "steps_applied" not in out and "kl_stop" not in out
            assert not any(t == "diag/steps_applied" for t, _, _ in logged)


@pytest.mark.parametrize("epoch,mb", [(0, 0), (0, 3), (1, 0), (2, 4)])
def test_a_stop_ends_the_update_after_its_epoch(epoch, mb):
    nb = 5
    eps = [rows(nb, s) for s in range(epoch)]
    eps.append(rows(nb, 99, stop=mb, skipped_from=mb + 1 if mb + 1 < nb else None))
    eps += [rows(nb, 50 + s) for s in range(4 - len(eps))]           # never read: the update has ended
    book, out, logged, ran = run(eps, True, diag=True)
    assert ran == epoch + 1
    n_logged = epoch * nb + mb + 1
    assert [s for t, _, s in logged if t == "loss/loss"] == list(range(10, 10 + n_logged))
    for name in NAMES:
        assert len([1 for t, _, _ in logged if t == "diag/" + name]) == n_logged
    assert book.loss_iter == 10 + n_logged
    assert out["kl_stop"] == (epoch, mb)
    assert out["steps_applied"] == n_logged - 1
    assert ("diag/steps_applied", float(n_logged - 1), 2) in logged
    assert [s for t, _, s in logged if t == "loss/epoch_loss"] == [8 + e for e in range(epoch + 1)]
    last = eps[epoch][:mb + 1]
    assert [v for t, v, s in logged if t == "loss/epoch_loss"][-1] == pytest.approx(losses(last)[:, 0].sum(),
                                                                                      rel=1e-14)
    per_epoch = [losses(st).sum(0) for st in eps[:epoch]] + [losses(last).sum(0)]
    assert out["total_loss"] == pytest.approx(np.sum(per_epoch, 0)[0] / (epoch + 1), rel=1e-14)
    # diagnostics means exclude the skipped rows
    kept = np.concatenate([st[:, 8] / st[:, 4] for st in eps[:epoch]] + [last[:, 8] / last[:, 4]])
    assert out["total_approx_kl"] == pytest.approx(kept.mean(), rel=1e-14)


def test_skipped_rows_alone_end_the_update_and_log_nothing():
    eps = [rows(4, 0), rows(4, 1, skipped_from=0), rows(4, 2)]
    book, out, logged, ran = run(eps, True)
    assert ran == 2 and out["kl_stop"] is None and out["steps_applied"] == 4
    assert [s for t, _, s in logged if t == "loss/loss"] == [10, 11, 12, 13]
    # an epoch with no logged row still counts as an epoch that ran
    assert [v for t, v, s in logged if t == "loss/epoch_loss"][1] == 0.0
    assert out["total_loss"] == pytest.approx(losses(eps[0])[:, 0].sum() / 2, rel=1e-14)


def test_markers_are_ignored_while_the_stop_is_off():
    eps = [rows(3, s, stop=1) for s in range(3)]
    _, out, logged, ran = run(eps, False, opt_num_epochs=3)
    assert ran == 3 and len([1 for t, _, _ in logged if t == "loss/loss"]) == 9


def test_device_criterion_in_numpy_float32():
    """The criterion the kernels evaluate, replayed in numpy float32: S8 > fp32(1.5 * target) * max(S4, 1)."""
    def stops(s8, s4, target):
        limit = np.float32(1.5 * float(target))
        return bool(np.float32(s8) > np.float32(limit * np.maximum(np.float32(s4), np.float32(1))))
    assert not stops(0.0, 0.0, 1e-3)                 # no exps != 0 graph
    assert not stops(float("nan"), 10.0, 1e-3)
    assert stops(1.0, 10.0, 0.06) and not stops(1.0, 10.0, 0.07)
