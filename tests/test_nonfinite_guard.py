"""The non-finite guard (`skip_nonfinite`, upb_set_nonfinite_guard) without a GPU: the argument checks, the exported
symbol and the update log's bookkeeping of the rows the guard skipped (statistics slot 19)."""
import types

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib
from drl_urban_planning_b200.diagnostics import NAMES
from drl_urban_planning_b200.engine import Engine, check_skip_nonfinite
from drl_urban_planning_b200.ppo import (KL_SKIP_SLOT, KL_STOP_SLOT, KLPEN_SLOT, NONFINITE_COUNT_SLOT, NONFINITE_SLOT,
                                         UpdateLog, unguarded_nonfinite)
from harness import Cfg

BAD = [0.5, 2, -1, "yes", None, float("nan")]


def test_check_skip_nonfinite_values():
    assert check_skip_nonfinite(False) is False and check_skip_nonfinite(True) is True
    assert check_skip_nonfinite(0) is False and check_skip_nonfinite(np.bool_(True)) is True
    for bad in BAD:
        with pytest.raises(ValueError, match="skip_nonfinite"):
            check_skip_nonfinite(bad)


@pytest.mark.parametrize("bad", BAD)
def test_bad_skip_nonfinite_is_rejected_before_any_cuda_call(bad, monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("reached CUDA")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    with pytest.raises(ValueError, match="skip_nonfinite"):
        Engine("cuda:0", 16, 16, skip_nonfinite=bad)
    from drl_urban_planning_b200.ppo import PPOUpdater
    with pytest.raises(ValueError, match="skip_nonfinite"):
        PPOUpdater(np.zeros(_lib.UPB_NUM_PARAMS, np.float32), 16, 16, "cuda:0", skip_nonfinite=bad)
    from drl_urban_planning_b200.agent import B200Update
    for kind in ("rl-sgnn", "rl-mlp"):
        cfg = Cfg(64, 64)
        cfg.agent, cfg.clip_epsilon = kind, 0.2
        with pytest.raises(ValueError, match="skip_nonfinite"):
            B200Update(types.SimpleNamespace(cfg=cfg, device=torch.device("cuda", 0)), skip_nonfinite=bad)


def test_c_entry_point_is_exported_and_validates_without_a_context():
    assert "upb_set_nonfinite_guard" in _lib.EXPORTED_SYMBOLS
    L = _lib.lib()
    assert L.upb_set_nonfinite_guard(None, 1) == -1 and b"set_nonfinite_guard" in L.upb_last_error()


def rows(nb, seed):
    rng = np.random.default_rng(seed)
    st = np.zeros((nb, 20))
    st[:, 0:3] = rng.random((nb, 3))
    st[:, 3], st[:, 4] = 32, 28
    st[:, 8:13] = rng.random((nb, 5))
    st[:, KLPEN_SLOT] = rng.random(nb)
    return st


def skipped(st, i, cause):
    """Row i as a skipped step leaves it: slot 19 set and non-finite sums."""
    st[i, NONFINITE_SLOT] = 1.0
    if cause == "count":
        st[i, 0:3] = np.nan
        st[i, NONFINITE_COUNT_SLOT] = 32
    else:
        st[i, 1] = np.inf


def test_which_counted_rows_raise():
    """Off: any row that counts a non-finite result (a NaN count included).  On: only a counted row the guard did not
    skip, which covers the row that stopped on the KL criterion first (its logged losses are not finite)."""
    st = rows(4, 0)
    assert not unguarded_nonfinite(st, False) and not unguarded_nonfinite(st, True)
    skipped(st, 1, "inf")
    assert not unguarded_nonfinite(st, False) and not unguarded_nonfinite(st, True)
    skipped(st, 2, "count")
    assert unguarded_nonfinite(st, False) and not unguarded_nonfinite(st, True)
    for count in (3.0, np.nan):
        stop = rows(4, 1)
        stop[1, NONFINITE_COUNT_SLOT], stop[1, KL_STOP_SLOT], stop[1, 0] = count, 1.0, np.nan
        assert unguarded_nonfinite(stop, False) and unguarded_nonfinite(stop, True)
        plain = rows(4, 2)
        plain[3, NONFINITE_COUNT_SLOT] = count
        assert unguarded_nonfinite(plain, False) and unguarded_nonfinite(plain, True)


def run(eps, diag=False, **kw):
    logged = []
    book = UpdateLog(len(eps), 0.5, 0.01, 3, 100, lambda t, v, s: logged.append((t, v, s)), **kw)
    for e, st in enumerate(eps):
        if book.epoch(e, st, {n: st[:, 8].copy() for n in NAMES} if diag else None):
            break
    return book, logged


@pytest.mark.parametrize("diag", [False, True])
def test_skipped_rows_are_left_out_and_counted(diag):
    eps = [rows(4, 0), rows(4, 1)]
    skipped(eps[0], 1, "count")
    skipped(eps[1], 0, "inf")
    skipped(eps[1], 3, "inf")
    book, logged = run(eps, diag, skip_nonfinite=True, kl_coef=0.3)
    out = book.finish(diag)
    keep = [np.array([0, 2, 3]), np.array([1, 2])]
    ref_book, ref_logged = run([st[k] for st, k in zip(eps, keep)], diag, kl_coef=0.3)
    ref = ref_book.finish(diag)
    assert out.pop("nonfinite_skips") == 3 and ("diag/nonfinite_skips", 3.0, 3) in logged
    assert out == ref and all(np.isfinite(v) for v in out.values() if isinstance(v, float))
    assert [x for x in logged if x[0] != "diag/nonfinite_skips"] == ref_logged
    assert book.steps == 5 and book.loss_iter == 105 and book.epochs == 2
    # kl_rows: the last epoch's rows that ran
    assert book.kl_rows == (float(eps[1][keep[1], KLPEN_SLOT].sum()), 56.0)
    if diag:
        assert np.isclose(out["total_approx_kl"], ref["total_approx_kl"])


def test_off_ignores_slot_19_and_reports_nothing():
    eps = [rows(3, 0)]
    eps[0][1, NONFINITE_SLOT] = 1.0
    book, logged = run(eps)
    out = book.finish(False)
    assert "nonfinite_skips" not in out and book.steps == 3
    assert not [x for x in logged if x[0] == "diag/nonfinite_skips"]
    book, _ = run([rows(3, 0)[:, :19]])           # a context without the guard may hand over 19 columns
    assert book.steps == 3


def test_no_skip_is_the_plain_log():
    eps = [rows(3, 0), rows(3, 1)]
    book, logged = run(eps, skip_nonfinite=True)
    out = book.finish(False)
    ref_book, ref_logged = run(eps)
    assert out.pop("nonfinite_skips") == 0 and out == ref_book.finish(False)
    assert [x for x in logged if x[0] != "diag/nonfinite_skips"] == ref_logged


def test_every_step_skipped_raises():
    eps = [rows(2, 0), rows(2, 1)]
    for st in eps:
        skipped(st, 0, "count")
        skipped(st, 1, "inf")
    book, logged = run(eps, skip_nonfinite=True)
    assert book.nonfinite_skips == 4 and book.steps == 0
    assert not [x for x in logged if x[0].startswith("loss/") and not x[0].startswith("loss/epoch")]
    with pytest.raises(FloatingPointError, match="every optimiser step"):
        book.finish(False)


def test_mixed_with_the_kl_stop_rows():
    """Epoch 0: a skipped row among rows that ran.  Epoch 1: a skipped row, then the step that stopped (slot 13, logged,
    no Adam), then rows skipped after it (slot 14, zeros).  The update ends there."""
    eps = [rows(4, 0), rows(4, 1), rows(4, 2)]
    skipped(eps[0], 2, "inf")
    skipped(eps[1], 0, "count")
    eps[1][1, KL_STOP_SLOT] = 1.0
    eps[1][2:] = 0.0
    eps[1][2:, KL_SKIP_SLOT] = 1.0
    book, logged = run(eps, skip_nonfinite=True, kl_stop=True)
    out = book.finish(False)
    assert book.epochs == 2 and out["nonfinite_skips"] == 2
    assert out["kl_stop"] == (1, 1) and book.steps == 4 and out["steps_applied"] == 3
    # only a skipped row and the stopping step: nothing was applied
    only = [rows(2, 3)]
    skipped(only[0], 0, "inf")
    only[0][1, KL_STOP_SLOT] = 1.0
    book, _ = run(only, skip_nonfinite=True, kl_stop=True)
    with pytest.raises(FloatingPointError):
        book.finish(False)
