"""FullSystem::optimize's iteration budget and convergence exit (FullSystem.cc:727-732, :829) on the CPU: the budget rule of the C ABI,
and the canbreak sequences the oracle and the reference's own back end produce on the windows tests/test_gpu_optimize_exit.py runs
on the device. No GPU needed."""
import numpy as np
import pytest

from ldso_b200 import build as lbuild
from ldso_b200 import capi, synth
from tests import oracle_py

# (window, canbreak of iterations 0..19 -- 1 = doStepFromBackup returned true -- and the body after which LDSO's loop stops)
EXIT_TABLE = [
    (dict(nF=8, pts_per_frame=250, seed=42), "00000010111111111111", 6),                   # BASELINE configs[1]: the budget ends it
    (dict(nF=4, pts_per_frame=64, w=320, h=240, seed=11), "00000000111111111111", 6),      # the smoke() window: the budget ends it
    (dict(nF=3, pts_per_frame=250, seed=4), "00000100010101111111", 6),                    # young window: the exit ends it at 6 of 15
    (dict(nF=2, pts_per_frame=250, seed=3), "00000000010001000000", 10),                   # young window: the exit ends it at 10 of 15
]
MAX_OPT_ITERATIONS, MIN_OPT_ITERATIONS = 6, 1       # setting_maxOptIterations, setting_minOptIterations (Setting.cc:36-37)


def budget_rule(nF, max_its):
    """FullSystem.cc:727-732 as written: the `< 3 -> 20` assignment is overwritten by the `< 4 -> 15` one."""
    if nF < 2:
        return 0
    its = max_its
    if nF < 3:
        its = 20
    if nF < 4:
        its = 15
    return its


def bodies_run(canbreak, budget, min_its=MIN_OPT_ITERATIONS, first=0):
    """The loop's stopping rule: the first body whose canbreak fires once iteration >= min_its, within the budget."""
    for k in range(budget):
        if canbreak[k] and first + k >= min_its:
            return k + 1
    return budget


@pytest.fixture(scope="module")
def lib():
    lbuild.build()
    return capi.load()


def test_iteration_budget(lib):
    assert [capi.optimize_iteration_budget(nF, 6) for nF in range(9)] == [0, 0, 15, 15, 6, 6, 6, 6, 6]
    for max_its in (0, 1, 3, 10, 25):
        assert [capi.optimize_iteration_budget(nF, max_its) for nF in range(9)] == [budget_rule(nF, max_its) for nF in range(9)]
    assert lib.ldso_b200_optimize_iteration_budget(5, -1) == -1          # LDSO_B200_ERR_ARG
    with pytest.raises(capi.Error):
        capi.optimize_iteration_budget(5, -1)


def test_stopping_rule():
    assert bodies_run([0, 1, 1], 6) == 2            # iteration 0 is below the minimum: its canbreak does not count
    assert bodies_run([1, 1], 6, min_its=0) == 1
    assert bodies_run([1, 1], 6, min_its=1) == 2
    assert bodies_run([0] * 6, 6) == 6
    assert bodies_run([1] * 6, 0) == 0


def _sequence(model, n=20):
    model.optimize_begin()
    return "".join("1" if model.gn_iteration(i) else "0" for i in range(n))


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)))
def test_exit_table_oracle(idx):
    kw, seq, stop = EXIT_TABLE[idx]
    win = synth.make_window(**kw)
    got = _sequence(oracle_py.OracleBA(win, threads_mode=0))
    assert got == seq
    cb = [c == "1" for c in got]
    assert bodies_run(cb, budget_rule(win.nF, MAX_OPT_ITERATIONS)) == stop


@pytest.mark.skipif(oracle_py.ref_lib() is None, reason="oracle/_ref/libref_ba.so is built only where the reference tree is mounted (make -C oracle ref_pin)")
@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)))
def test_exit_table_reference(idx):
    """The reference's own back-end translation units (oracle/_ref/libref_ba.so) give the same sequences as the oracle."""
    kw, seq, stop = EXIT_TABLE[idx]
    win = synth.make_window(**kw)
    got = _sequence(oracle_py.RefBA(win, multithreaded=False))
    assert got == seq
    assert bodies_run([c == "1" for c in got], budget_rule(win.nF, MAX_OPT_ITERATIONS)) == stop
