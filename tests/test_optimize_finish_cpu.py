"""The end of FullSystem::optimize (FullSystem.cc:833-863) on the CPU: the epilogue composed from the oracle's pieces
(tests/finish_oracle.py) on the windows of tests/test_optimize_exit_cpu.py, and the cases the device tests rely on. No GPU needed."""
import numpy as np
import pytest

from ldso_b200 import synth
from tests import finish_oracle as fo
from tests.test_optimize_exit_cpu import EXIT_TABLE, MAX_OPT_ITERATIONS, budget_rule


@pytest.fixture(scope="module")
def finished():
    out = {}
    for idx, (kw, _, stop) in enumerate(EXIT_TABLE):
        win = synth.make_window(**kw)
        o, n = fo.run_loop(win, budget_rule(win.nF, MAX_OPT_ITERATIONS))
        loop = dict(f=o.frames(), pts=o.points(), res=o.residuals(), post_step_active=int((o.residuals()["isActive"] != 0).sum()))
        out[idx] = (win, n, stop, loop, fo.optimize_finish(o, win))
    return out


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=["cfg2", "smoke", "nF3", "nF2"])
def test_finish_on_exit_windows(idx, finished):
    """The oracle's epilogue after its own loop: setEvalPT's state rule, every residual active or dropped, the counts consistent."""
    win, n, stop, loop, r = finished[idx]
    assert n == stop
    nF = win.nF
    f = r["frames"]
    assert np.array_equal(f["state"][nF - 1], r["newest_state_zero"])
    assert np.all(r["newest_state_zero"][[0, 1, 2, 3, 4, 5, 8, 9]] == 0)
    assert np.array_equal(r["newest_state_zero"][6:8], loop["f"]["state"][nF - 1][6:8])
    assert np.allclose(r["newest_evalR"] @ r["newest_evalR"].T, np.eye(3), atol=1e-12)
    # the pose of the newest frame does not move, so the current-pose pair records stay; the eval-point ones move
    assert np.allclose(f["precalc"][:, 24:36], loop["f"]["precalc"][:, 24:36], rtol=1e-5, atol=1e-6)
    assert np.array_equal(r["res_dropped"], r["res_state"] != fo.RES_IN)
    assert r["res_dropped"].sum() > 0
    assert int(r["pt_n_good"].sum()) == int((~r["res_dropped"]).sum())
    assert np.all(r["pt_relBS_max"][r["pt_n_good"] == 0] == 0) and np.all(r["pt_relBS_max"][r["pt_n_good"] > 0] > 0)
    assert np.isfinite(r["energy"]) and not r["is_lost"]


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=["cfg2", "smoke", "nF3", "nF2"])
def test_finish_from_loop_state(idx, finished):
    """The path the device tests take -- the window rebuilt from a loop's results, then finished by the oracle -- gives what the
    oracle's epilogue after its own loop gives."""
    win, _, _, loop, r = finished[idx]
    g = fo.finish_from(win, loop["f"], loop["pts"], loop["res"], r["resInA"])
    for k in ("newest_evalR", "newest_evalT", "newest_state_zero", "res_state", "res_dropped", "pt_n_good"):
        assert np.array_equal(g[k], r[k]), k
    for k in ("adHost", "adTarget"):
        assert np.array_equal(g["frames"][k], r["frames"][k]), k
    # the calibration is rebuilt as value_zero + (value - value_zero): at most an ulp away, which the float records may show
    assert np.allclose(g["frames"]["precalc"], r["frames"]["precalc"], rtol=1e-6, atol=1e-6)
    assert np.allclose(g["pt_relBS_max"], r["pt_relBS_max"], rtol=1e-6, atol=0)
    assert g["energy"] == pytest.approx(r["energy"], rel=1e-9)


def test_single_frame_returns_zero():
    win = synth.make_window(nF=2, pts_per_frame=16, seed=3)
    win.nF = 1
    r = fo.optimize_finish(None, win)       # nothing runs: no oracle needed
    assert r == dict(rmse=0.0, energy=0.0, is_lost=False)


def test_non_finite_energy_is_lost():
    """One non-finite colour sample of one point makes the fixed linearisation's energy NaN: the frame is reported lost."""
    win = synth.make_window(nF=2, pts_per_frame=64, seed=3)
    win.pt_color = np.array(win.pt_color, np.float32)
    win.pt_color[0, 4] = np.inf
    o, _ = fo.run_loop(win, 0)
    r = fo.optimize_finish(o, win)
    assert r["is_lost"] and not np.isfinite(r["energy"])


def test_rmse_uses_resInA_of_the_last_solve():
    """After one body, the count of active residuals the step left behind differs from the count its solve used; the RMSE divides
    by the latter, as FullSystem::optimize's `ef->resInA` does."""
    win = synth.make_window(**EXIT_TABLE[0][0])
    o, n = fo.run_loop(win, 1)
    post_step = int((o.residuals()["isActive"] != 0).sum())
    solved = o.res_counts()[0]      # EnergyFunctional::resInA, written by the body's solveSystemF
    r = fo.optimize_finish(o, win)
    assert n == 1 and solved != post_step and r["resInA"] == solved
    assert r["rmse"] == float(np.sqrt(np.float32(r["energy"] / (8 * solved))))
