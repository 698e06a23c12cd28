"""The end of FullSystem::optimize on the device (ldso_b200_optimize_finish, get_finish, optimize_from_host_full): against the CPU
epilogue (tests/finish_oracle.py) started from the state the device loop left, bit-identical across its forms, and the state rule."""
import numpy as np
import pytest

from ldso_b200 import capi, synth
from tests import finish_oracle as fo
from tests.parity import rel_err
from tests.test_optimize_exit_cpu import EXIT_TABLE, MAX_OPT_ITERATIONS, MIN_OPT_ITERATIONS

pytestmark = pytest.mark.gpu
IDS = ["cfg2", "smoke", "nF3", "nF2"]
KEYS = ("energy", "rmse", "is_lost", "res_state", "res_dropped", "pt_relBS_max", "pt_n_good", "newest_evalR", "newest_evalT",
        "newest_state_zero")


def _ctx(win):
    ctx = capi.Context(win.w, win.h, win.levels)
    ctx.load_synth_window(win)
    return ctx


def _loop(win, budget):
    c = _ctx(win)
    c.optimize_begin()
    c.gn_iterations_until(0, budget, MIN_OPT_ITERATIONS)
    return c


def _finish(c):
    c.optimize_finish()
    out = c.finish_results()
    fr = c.frames()
    for k in ("state", "frameEnergyTH", "precalc", "adHost", "adTarget", "adHTdeltaF"):
        out["frames." + k] = fr[k]
    return out


def _same(a, b, what):
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k]), equal_nan=True), f"{what}: {k} differs"


def _resInA_solved(win, n):
    """resInA of the solve of body n: the active count the accumulate after body n - 1 (or the prologue) produced."""
    c = _ctx(win)
    c.optimize_begin()
    if n > 1:
        c.gn_iterations(0, n - 1)
    r = c.system()["resInA"]
    c.close()
    return r


@pytest.fixture(scope="module")
def runs():
    out = {}
    for idx, (kw, _, stop) in enumerate(EXIT_TABLE):
        win = synth.make_window(**kw)
        budget = capi.optimize_iteration_budget(win.nF, MAX_OPT_ITERATIONS)
        c = _loop(win, budget)
        n = c.iterations_run()
        loop = dict(f=c.frames(), pts=c.points(), res=c.residuals(with_J=False))
        dev = _finish(c)
        c.close()
        out[idx] = dict(win=win, budget=budget, n=n, stop=stop, loop=loop, dev=dev, resInA=_resInA_solved(win, n))
    return out


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=IDS)
def test_finish_matches_oracle(idx, runs):
    r = runs[idx]
    win, d = r["win"], r["dev"]
    assert r["n"] == r["stop"]
    L = r["loop"]
    o = fo.finish_from(win, L["f"], L["pts"], L["res"], r["resInA"])
    # new evaluation point and state of the newest frame (f64)
    assert np.allclose(d["newest_evalR"], o["newest_evalR"], rtol=0, atol=1e-12)
    assert np.allclose(d["newest_evalT"], o["newest_evalT"], rtol=1e-12, atol=1e-12)
    assert np.array_equal(d["newest_state_zero"], o["newest_state_zero"])
    assert np.array_equal(d["frames.state"][-1], o["newest_state_zero"])
    of = o["frames"]
    for k in ("adHost", "adTarget"):
        err = np.abs(d["frames." + k] - of[k]) / np.maximum(np.abs(of[k]), 1.0)
        assert err.max() <= 1e-12, (k, float(err.max()))
    # pair records: float products of K R K^-1 cancel terms of the size of fx, so each record's error is taken relative to its norm
    # (the measure and bar tests/test_gpu_ba.py applies to the same records after set_frames)
    pd, po = d["frames.precalc"].astype(np.float64), of["precalc"].astype(np.float64)
    err = np.linalg.norm(pd - po, axis=1) / np.linalg.norm(po, axis=1)
    assert err.max() <= 1e-5, ("precalc", int(np.argmax(err)), float(err.max()))
    # residual states: equal up to threshold ties (energy == frameEnergyTH to float rounding), which are counted
    ties = np.nonzero(d["res_state"] != o["res_state"])[0]
    assert len(ties) <= max(2, win.nR // 500), f"{len(ties)} residual states differ"
    assert np.array_equal(d["res_dropped"] != 0, d["res_state"] != fo.RES_IN)
    assert np.array_equal(d["res_dropped"] != 0, o["res_dropped"]) or len(ties) > 0
    ok = np.ones(win.nP, bool)
    ok[win.res_point[ties]] = False
    assert np.array_equal(d["pt_n_good"][ok], o["pt_n_good"][ok])
    assert np.all(np.abs(d["pt_relBS_max"][ok] - o["pt_relBS_max"][ok]) <= 1e-5 * np.abs(o["pt_relBS_max"][ok]))
    assert abs(d["energy"] - o["energy"]) <= 1e-5 * abs(o["energy"])
    assert abs(d["rmse"] - o["rmse"]) <= 1e-5 * o["rmse"]
    assert not d["is_lost"] and not o["is_lost"]
    print(f"{IDS[idx]}: bodies {r['n']}, dropped {int(d['res_dropped'].sum())}, threshold ties {len(ties)}, energy {d['energy']:.6g}, "
          f"rmse {d['rmse']:.6g}")


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=IDS)
def test_finish_same_bits_every_form(idx, runs, monkeypatch):
    """Twice on identical inputs, host-driven loop (no CUDA graphs), and with kernel_times collecting: the same bits."""
    r = runs[idx]
    c = _loop(r["win"], r["budget"])
    _same(r["dev"], _finish(c), "second run")
    c.close()
    monkeypatch.setenv("LDSO_B200_NO_GRAPH", "1")
    c = _loop(r["win"], r["budget"])
    assert c.until_form() == "host"
    _same(r["dev"], _finish(c), "host-driven")
    c.close()
    monkeypatch.delenv("LDSO_B200_NO_GRAPH")
    c = _ctx(r["win"])
    c.optimize_begin()
    c.kernel_times(True)
    c.gn_iterations_until(0, r["budget"], MIN_OPT_ITERATIONS)
    c.kernel_times(False)
    _same(r["dev"], _finish(c), "kernel_times")
    c.close()


def test_full_host_call(runs):
    """optimize_from_host_full == optimize_from_host_until + optimize_finish + get_finish, bit for bit; so is the split form with a
    second context in flight."""
    r = runs[2]
    win = r["win"]
    ref = _ctx(win)
    io = capi.StepIO(ref, win)
    loop_out = {k: v.copy() for k, v in io.fused_until(0, r["budget"], MIN_OPT_ITERATIONS).items()}
    ref.optimize_finish()
    fin = ref.finish_results()
    ref.close()
    _same({k: r["dev"][k] for k in KEYS}, {k: fin[k] for k in KEYS}, "from host buffers vs loaded window")
    a, b = _ctx(win), _ctx(win)
    ia, ib = capi.StepIO(a, win), capi.StepIO(b, win)
    out, f = ia.fused_full(0, r["budget"], MIN_OPT_ITERATIONS)
    assert ia.iterations_run == r["n"]
    _same(loop_out, out, "full: loop outputs")
    _same({k: fin[k] for k in KEYS}, {k: f[k] for k in KEYS}, "full: finish")
    ia.submit_full(0, r["budget"], MIN_OPT_ITERATIONS)
    ib.submit_full(0, r["budget"], MIN_OPT_ITERATIONS)
    out_a, f_a = ia.wait_full()
    out_a = {k: v.copy() for k, v in out_a.items()}
    f_a = {k: np.copy(f_a[k]) for k in KEYS}
    out_b, f_b = ib.wait_full()
    for o_, f_ in ((out_a, f_a), (out_b, f_b)):
        _same(loop_out, o_, "split: loop outputs")
        _same({k: fin[k] for k in KEYS}, {k: f_[k] for k in KEYS}, "split: finish")
    a.close(); b.close()


def test_state_rule_and_marginalize_after_set_window(runs):
    """After the finish the window and solve entry points refuse to run until set_window / set_frames. set_window with the reduced
    window followed by marginalize_points (flagPointsForRemoval's order) matches the oracle marginalising the same points of its own
    finished window (its linearizeAll(true) removed the dropped residuals), at the bar tests/test_gpu_ba.py uses for marginalize_points."""
    r = runs[1]
    win = r["win"]
    c = _loop(win, r["budget"])
    pts = c.points()
    d = _finish(c)
    for call in (lambda: c.linearize_all(True), lambda: c.optimize_begin(), lambda: c.gn_iterations(0, 1),
                 lambda: c.marginalize_points([0])):
        with pytest.raises(capi.Error):
            call()
    keep = d["res_dropped"] == 0
    rp = win.res_point
    res_begin = np.concatenate([[0], np.cumsum(np.bincount(rp[keep], minlength=win.nP))]).astype(np.int32)
    c.set_window(win.pt_host, win.pt_u, win.pt_v, pts["idepth"], pts["idepth_zero"], win.pt_has_prior, win.pt_color, win.pt_weights,
                 res_begin, np.asarray(win.res_target)[keep], res_state=d["res_state"][keep])
    with pytest.raises(capi.Error):
        c.gn_iterations(0, 1)                 # the solve also needs set_frames
    idx = np.arange(0, win.nP, 7, dtype=np.int32)
    c.marginalize_points(idx)
    HMg, bMg = c.marg_prior()
    c.close()
    L = r["loop"]
    o = fo.finish_from(win, L["f"], L["pts"], L["res"], r["resInA"])
    assert np.array_equal(o["res_dropped"], d["res_dropped"] != 0)
    o["oracle"].marginalize_points(idx)
    HMo, bMo = o["oracle"].marg_prior()
    eH, eb = rel_err(HMg, HMo), rel_err(bMg, bMo)
    print(f"marginalize after finish: HM rel err {eH:.3g}, bM rel err {eb:.3g}")
    assert np.any(HMo != 0) and eH < 1e-4 and eb < 1e-4, (eH, eb)


def test_rmse_divides_by_the_solved_count():
    """One body on cfg2: the active count the step leaves behind differs from the count its solve used; the device's RMSE divides by
    the latter (FullSystem.cc:863's ef->resInA), i.e. matches the oracle's epilogue given that count."""
    win = synth.make_window(**EXIT_TABLE[0][0])
    solved = _resInA_solved(win, 1)
    c = _loop(win, 1)
    post_step = c.system()["resInA"]
    loop = dict(f=c.frames(), pts=c.points(), res=c.residuals(with_J=False))
    d = _finish(c)
    c.close()
    assert solved != post_step
    o = fo.finish_from(win, loop["f"], loop["pts"], loop["res"], solved)
    assert abs(d["rmse"] - o["rmse"]) <= 1e-5 * o["rmse"]
    assert abs(d["rmse"] - float(np.sqrt(np.float32(d["energy"] / (8 * post_step))))) > 1e-5 * o["rmse"]


def test_non_finite_energy_is_lost():
    """One non-finite colour sample of one point makes the fixed linearisation's energy NaN: the device reports the frame lost."""
    win = synth.make_window(nF=2, pts_per_frame=64, seed=3)
    win.pt_color = np.array(win.pt_color, np.float32)
    win.pt_color[0, 4] = np.inf
    c = _ctx(win)
    c.optimize_begin()
    c.optimize_finish()
    r = c.finish_results()
    assert r["is_lost"] and not np.isfinite(r["energy"])
    c.close()
