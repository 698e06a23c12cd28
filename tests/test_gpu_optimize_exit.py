"""FullSystem::optimize's convergence exit and iteration budget on the device (ldso_b200_gn_iterations_until and the fused host
forms): the device-side decision inside the CUDA graph gives the same bits as the host applying LDSO's rule after every body, the same
canbreak sequence and stopping body as LDSO (the oracle), and the same bits in its host-driven form."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ldso_b200 import capi, synth
from tests import oracle_py
from tests.test_optimize_exit_cpu import EXIT_TABLE, MAX_OPT_ITERATIONS, MIN_OPT_ITERATIONS, bodies_run

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDS = ["cfg2", "smoke", "nF3", "nF2"]


def _ctx(win):
    ctx = capi.Context(win.w, win.h, win.levels)
    ctx.load_synth_window(win)
    return ctx


def _state(ctx):
    """Everything the loop leaves behind that a caller can read: the last solve, energy and canbreak, frame states, points, residuals."""
    out = dict(ctx.last_solution())
    e, cb = ctx.energy()
    out["energy"], out["canbreak"] = np.array(e), np.array(cb)
    fr = ctx.frames()
    for k in ("state", "step", "frameEnergyTH", "calib_value", "adHTdeltaF"):
        out["frames." + k] = fr[k]
    for k, v in ctx.points().items():
        out["points." + k] = v
    for k, v in ctx.residuals(with_J=False).items():
        out["res." + k] = v
    return out


def _assert_same(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{what}: {k} differs"


def _host_rule(ctx, budget, min_its=MIN_OPT_ITERATIONS, first=0):
    """LDSO's loop driven from the host: one body, read canbreak, break by FullSystem.cc:829."""
    cbs, energies = [], []
    for k in range(budget):
        ctx.gn_iterations(first + k, 1)
        e, cb = ctx.energy()
        cbs.append(cb)
        energies.append(e)
        if cb and first + k >= min_its:
            break
    return cbs, energies


def _until_run(win, budget, min_its=MIN_OPT_ITERATIONS):
    ctx = _ctx(win)
    ctx.optimize_begin()
    ctx.gn_iterations_until(0, budget, min_its)
    n = ctx.iterations_run()
    form = ctx.until_form()
    st = _state(ctx)
    ctx.close()
    return n, form, st


@pytest.fixture(scope="module")
def runs():
    """Per window: the device-side exit (A) and the host-driven rule on a second context (B)."""
    out = {}
    for idx, (kw, _, _) in enumerate(EXIT_TABLE):
        win = synth.make_window(**kw)
        budget = capi.optimize_iteration_budget(win.nF, MAX_OPT_ITERATIONS)
        n, form, st = _until_run(win, budget)
        b = _ctx(win)
        b.optimize_begin()
        cbs, energies = _host_rule(b, budget)
        out[idx] = dict(win=win, budget=budget, n=n, form=form, state=st, cbs=cbs, energies=energies, host_state=_state(b))
        b.close()
    return out


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=IDS)
def test_until_matches_host_rule(idx, runs):
    r = runs[idx]
    assert r["form"] in ("graph+pdl", "graph"), r["form"]       # the decision ran inside the graph
    assert r["n"] == len(r["cbs"])
    _assert_same(r["state"], r["host_state"], "until vs host rule")
    # ... and it is exactly the fixed-count loop of that many bodies
    c = _ctx(r["win"])
    c.optimize_begin()
    c.gn_iterations(0, r["n"])
    _assert_same(r["state"], _state(c), "until vs gn_iterations(0, n)")
    c.close()


def _canbreak_ratios(o):
    """doStepFromBackup's four quantities over their thresholds (FullSystem.cc:1617-1621) after the oracle's last body:
    canbreak fires when all four are below 1."""
    f, p = o.frames(), o.points()
    st = f["step"][:, :8]
    th = 1.2                                      # setting_thOptIterations
    nid = np.mean(np.abs(p["idepth"].astype(np.float64) - p["step"]))
    return np.array([np.sqrt(np.mean(st[:, 6] ** 2)) / (5e-4 * th), np.sqrt(np.mean(st[:, 7] ** 2)) / (5e-5 * th),
                     np.sqrt(np.mean(np.sum(st[:, 3:6] ** 2, 1))) / (5e-5 * th),
                     np.sqrt(np.mean(np.sum(st[:, 0:3] ** 2, 1))) * nid / (5e-5 * th)])


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=IDS)
def test_until_matches_ldso(idx, runs):
    """The device's per-iteration canbreak and its stopping body are LDSO's (the oracle's); energies agree to the 2e-3 bar."""
    kw, seq, stop = EXIT_TABLE[idx]
    r = runs[idx]
    o = oracle_py.OracleBA(r["win"], threads_mode=0)
    o.optimize_begin()
    for k in range(len(r["cbs"])):
        cb_o = o.gn_iteration(k)
        assert cb_o == (seq[k] == "1")
        assert r["cbs"][k] == cb_o, f"iteration {k}: device canbreak {r['cbs'][k]}, oracle {cb_o} (oracle ratios {_canbreak_ratios(o)})"
        assert abs(r["energies"][k] - o.energy()) <= 2e-3 * abs(o.energy()), (k, r["energies"][k], o.energy())
    assert r["n"] == stop == bodies_run([c == "1" for c in seq], r["budget"])


def test_min_iterations():
    """On a converged window (canbreak fires at every iteration from 8 on) the minimum decides: a body below it never ends the loop."""
    win = synth.make_window(**EXIT_TABLE[1][0])
    got = {}
    for min_its in (13, 12, 0):
        c = _ctx(win)
        c.optimize_begin()
        c.gn_iterations(0, 12)
        assert c.energy()[1]
        c.gn_iterations_until(12, 6, min_its)
        got[min_its] = c.iterations_run()
        c.close()
    assert got == {13: 2, 12: 1, 0: 1}


def test_max_iterations():
    win = synth.make_window(**EXIT_TABLE[3][0])      # the exit fires at body 10
    c = _ctx(win)
    c.optimize_begin()
    c.gn_iterations(0, 2)
    before = _state(c)
    launches = c.launch_count()
    c.gn_iterations_until(2, 0, 1)                    # max = 0: nothing runs, nothing changes
    assert c.iterations_run() == 0 and c.launch_count() == launches
    _assert_same(before, _state(c), "max = 0")
    c.close()
    a = _ctx(win)
    a.optimize_begin()
    a.gn_iterations_until(0, 4, 1)                    # a maximum below the exit point runs exactly that many bodies
    assert a.iterations_run() == 4
    b = _ctx(win)
    b.optimize_begin()
    b.gn_iterations(0, 4)
    _assert_same(_state(a), _state(b), "max = 4")
    a.close(); b.close()


@pytest.mark.parametrize("idx", range(len(EXIT_TABLE)), ids=IDS)
def test_host_driven_form_same_bits(idx, runs, monkeypatch):
    """Without CUDA graphs (read at context creation) and while kernel_times collects, the exit runs host-driven: same bits."""
    r = runs[idx]
    monkeypatch.setenv("LDSO_B200_NO_GRAPH", "1")
    n, form, st = _until_run(r["win"], r["budget"])
    assert form == "host" and n == r["n"]
    _assert_same(r["state"], st, "host-driven vs graph")
    monkeypatch.delenv("LDSO_B200_NO_GRAPH")
    c = _ctx(r["win"])
    c.optimize_begin()
    c.kernel_times(True)
    c.gn_iterations_until(0, r["budget"], MIN_OPT_ITERATIONS)
    c.kernel_times(False)
    assert c.until_form() == "host" and c.iterations_run() == r["n"]
    _assert_same(r["state"], _state(c), "kernel_times vs graph")
    c.close()


def test_fused_host_until():
    """optimize_from_host_until == the individual calls, bit for bit; so is the split form with a second context in flight."""
    win = synth.make_window(**EXIT_TABLE[2][0])       # the exit fires at body 6 of 15
    budget = capi.optimize_iteration_budget(win.nF, MAX_OPT_ITERATIONS)
    ref = _ctx(win)
    ref.optimize_begin(want_energy=False)
    ref.gn_iterations_until(0, budget, MIN_OPT_ITERATIONS)
    n_ref = ref.iterations_run()
    sol, pts, res = ref.last_solution(), ref.points(), ref.residuals(with_J=False)
    e_ref, cb_ref = ref.energy()
    ref.close()
    expect = dict(lastHS=sol["lastHS"], lastbS=sol["lastbS"], lastX=sol["lastX"], idepth=pts["idepth"], step=pts["step"], HdiF=pts["HdiF"],
                  state_state=res["state_state"], state_NewState=res["state_NewState"], state_energy=res["state_energy"])
    assert n_ref == 6

    ctx = _ctx(win)
    io = capi.StepIO(ctx, win)
    out = io.fused_until(0, budget, MIN_OPT_ITERATIONS)
    assert io.iterations_run == n_ref and io.scalars() == (e_ref, cb_ref)
    for k in expect:
        assert np.array_equal(out[k], expect[k]), k
    other = _ctx(win)
    io2 = capi.StepIO(other, win)
    io.submit_until(0, budget, MIN_OPT_ITERATIONS)
    io2.submit_until(0, budget, MIN_OPT_ITERATIONS)
    split = {k: v.copy() for k, v in io.wait_until().items()}
    assert io.iterations_run == n_ref and io.scalars() == (e_ref, cb_ref)
    split2 = io2.wait_until()
    assert io2.iterations_run == n_ref
    for k in expect:
        assert np.array_equal(split[k], expect[k]) and np.array_equal(split2[k], expect[k]), k
    other.close(); ctx.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_until_peer_exchange_two_gpus():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29523", os.path.join(ROOT, "tools", "until_multi_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "UNTIL_MULTI_CHECK OK" in r.stdout
