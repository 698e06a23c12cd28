"""The end of FullSystem::optimize (FullSystem.cc:833-863) on the CPU, run by the oracle's own code.

TEST INFRASTRUCTURE ONLY. tests/cpp/finish_probe.cc drives the oracle's Window through the epilogue (setEvalPT of the newest frame,
setAdjointsF, setPrecalcValues, linearizeAll(true) with its relBS / maxRelBaseline and dropResidual); it is compiled together with the
oracle's unmodified sources into a temporary shared object, which also serves every OracleBA this module creates. The epilogue can
start from the oracle's own loop (optimize_finish) or from the state another implementation's loop left (finish_from).
"""
from __future__ import annotations

import copy
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import oracle_py

RES_IN, RES_OOB, RES_OUTLIER = 0, 1, 2
PATTERN_NUM = 8
PROBE_SRC = os.path.join(oracle_py.ROOT, "tests", "cpp", "finish_probe.cc")
ORACLE_SRC = [os.path.join(oracle_py.ORACLE_DIR, f) for f in ("ba.cc", "tracker.cc", "trace.cc", "initializer.cc", "capi.cc")]
_probe = None


def probe_lib():
    """liboracle.so's sources and flags (oracle/Makefile) plus the probe, built once per source state into the temp directory."""
    global _probe
    if _probe is None:
        srcs = ORACLE_SRC + [PROBE_SRC] + [os.path.join(oracle_py.ORACLE_DIR, f) for f in os.listdir(oracle_py.ORACLE_DIR) if f.endswith(".h")]
        key = hashlib.sha1(b"".join(open(f, "rb").read() for f in sorted(srcs))).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"ldso_b200_finish_probe_{os.getuid()}_{key}.so")
        if not os.path.exists(out):
            tmp = out + f".{os.getpid()}"
            subprocess.check_call(["g++", "-std=c++17", "-O3", "-march=native", "-fPIC", "-shared", "-pthread", "-ffp-contract=off",
                                   *ORACLE_SRC, PROBE_SRC, "-o", tmp])
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.oracle_ba_create.restype = C.c_void_p
        L.oracle_ba_create.argtypes = [C.c_int, C.c_int, C.c_int]
        L.oracle_ba_destroy.argtypes = [C.c_void_p]
        for f in ("oracle_ba_optimize_begin", "oracle_ba_linearize_all", "oracle_ba_last_energy", "oracle_ba_calc_m_energy",
                  "oracle_ba_calc_l_energy", "oracle_ba_time_gn", "finish_probe_run"):
            getattr(L, f).restype = C.c_double
        _probe = L
    return _probe


class ProbeBA(oracle_py.OracleBA):
    """An OracleBA whose window lives in the probe's copy of the oracle (same sources, same flags as liboracle.so)."""

    def __init__(self, win, calib_delta=None):
        saved = oracle_py._libs.get("ieee")
        oracle_py._libs["ieee"] = probe_lib()
        try:
            super().__init__(win, threads_mode=0, calib_delta=calib_delta)
        finally:
            if saved is None:
                del oracle_py._libs["ieee"]
            else:
                oracle_py._libs["ieee"] = saved

    def finish(self):
        """FullSystem.cc:833-863 on this window (tests/cpp/finish_probe.cc)."""
        nP, nR = self.win.nP, self.win.nR
        o = dict(newest_evalR=np.zeros((3, 3)), newest_evalT=np.zeros(3), newest_state_zero=np.zeros(10),
                 pt_relBS_max=np.zeros(nP, np.float32), pt_n_good=np.zeros(nP, np.int32), res_state=np.zeros(nR, np.int32),
                 res_dropped=np.zeros(nR, np.uint8))
        resInA = C.c_int()
        d, f, i = oracle_py._d, oracle_py._f, (lambda a: a.ctypes.data_as(oracle_py.c_ip))
        o["energy"] = self.L.finish_probe_run(self.o, d(o["newest_evalR"]), d(o["newest_evalT"]), d(o["newest_state_zero"]),
                                              f(o["pt_relBS_max"]), i(o["pt_n_good"]), i(o["res_state"]),
                                              o["res_dropped"].ctypes.data_as(oracle_py.c_bp), C.byref(resInA))
        o["resInA"] = resInA.value
        o["res_dropped"] = o["res_dropped"] != 0
        o["frames"] = self.frames()
        return o


def run_loop(win, budget, min_its=1):
    """FullSystem::optimize's prologue and loop with its exit (FullSystem.cc:734-831) on the oracle: (oracle, bodies run)."""
    o = ProbeBA(win)
    o.optimize_begin()
    n = 0
    for k in range(budget):
        cb = o.gn_iteration(k)
        n += 1
        if cb and k >= min_its:
            break
    return o, n


def _returned(o, resInA):
    """:845-849 isLost, :863 the returned RMSE (resInA: EnergyFunctional::resInA, set by the accumulateAF_MT of the last solve)."""
    with np.errstate(divide="ignore", invalid="ignore"):     # resInA = 0 when no solve ran
        o["rmse"] = float(np.sqrt(np.float32(np.float64(o["energy"]) / np.float64(PATTERN_NUM * resInA))))
    o["is_lost"] = not np.isfinite(o["energy"])
    return o


def optimize_finish(o, win):
    """FullSystem.cc:833-863 after the ProbeBA `o` ran the loop on `win` (run_loop)."""
    if win.nF < 2:       # FullSystem.cc:727-728: optimize returns 0 before anything runs
        return dict(rmse=0.0, energy=0.0, is_lost=False)
    r = o.finish()
    return _returned(r, r["resInA"])


def finish_from(win, f, pts, res, resInA):
    """The epilogue from the state another loop left behind: frames (state, calib_value, frameEnergyTH), points (idepth, idepth_zero),
    residuals (state_state, state_energy) and the resInA of that loop's last solve. The window is rebuilt in the oracle at its
    original evaluation points with those states (so PRE_worldToCam is the loop's pose), then finished by the oracle."""
    w2 = copy.copy(win)
    w2.state = np.array(f["state"], np.float64)
    w2.pt_idepth = np.array(pts["idepth"], np.float32); w2.pt_idepth_zero = np.array(pts["idepth_zero"], np.float32)
    value_zero = ProbeBA(win).frames()["calib_value"]
    o2 = ProbeBA(w2, calib_delta=np.asarray(f["calib_value"]) - value_zero)
    for i in range(win.nF):          # the loop's energy thresholds, as its last setNewFrameEnergyTH left them
        o2.L.oracle_ba_set_frame_energy_th(o2.o, i, C.c_float(float(f["frameEnergyTH"][i])))
    st = np.ascontiguousarray(res["state_state"], np.int32)
    en = np.ascontiguousarray(res["state_energy"], np.float64)
    o2.L.finish_probe_set_residuals(o2.o, st.ctypes.data_as(oracle_py.c_ip), oracle_py._d(en))
    r = o2.finish()
    r["oracle"] = o2
    return _returned(r, resInA)
