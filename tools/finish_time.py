"""Time one keyframe's FullSystem::optimize from host buffers in three forms (DESIGN.md §4, "The end of optimize"):

  full   optimize_from_host_full: the loop with its exit, then the finish on the device (ldso_b200_optimize_finish + get_finish)
  host   optimize_from_host_until, then the host epilogue a caller needs without the finish: get_frames -> the newest evaluation
         point composed on the host -> set_frames -> linearize_all(1) -> get_residuals -> relBS per point on the host
  floor  optimize_from_host_until alone

on BASELINE config 2 (8 keyframes x 250 points) and on the nF = 3 window of tests/test_optimize_exit_cpu.py. Each call is timed by the
host clock around work that ends in a device synchronise (every form returns its results to host memory), with the L2 flushed before
it; the forms alternate and the medians are reported. Needs a GPU.

    python tools/finish_time.py [--runs 30]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ldso_b200 import capi, synth  # noqa: E402

WINDOWS = {"config2": dict(nF=8, pts_per_frame=250, seed=42), "nF3": dict(nF=3, pts_per_frame=250, seed=4)}


def se3_exp(a):
    """Sophus SE3::exp of [upsilon, omega] as rotation matrix + translation (the host side of today's epilogue)."""
    om, ups = a[3:6], a[0:3]
    th = np.linalg.norm(om)
    O = np.array([[0, -om[2], om[1]], [om[2], 0, -om[0]], [-om[1], om[0], 0]])
    if th < 1e-10:
        A, B, Cc = 1.0, 0.5, 1.0 / 6.0
    else:
        A, B, Cc = np.sin(th) / th, (1 - np.cos(th)) / th ** 2, (th - np.sin(th)) / th ** 3
    R = np.eye(3) + A * O + B * O @ O
    V = np.eye(3) + B * O + Cc * O @ O
    return R, V @ ups


def host_epilogue(ctx, win, Rcw, tcw):
    """What a caller does today after optimize_from_host_until to finish optimize() (FullSystem.cc:833-863)."""
    nF = win.nF
    fr = ctx.frames()
    st = fr["state"].copy()
    s = st[nF - 1]
    Re, te = se3_exp(np.concatenate([0.5 * s[0:3], s[3:6]]))
    R, t = Rcw.copy(), tcw.copy()
    R[nF - 1], t[nF - 1] = Re @ Rcw[nF - 1], Re @ tcw[nF - 1] + te
    sz = np.array(win.state_zero, np.float64).copy()
    nsz = np.zeros(10); nsz[6:8] = s[6:8]
    sz[nF - 1] = nsz; st[nF - 1] = nsz
    Kz = np.asarray(win.K, np.float64) * np.float64(np.float32(1.0) / np.float32(50.0))
    Ks = fr["calib_value"] * 50.0
    ctx.set_frames(R, t, sz, st, win.ab_exposure, win.frame_id, list(range(nF)), Ks, K_zero=Kz, frame_energy_th=fr["frameEnergyTH"])
    ctx.linearize_all(True)
    res = ctx.residuals_light()
    pc = ctx.frames()["precalc"]
    act = np.nonzero(res["isActive"])[0]
    p = win.res_point[act]
    q = win.pt_host[p] + nF * win.res_target[act]
    K, Kt = pc[q, 24:33].reshape(-1, 3, 3), pc[q, 33:36]
    uv1 = np.stack([win.pt_u[p], win.pt_v[p], np.ones(len(p), np.float32)], 1)
    inf = np.einsum("nij,nj->ni", K, uv1)
    ptp = inf + Kt * ctx.points()["idepth"][p][:, None]
    rel = 0.01 * np.hypot(inf[:, 0] / inf[:, 2] - ptp[:, 0] / ptp[:, 2], inf[:, 1] / inf[:, 2] - ptp[:, 1] / ptp[:, 2])
    mx = np.zeros(win.nP, np.float32)
    np.maximum.at(mx, p, rel.astype(np.float32))
    return mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("finish_time.py needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    out = {"card": card, "runs": args.runs, "unit": "ms per keyframe (median)"}
    for name, kw in WINDOWS.items():
        win = synth.make_window(**kw)
        budget = capi.optimize_iteration_budget(win.nF, 6)
        Rcw, tcw = np.array(win.Rcw, np.float64), np.array(win.tcw, np.float64)
        ctxs = {k: capi.Context(win.w, win.h, win.levels) for k in ("full", "host", "floor")}
        ios = {}
        for k, c in ctxs.items():
            c.load_synth_window(win)
            ios[k] = capi.StepIO(c, win)
        forms = {
            "full": lambda: ios["full"].fused_full(0, budget, 1),
            "host": lambda: (ios["host"].fused_until(0, budget, 1), host_epilogue(ctxs["host"], win, Rcw, tcw)),
            "floor": lambda: ios["floor"].fused_until(0, budget, 1),
        }
        times = {k: [] for k in forms}
        for k in forms:          # warm-up: module loads, graph capture
            forms[k]()
            forms[k]()
        order = list(forms)
        for i in range(args.runs):
            for k in order[i % 3:] + order[:i % 3]:
                flush.fill_(float(i))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                forms[k]()
                times[k].append(1e3 * (time.perf_counter() - t0))
        out[name] = {k: round(float(np.median(v)), 4) for k, v in times.items()}
        out[name]["bodies"] = ios["floor"].iterations_run
        for c in ctxs.values():
            c.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
