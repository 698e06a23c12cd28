"""What FullSystem::optimize's exit costs and saves on the device (ldso_b200_gn_iterations_until), timed with CUDA events on the
context's stream, the L2 flushed before every timed loop (as bench.py does), the two variants of each pair alternated:

  overhead   BASELINE configs[1] (8 KF x 2000 points), where the exit does not fire within the 6-iteration budget:
             gn_iterations(0, 6) against gn_iterations_until(0, 6, 1) -- the conditional WHILE node plus the continue kernel, per body
  young      the nF = 3 window (budget 15, LDSO's exit fires after body 6): 15 fixed bodies against gn_iterations_until(0, 15, 1)
  fallback   the host-driven form (a context created with LDSO_B200_NO_GRAPH=1): gn_iterations_until per body against the graph

Each timed loop starts from the same state (window reloaded, optimize() prologue run, outside the events). The outputs of the
variants that must agree (same number of bodies) are compared bit for bit. Prints the card, its power limit and one JSON line.

    python tools/exit_time.py [--reps 30]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ldso_b200 import capi, synth  # noqa: E402
import bench  # noqa: E402


def make_ctx(win, stream, no_graph=False):
    old = os.environ.pop("LDSO_B200_NO_GRAPH", None)
    if no_graph:
        os.environ["LDSO_B200_NO_GRAPH"] = "1"
    try:
        ctx = capi.Context(win.w, win.h, win.levels)
    finally:
        os.environ.pop("LDSO_B200_NO_GRAPH", None)
        if old is not None:
            os.environ["LDSO_B200_NO_GRAPH"] = old
    ctx.set_stream(stream.cuda_stream)
    ctx.load_synth_window(win)
    return ctx


def outputs(ctx):
    sol = ctx.last_solution()
    return np.concatenate([sol["lastX"], sol["lastbS"], ctx.points()["idepth"].astype(np.float64), [ctx.energy()[0]]])


def timed(ctx, win, stream, flush, run, reps):
    """ms per call of run(ctx) (events around the loop only) over reps calls, and the outputs of the last call"""
    ms = []
    for k in range(reps):
        ctx.load_synth_window(win, upload_images=False)
        ctx.optimize_begin(want_energy=False)
        flush.fill_(k & 0xff)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        run(ctx)
        b.record(stream)
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms)), outputs(ctx)


def pair(win, stream, flush, reps, variants):
    """variants: name -> (ctx, run). Alternated rep by rep; median / min ms and outputs per variant."""
    res = {name: [] for name in variants}
    outs = {}
    for r in range(reps):
        for name, (ctx, run) in variants.items():
            med, _, out = timed(ctx, win, stream, flush, run, 1)
            res[name].append(med)
            outs[name] = out
    return {name: (float(np.median(v)), float(np.min(v))) for name, v in res.items()}, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    stream = torch.cuda.Stream()          # a capturable stream (the legacy default stream cannot hold a CUDA graph)
    torch.cuda.set_stream(stream)
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2 (H100)
    card = bench.gpu_name(torch, 0)
    print("card:", card)
    result = {"card": card, "reps": args.reps}

    def fixed(n):
        return lambda c: c.gn_iterations(0, n)

    def until(n):
        return lambda c: c.gn_iterations_until(0, n, 1)

    # ---- overhead: config 2, the exit does not fire within 6 bodies
    cfg2 = synth.make_window(nF=8, pts_per_frame=250, seed=42)
    a, b = make_ctx(cfg2, stream), make_ctx(cfg2, stream)
    for c, run in ((a, fixed(6)), (b, until(6))):       # warm-up: captures, module loads
        timed(c, cfg2, stream, flush, run, 3)
    t, outs = pair(cfg2, stream, flush, args.reps, {"fixed6": (a, fixed(6)), "until6": (b, until(6))})
    n = b.iterations_run()
    result["cfg2"] = {"fixed6_ms": t["fixed6"], "until_ms": t["until6"], "until_bodies": n, "until_form": b.until_form(),
                      "overhead_us_per_body_median": 1e3 * (t["until6"][0] - t["fixed6"][0]) / 6,
                      "fixed_us_per_body_median": 1e3 * t["fixed6"][0] / 6,
                      "same_bits": bool(n == 6 and np.array_equal(outs["fixed6"], outs["until6"]))}
    a.close(); b.close()

    # ---- young window: 15 fixed bodies against the exit; the fallback's cost per body on the same window
    young = synth.make_window(nF=3, pts_per_frame=250, seed=4)
    a, b, h = make_ctx(young, stream), make_ctx(young, stream), make_ctx(young, stream, no_graph=True)
    for c, run in ((a, fixed(15)), (b, until(15)), (h, until(15))):
        timed(c, young, stream, flush, run, 3)
    t, outs = pair(young, stream, flush, args.reps, {"fixed15": (a, fixed(15)), "until15": (b, until(15)), "host15": (h, until(15))})
    n, nh = b.iterations_run(), h.iterations_run()
    a2 = make_ctx(young, stream)
    _, _, out_fixed_n = timed(a2, young, stream, flush, fixed(n), 1)
    a2.close()
    result["young_nF3"] = {"fixed15_ms": t["fixed15"], "until_ms": t["until15"], "until_bodies": n, "until_form": b.until_form(),
                           "host_driven_ms": t["host15"], "host_driven_bodies": nh, "host_driven_form": h.until_form(),
                           "host_driven_extra_us_per_body_median": 1e3 * (t["host15"][0] - t["until15"][0]) / max(n, 1),
                           "until_equals_fixed_n_bits": bool(np.array_equal(outs["until15"], out_fixed_n)),
                           "host_driven_equals_graph_bits": bool(nh == n and np.array_equal(outs["host15"], outs["until15"]))}
    a.close(); b.close(); h.close()
    print(json.dumps(result), flush=True)
    ok = result["cfg2"]["same_bits"] and result["young_nF3"]["until_equals_fixed_n_bits"] and result["young_nF3"]["host_driven_equals_graph_bits"]
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
