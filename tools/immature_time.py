"""Time the immature-point life cycle on the device store against the host-array entry points, on the bench-sized window
(640x480, 8 keyframes, 7 hosts with DetectCorners' features at 1500 = setting_desiredImmatureDensity):

  per frame     trace_new_coarse (store, no copies; followed by a synchronise)  vs  trace_immature (16 uploads, 6 read-backs)
  per keyframe  make_new_traces                                                  vs  detect_corners + immature_init
                activate_immature                                                vs  select_activation + optimize_immature

Each measurement is the host clock around calls that end in a synchronise, after the L2 cache has been flushed by writing 256 MB.
The two sides alternate in every round and the medians over --runs rounds are reported. Activation releases candidates, so
before each activation round the store is re-seeded and traced again (untimed); the host-array side gets the same candidates, read
back from the store. Needs a GPU. Prints one JSON line, with the card and its power limit.

    python tools/immature_time.py [--runs 30]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ldso_b200 import capi, synth  # noqa: E402

NFEAT = 1500


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("immature_time.py needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)
    flush_buf = torch.empty(64 << 20, dtype=torch.float32, device="cuda")

    def flush():
        flush_buf.zero_()
        torch.cuda.synchronize()

    def timed(fn):
        flush()
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    win = synth.make_window(nF=8, pts_per_frame=250, seed=42)
    tc = synth.make_trace_case(win, 1, seed=5)          # the per-host KRKi / Kt / aff of every (new, host) pair
    pattern = np.load(os.path.join(ROOT, "tests", "golden", "corners_synth_640x480.npz"))["pattern"]
    ctx = capi.Context(win.w, win.h, win.levels)
    ctx.set_orb_pattern(pattern)
    ctx.load_synth_window(win)
    ctx.upload_frame(8, win.pyramids[0])                # the keyframe seeded by the per-keyframe timing
    nF, new = win.nF, win.nF - 1
    hosts = np.arange(nF - 1, dtype=np.int32)
    feats = {int(f): ctx.make_new_traces(int(f), NFEAT) for f in hosts}
    n_cand = sum(len(v["u"]) for v in feats.values())
    K, t, a = tc.KRKi[new][hosts], tc.Kt[new][hosts], tc.aff[new][hosts]

    def reseed():
        for f in hosts:
            ctx.immature_seed(int(f), feats[int(f)]["u"], feats[int(f)]["v"])
        for fr in (nF - 2, nF - 1):
            ctx.trace_new_coarse(fr, hosts, tc.KRKi[fr][hosts], tc.Kt[fr][hosts], tc.aff[fr][hosts])
        ctx.synchronize()

    def host_arrays():
        segs = [ctx.immature_read(int(f)) for f in hosts]
        cat = {k: np.concatenate([s[k] for s in segs]) for k in segs[0]}
        cat["host"] = np.concatenate([np.full(len(s["u"]), i, np.int32) for i, s in enumerate(segs)])
        return cat

    # per frame: both sides trace the same candidates from the same state
    reseed()
    h = host_arrays()
    pts = dict(u=h["u"], v=h["v"], host=h["host"], color=h["color"], weights=h["weights"], gradH=h["gradH"], energyTH=h["energyTH"],
               idepth_min=h["idepth_min"].copy(), idepth_max=h["idepth_max"].copy(), quality=h["quality"].copy(), status=h["status"].copy(),
               uv=h["uv"].copy(), interval=h["interval"].copy())

    def store_trace():
        ctx.trace_new_coarse(new, hosts, K, t, a)
        ctx.synchronize()

    def host_trace():
        ctx.trace_immature(new, pts, K, t, a)

    def store_seed():
        ctx.make_new_traces(8, NFEAT)

    def host_seed():
        f = ctx.detect_corners(8, NFEAT)
        ctx.immature_init(8, f["u"], f["v"])

    for _ in range(3):
        store_trace(); host_trace(); store_seed(); host_seed()
    res = {k: [] for k in ("trace_store", "trace_host", "seed_store", "seed_host", "activate_store", "activate_host")}
    for r in range(args.runs):
        pair = [("trace_store", store_trace), ("trace_host", host_trace), ("seed_store", store_seed), ("seed_host", host_seed)]
        if r % 2:
            pair = [pair[1], pair[0], pair[3], pair[2]]
        for name, fn in pair:
            res[name].append(timed(fn))
    # per keyframe activation: a fresh store state every round
    flagged = np.zeros(nF, np.uint8); flagged[0] = 1
    n_sel = []
    for r in range(args.runs + 2):
        reseed()
        h = host_arrays()
        m = h["live"]
        c = {k: v[m] for k, v in h.items()}
        sel_args = (c["u"], c["v"], c["host"], c["idepth_min"], c["idepth_max"], c["status"], c["interval"], c["quality"], c["my_type"])

        def host_act():
            act = ctx.select_activation(new, 2.0, *sel_args, frame_flagged=flagged)
            s = act == 1
            ctx.optimize_immature(c["u"][s], c["v"][s], c["host"][s], c["idepth_min"][s], c["idepth_max"][s], c["color"][s], c["weights"][s],
                                  c["energyTH"][s])
            n_sel.append(int(s.sum()))

        def store_act():
            ctx.activate_immature(2.0, frame_flagged=flagged)

        if r % 2:
            ts = timed(store_act); th = timed(host_act)
        else:
            th = timed(host_act); ts = timed(store_act)
        if r >= 2:
            res["activate_host"].append(th); res["activate_store"].append(ts)
    ctx.close()
    med = {k: round(float(np.median(v)) * 1e3, 4) for k, v in res.items()}
    print(json.dumps({"card": card, "geometry": f"{win.w}x{win.h}, {len(hosts)} hosts, {n_cand} candidates, {NFEAT} features",
                      "unit": "ms (median, L2 flushed)", "runs": args.runs, "selected_per_activation": int(np.median(n_sel)), **med}))


if __name__ == "__main__":
    main()
